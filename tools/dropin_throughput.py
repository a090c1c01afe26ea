#!/usr/bin/env python
"""Drop-in throughput (VERDICT r1 #5): N concurrent encoders driven by the multi-stream driver of
vorbis_b200/host/vb200_mapping0.c (their ready blocks go to the device together) on its device path (the packets are
entropy coded on the device) and with the host path forced (the reference's own floor1_encode and residue backend
write the bits on the host threads), against the stock reference encoder on one host thread, same streams, same box.
Prints one JSON object; packets are cross-checked by hash.  With VB200MS_PROFILE=1 the driver prints its phases
(envelope, blockout, stage, device call, host half; seconds) to stderr when each run closes.

usage: python tools/dropin_throughput.py [--streams 1000] [--seconds 2.0]
Needs oracle/_ref/*.so (built by __graft_entry__.build() where the reference sources exist)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pyref  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--streams", type=int, default=1000)
ap.add_argument("--seconds", type=float, default=2.0)
ap.add_argument("--stock-streams", type=int, default=64, help="streams encoded by the stock reference for the rate and the hash check")
args = ap.parse_args()
ch, rate, q = 2, 44100, 0.5
ns, n = args.streams, int(rate * args.seconds)
rng = np.random.default_rng(3)
t = np.arange(n, dtype=np.float32)
base = (0.25 * rng.uniform(-1, 1, (8, ch, n)) + 0.5 * np.sin(2 * np.pi * (440 + 110 * np.arange(ch)).reshape(1, ch, 1) * t / rate)).astype(np.float32)
for k in range(8):                                          # a few transients so that both block sizes occur
    for a in rng.integers(3000, n - 3000, 3):
        base[k, :, a:a + 200] *= 0.02
        base[k, :, a + 200:a + 260] = rng.uniform(-0.9, 0.9, (ch, 60))
pcm = np.ascontiguousarray(base[np.arange(ns) % 8])         # [ns][ch][n]: 8 distinct signals, cycled
from oracle import encode_packets  # noqa: E402
runs = {}
for host in (True, False):
    encode_packets.ms_encode(pcm[:min(ns, 16)], ch, rate, q, host_entropy=host)     # warm-up
    t0 = time.perf_counter()
    blocks, summ, on_device = encode_packets.ms_encode(pcm, ch, rate, q, host_entropy=host)
    runs[host] = (blocks, summ, on_device, time.perf_counter() - t0)
    assert on_device == (not host)
    assert blocks > 0, "multi-stream driver failed"
blocks, summ, _, dt_ms = runs[False]
assert [s for s in runs[True][1]] == summ, "the host and the device path give different packets"
counts = [s[0] for s in summ]
nbytes = [s[1] for s in summ]
hashes = [s[2] for s in summ]
L = pyref.lib()
L.ref_stock_encode_summary.restype = C.c_long
k = min(args.stock_streams, ns)
t0 = time.perf_counter()
sb = 0
for i in range(k):
    h, b, c = C.c_uint64(0), C.c_long(0), C.c_long(0)
    sb += L.ref_stock_encode_summary(ch, C.c_long(rate), C.c_float(q), pcm[i].ctypes.data_as(C.c_void_p), C.c_long(n), C.byref(h), C.byref(b), C.byref(c))
    assert (h.value, b.value, c.value) == (hashes[i], nbytes[i], counts[i]), "stream %d: packets differ from the stock reference" % i
dt_stock = time.perf_counter() - t0
pk = sum(counts)
print(json.dumps({
    "what": "N concurrent vorbis encoders (44.1 kHz stereo q=0.5, %.1f s each): multi-stream drop-in driver vs stock reference, one host thread each" % args.seconds,
    "streams": ns, "blocks": int(blocks), "packets": int(pk),
    "dropin_packets_per_s": pk / dt_ms, "dropin_blocks_per_s": blocks / dt_ms, "dropin_seconds": dt_ms,
    "dropin_realtime_factor": ns * args.seconds / dt_ms,
    "host_path_packets_per_s": pk / runs[True][3], "host_path_seconds": runs[True][3],
    "stock_streams_timed": k, "stock_packets_per_s": sum(counts[i] for i in range(k)) / dt_stock, "stock_blocks_per_s": sb / dt_stock,
    "stock_realtime_factor": k * args.seconds / dt_stock,
    "speedup_one_host_thread": (blocks / dt_ms) / (sb / dt_stock),
    "packets_identical_to_stock": True,
    "note": "dropin_*: the device path (one vb200_encode_packets call per block size and round); host_path_*: the same "
            "driver with the reference's floor1_encode and residue packing on the host threads"}))
