#!/usr/bin/env python
"""Bitrate-managed whole streams (vb200_encode_streams_managed_dev) on the mixed-block workload of bench.py's
streams leg: 44.1 kHz stereo q 0.5, int16 interleaved timelines with level drops and bursts (so the encoder
switches block sizes), every stream `--stream-blocks` long blocks long.  The managed outputs are 15 curves per
block, so the default job is smaller than the streams leg's 10000 streams.

The un-managed call (vb200_encode_streams_dev, blob 7) on the same streams alternates with the managed one on one
context, `--reps` measurements of each, every measurement the mean of `--launches` calls between CUDA events.  The
middle curve of the managed call is checked against the un-managed call's output.  Prints one JSON line: the
card's name and power limit (read in the same run), every measurement, blocks per second per mode.

Second part, 128 kbit/s nominal stereo: `--driver-streams` streams of `--driver-secs` seconds (noise, tones and
bursts) through the managed multi-stream driver (vb200ms_open_managed), through the single-block managed seam
(vorbis_analysis with vb200_mapping0_exportbundle, one stream after another) and through the stock reference
encoder (one CPU thread, one stream after another), wall clock each; the streams whose packets (count, bytes,
FNV-1a hash) differ from the stock encoder's are listed per path.  Needs oracle/_ref (built where the reference sources
exist); without it that part is reported as not measured.

usage:  python tools/managed_throughput.py [--streams 1000] [--stream-blocks 50] [--reps 5] [--launches 3]
                                            [--driver-streams 16] [--driver-secs 4]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import GOLD, gpu_identity, synth_timelines_s16  # noqa: E402
from vorbis_b200 import abi, lib  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=1000)
    ap.add_argument("--stream-blocks", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--driver-streams", type=int, default=16)
    ap.add_argument("--driver-secs", type=float, default=4.0)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    sptr = torch.cuda.current_stream().cuda_stream
    setup = abi.SetupHolder.load(os.path.join(GOLD, "setup_44k_stereo_q5.npz"))
    ctx = lib.Context(setup, device=args.device)
    ch, ns = setup.channels, args.streams
    bs0, bs1 = setup.blocksize(0), setup.blocksize(1)
    stride = ((args.stream_blocks + 2) * (bs1 // 2) + 3) & ~3
    pcm = synth_timelines_s16(torch, 0, ns, stride, ch, setup.rate, dev)
    max_blocks = stride // (bs0 // 2) + 8
    cap = [ns * (stride // (bs0 // 2) + 8) // 4 + 64, ns * (stride // (bs1 // 2) + 8)]
    plen = torch.full((ns,), stride, dtype=torch.int64, device=dev)

    def make_io(curves):
        io = abi.StreamsIO()
        plan = torch.zeros((ns, max_blocks, 6), dtype=torch.int32, device=dev)
        nblk = torch.zeros(ns, dtype=torch.int32, device=dev)
        io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = pcm.data_ptr(), lib.PCM_S16_INTERLEAVED, max_blocks, stride
        io.pcm_len, io.eof, io.plan, io.nblocks = plen.data_ptr(), None, plan.data_ptr(), nblk.data_ptr()
        keep = [plan, nblk]
        for w, bsz in ((0, bs0), (1, bs1)):
            io.cap[w] = cap[w]
            o = {"posts": torch.empty((curves, cap[w], ch, abi.FLOOR1_STRIDE), dtype=torch.int32, device=dev),
                 "nonzero": torch.empty((curves, cap[w], ch), dtype=torch.int32, device=dev),
                 "iwork": torch.empty((curves, cap[w], ch, bsz // 2), dtype=torch.int32, device=dev),
                 "ampmax_out": torch.empty(cap[w], dtype=torch.float32, device=dev)}
            io.posts[w], io.nonzero[w], io.iwork[w], io.ampmax_out[w] = (o[k].data_ptr() for k in ("posts", "nonzero", "iwork", "ampmax_out"))
            keep.append(o)
        return io, keep

    io_m, keep_m = make_io(abi.PACKETBLOBS)
    io_u, keep_u = make_io(1)

    def call(managed):
        rc = (ctx.L.vb200_encode_streams_managed_dev(ctx.h, ns, C.byref(io_m), sptr) if managed
              else ctx.L.vb200_encode_streams_dev(ctx.h, ns, abi.PACKETBLOBS // 2, C.byref(io_u), sptr))
        if rc:
            raise RuntimeError("rc %d: %s" % (rc, ctx.L.vb200_last_error()))

    for m in (True, False):
        call(m)
    torch.cuda.synchronize()
    counts = [int(io_m.count[0]), int(io_m.count[1])]
    assert counts == [int(io_u.count[0]), int(io_u.count[1])]
    for w in (0, 1):
        for k in ("posts", "nonzero", "iwork"):
            if not torch.equal(keep_m[2 + w][k][abi.PACKETBLOBS // 2, :counts[w]], keep_u[2 + w][k][0, :counts[w]]):
                raise RuntimeError("managed curve 7 differs from the un-managed call: W=%d %s" % (w, k))
    ms = {"managed": [], "unmanaged": []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.reps):
        for m in (True, False):
            e0.record()
            for _ in range(args.launches):
                call(m)
            e1.record()
            torch.cuda.synchronize()
            ms["managed" if m else "unmanaged"].append(e0.elapsed_time(e1) / args.launches)
    blocks = counts[0] + counts[1]
    res = {"gpu": gpu_identity(args.device), "streams": ns, "blocks": blocks, "short_blocks": counts[0],
           "long_blocks": counts[1], "ms": ms}
    for k, v in ms.items():
        res[k + "_blocks_per_s_median"] = blocks / (sorted(v)[len(v) // 2] * 1e-3)
    res["drop_in"] = driver_leg(args)
    print(json.dumps(res))


def fnv_summary(packets):
    """(count, bytes, hash) as oracle/ref_managed.c summarises a stream's packets"""
    h, m = 1469598103934665603, (1 << 64) - 1
    for p in packets:
        for b in p:
            h = ((h ^ b) * 1099511628211) & m
        h = ((h ^ len(p)) * 1099511628211) & m
    return len(packets), sum(len(p) for p in packets), h


def driver_leg(args):
    from oracle import managed, pyref
    if not (managed.available() and pyref.dropin_available()):
        return "not measured (oracle/_ref not built)"
    ch, rate, nominal = 2, 44100, 128000
    n = int(rate * args.driver_secs)
    rng = np.random.default_rng(5)
    t = np.arange(n) / rate
    pcm = np.empty((args.driver_streams, ch, n), np.float32)
    for s in range(args.driver_streams):
        x = 0.05 * rng.standard_normal((ch, n)) + 0.3 * np.sin(2 * np.pi * rng.uniform(100, 4000) * t)
        for b in rng.integers(0, n - 2000, 6):
            x[:, b:b + 2000] += rng.uniform(0.3, 0.8) * rng.standard_normal((ch, 2000))
        pcm[s] = np.clip(x, -1, 1)
    t0 = time.perf_counter()
    blocks, rounds, launches, got = managed.ms_encode(ch, rate, -1, nominal, -1, pcm, device=args.device)
    t_driver = time.perf_counter() - t0
    t0 = time.perf_counter()
    stock = [managed.stock_summary(ch, rate, -1, nominal, -1, pcm[s])[1:] for s in range(args.driver_streams)]
    t_stock = time.perf_counter() - t0
    t0 = time.perf_counter()
    seam = []
    for s in range(args.driver_streams):
        enc = pyref.Ref(ch, rate, nominal_bitrate=nominal, dropin=True, device=args.device)
        enc.L.ref_use_block_seam(1)
        try:
            enc.L.ref_encode_capture(enc.h, np.ascontiguousarray(pcm[s]), n, None, None)
        finally:
            enc.L.ref_use_block_seam(0)
        seam.append(enc.packets())
        enc.close()
    t_seam = time.perf_counter() - t0
    seam = [fnv_summary(p) for p in seam]
    return {"streams": args.driver_streams, "seconds_per_stream": args.driver_secs, "blocks": blocks,
            "rounds": rounds, "launches": launches, "driver_s": t_driver, "stock_s": t_stock, "seam_s": t_seam,
            "driver_blocks_per_s": blocks / t_driver, "stock_blocks_per_s": blocks / t_stock,
            "seam_blocks_per_s": blocks / t_seam,
            "driver_streams_differing_from_stock": [i for i in range(len(stock)) if tuple(got[i]) != tuple(stock[i])],
            "seam_streams_differing_from_stock": [i for i in range(len(stock)) if tuple(seam[i]) != tuple(stock[i])]}


if __name__ == "__main__":
    main()
