#!/usr/bin/env python
"""Decode throughput of many streams: the stock decoder (vorbis_synthesis -> blockin -> pcmout) on all host threads
against the multi-stream decode driver (vb200md_*, vorbis_b200/host/vb200_decode.c) fed 1, 4 and 16 packets per
stream per round, on its device path (packets decoded by vb200_decode_packets_resume_dev) and on the forced host
entropy path (vb200md_set_host_entropy).  Default workload: 1000 streams of 44.1 kHz stereo at q = 0.5, 30 s each (8 distinct encoded
streams, repeated).  Prints one JSON line per configuration and the GPU's name and power limit read in the same run.

usage: python tools/decode_throughput.py [--streams 1000] [--seconds 30] [--distinct 8] [--out DIR]
Needs oracle/_ref (built by __graft_entry__.build() where the reference sources exist) and a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import decode  # noqa: E402
from oracle import decode_packets  # noqa: E402


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, watts = [x.strip() for x in out.split(",")[:2]]
    return {"gpu": name, "power_limit_w": float(watts)}


def signal(ch, rate, secs, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(int(rate * secs)) / rate
    f = rng.uniform(150, 2000, (ch, 3))
    x = sum(0.2 * np.sin(2 * np.pi * f[:, k:k + 1] * t * (1 + 0.01 * np.sin(t))) for k in range(3))
    return (x + 0.02 * rng.standard_normal(x.shape)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=1000)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/decode_throughput.jsonl")
    a = ap.parse_args()
    if not (decode.available() and decode_packets.available()):
        sys.exit("oracle/_ref/libvorbis_{ref,dropin}_decode.so not built")
    ch, rate, q = 2, 44100, 0.5
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i)) for i in range(a.distinct)]
    bufs, metas, off = [], [], 0
    for p in enc:
        m = p.audio.copy()
        m[:, 0] += off
        bufs.append(p.buf)
        metas.append(m)
        off += len(p.buf)
    rows = np.cumsum([0] + [len(m) for m in metas])
    meta = np.concatenate(metas)
    pick = np.arange(a.streams) % a.distinct
    joined = (np.concatenate(bufs), np.ascontiguousarray(enc[0].meta[:3]), meta, rows[pick].astype(np.int64),
              np.array([len(metas[i]) for i in pick], np.int64))
    packets = int(joined[4].sum())
    lines = []
    ident = gpu_identity()

    t0 = time.perf_counter()
    samples = decode.stock_decode_many(joined)
    dt = time.perf_counter() - t0
    lines.append(dict(ident, config="stock decoder, all host threads (%d)" % os.cpu_count(), streams=a.streams,
                      packets=packets, seconds=dt, packets_per_s=packets / dt, samples_per_s=samples / dt))
    for per in (1, 4, 16):
        sched = np.full((1, a.streams), per, np.int32)
        rounds = int(np.ceil(joined[4].max() / per)) + 1
        sched = np.repeat(sched, rounds, axis=0)
        for host in (False, True):
            t0 = time.perf_counter()
            _, st = decode_packets.md_run(joined, sched, ch, host_entropy=host, keep=False)
            dt = time.perf_counter() - t0
            n = int(st["samples"].sum())
            assert n == samples, "driver samples %d != stock %d" % (n, samples)
            assert st["entropy_on_device"] == (not host)
            lines.append(dict(ident, config="vb200md %s path, %d packets per stream per round"
                              % ("host" if host else "device", per), streams=a.streams,
                              packets=packets, seconds=dt, packets_per_s=packets / dt, samples_per_s=n / dt,
                              rounds=st["rounds"], device_ms_per_round=1e3 * st["device_s"] / st["rounds"],
                              host_ms_per_round=1e3 * st["host_s"] / st["rounds"],
                              launches_per_round=st["launches"] / st["rounds"]))
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "decode_throughput.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
