"""Whole streams to packets in pieces: vb200_encode_streams_packets[_managed]_resume fed N stereo 44.1 kHz streams in
pieces of 20 ms, 100 ms and 1 s, against one vb200_encode_streams_packets[_managed] call on the same timelines.
Prints per-call latency (median of a pass), blocks/s over the pass and kernel launches per call, one JSON line per
arm and repetition; the arms alternate.  The packets of every pieced pass must equal the one call's.

    python tools/stream_resume_bench.py --streams 32 --secs 5 --reps 3 [--managed] [--out DIR]

The timelines are synthetic (a zero preamble of blocksizes[1]/2 samples, the PCM, a zero tail): LPC extrapolation
stays with the caller, and the planner does not care where the samples came from."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def timelines(ns, secs, rate, half, seed=1):
    from test_plan_vs_ref import burst_signal
    n = int(rate * secs)
    tl = np.zeros((ns, 2, half + n + 4 * half), np.float32)
    for s in range(ns):
        tl[s, :, half:half + n] = burst_signal(2, rate, secs, seed + s)[:, :n]
    return tl, np.full(ns, tl.shape[2], np.int64), np.full(ns, half + n, np.int64)


def pieced(ctx, tl, eof, piece, managed):
    """feed every stream in pieces of `piece` samples; returns (packets per stream, call times, launches, calls)"""
    ns, ch, total = tl.shape
    carry = ctx.encode_carry_init(ns)
    pk = [[] for _ in range(ns)]
    times, launches, end = [], 0, 0
    while not ctx.encode_carry_head(carry)["done"].all():
        # the samples up to EOF in pieces, then the extrapolated tail with eof (a tail that arrived without eof
        # would be planned as ordinary samples)
        stop = int(eof.max())
        end = min(end + piece, stop) if end < stop else total
        base = ctx.encode_carry_head(carry)["base"]
        lens = np.maximum(end - base, 0)
        stride = max(int(lens.max()), ctx.bs[1]) + 3 & ~3
        pcm = np.zeros((ns, ch, stride), np.float32)
        for s in range(ns):
            pcm[s, :, :lens[s]] = tl[s, :, base[s]:end]
        e = eof if end == total else np.zeros(ns, np.int64)
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        got = ctx.encode_streams_packets_resume(pcm, lens, carry, e, managed=managed)
        times.append(time.perf_counter() - t0)          # a host call: it ends in a stream synchronise
        launches += ctx.launch_count() - l0
        for s in range(ns):
            pk[s] += got["packets"][s]
    return pk, times, launches, len(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32)
    ap.add_argument("--secs", type=float, default=5.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--managed", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    name = "ABR 128 kbit/s" if a.managed else "VBR q0.5"
    rate = 44100
    if a.managed:
        from oracle import bitrate as B
        d = B.ManagedDriver(2, rate, -1, 128000, -1)
        ctx = d.ctx
        ctx.bitrate_setup(B.ref_bitrate_info(B.managed(2, rate, -1, 128000, -1))[0])
    else:
        from test_gpu_encode_packets import _driver
        d = _driver(2, rate, 0.5)
        ctx = d.ctx
    tl, pcm_len, eof = timelines(a.streams, a.secs, rate, ctx.bs[1] // 2)
    pieces = {"20ms": rate // 50, "100ms": rate // 10, "1s": rate}
    rows = []
    one = ctx.encode_streams_packets(tl, pcm_len, eof, managed=a.managed)      # warm-up of every shape
    for p in pieces.values():
        pieced(ctx, tl, eof, p, a.managed)
    blocks = int(one["nblocks"].sum())
    for rep in range(a.reps):
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        one = ctx.encode_streams_packets(tl, pcm_len, eof, managed=a.managed)
        t = time.perf_counter() - t0
        rows.append({"arm": "one call", "rep": rep, "calls": 1, "call_ms": t * 1e3, "blocks_per_s": blocks / t,
                     "launches_per_call": ctx.launch_count() - l0})
        for label, p in pieces.items():
            pk, times, launches, calls = pieced(ctx, tl, eof, p, a.managed)
            assert pk == one["packets"], label
            rows.append({"arm": label, "rep": rep, "calls": calls, "call_ms": float(np.median(times)) * 1e3,
                         "blocks_per_s": blocks / sum(times), "launches_per_call": launches / calls})
        for r in rows[-1 - len(pieces):]:
            r.update({"streams": a.streams, "secs": a.secs, "blocks": blocks, "managed": a.managed, "gpu": gpu,
                      "setup": name})
            print(json.dumps(r))
    d.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "stream_resume_%s.json" % ("managed" if a.managed else "unmanaged")), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
