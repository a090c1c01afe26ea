"""Raw PCM to packets: vb200_encode_pcm_packets (the LPC preamble and tail built on the device) against
vb200_encode_streams_packets_resume on timelines the CPU oracle prepared from the same PCM (oracle/lpc.py), N stereo
44.1 kHz VBR q0.5 streams fed in pieces of 1 s, the arms alternating.  Also times the case where the first write is the
whole file (the preamble's autocorrelation then runs over every sample of the stream), and, in a profiled pass of its
own, the LPC kernels alone (k_lpc_filter, k_pcm_timeline) from the CUDA activity trace.  Prints one JSON line per arm
and repetition with the card's name and power limit read in the same run; the packets of both arms must be equal.

    python tools/pcm_packets_bench.py --streams 500 --secs 20 --reps 2 [--out DIR]

Timelines are prepared for --distinct different signals and reused across the streams (the oracle's planner is slow);
the timings do not include that preparation."""
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


def signals(k, secs, rate):
    from test_plan_vs_ref import burst_signal
    n = int(rate * secs)
    return [burst_signal(2, rate, secs, 1 + i)[:, :n] for i in range(k)]


def resume_pass(ctx, tls, eofs, ns, piece):
    """arm (a): the oracle's timelines through vb200_encode_streams_packets_resume, 1 piece of input per call"""
    k = len(tls)
    carry = ctx.encode_carry_init(ns)
    pk = [[] for _ in range(ns)]
    times, end = [], 0
    total, stop = tls[0].shape[1], int(eofs[0])
    while not ctx.encode_carry_head(carry)["done"].all():
        end = min(end + piece, stop) if end < stop else total
        base = ctx.encode_carry_head(carry)["base"]
        lens = np.maximum(end - base, 0)
        pcm = np.zeros((ns, 2, max(int(lens.max()), 1)), np.float32)
        for s in range(ns):
            pcm[s, :, :lens[s]] = tls[s % k][:, base[s]:end]
        e = np.array([eofs[s % k] for s in range(ns)], np.int64) if end == total else None
        t0 = time.perf_counter()
        got = ctx.encode_streams_packets_resume(pcm, lens, carry, e, data_cap=ns * 131072)
        times.append(time.perf_counter() - t0)          # a host call: it ends in a stream synchronise
        for s in range(ns):
            pk[s] += got["packets"][s]
    return pk, times


def pcm_pass(ctx, pcms, ns, piece):
    """arm (b): the input through vb200_encode_pcm_packets, one write of `piece` samples per call, then the end"""
    k, n = len(pcms), pcms[0].shape[1]
    carry = ctx.encode_pcm_carry_init(ns)
    pk = [[] for _ in range(ns)]
    times = []
    while True:
        head = ctx.encode_pcm_carry_head(carry)
        if head["enc"]["done"].all():
            break
        raw, wr = head["raw_base"], head["written"]
        new = np.minimum(piece, n - wr)
        end = ((new == 0) & (head["ended"] == 0)).astype(np.int32)
        lens = wr + new - raw
        pcm = np.zeros((ns, 2, max(int(lens.max()), 1)), np.float32)
        for s in range(ns):
            pcm[s, :, :lens[s]] = pcms[s % k][:, raw[s]:raw[s] + lens[s]]
        t0 = time.perf_counter()
        got = ctx.encode_pcm_packets(pcm, lens, carry, end, data_cap=ns * 65536 * (2 + piece // 44100))
        times.append(time.perf_counter() - t0)
        for s in range(ns):
            pk[s] += got["packets"][s]
    return pk, times


def lpc_kernel_ms(fn):
    """device time of the LPC kernels in one run of fn, from torch.profiler's CUDA activity trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if "k_lpc_filter" in e.name or "k_pcm_timeline" in e.name:
            tag = e.name.split("(")[0].replace("void ", "")
            out[tag] = out.get(tag, 0.0) + e.device_time / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=500)
    ap.add_argument("--secs", type=float, default=20.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from oracle import lpc, pyoracle
    import refgold as G
    from test_gpu_encode_packets import _driver
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rate, piece, ns = 44100, 44100, a.streams
    d = _driver(2, rate, 0.5)
    ctx = d.ctx
    bs = tuple(ctx.bs)
    pcms = signals(a.distinct, a.secs, rate)
    n = pcms[0].shape[1]
    ora = pyoracle.Oracle(G.load_setup(2, rate, 0.5))
    writes = [piece] * (n // piece) + ([n % piece] if n % piece else [])
    prep = [lpc.timeline(ora, bs, p, writes) for p in pcms]
    tls, eofs = [t for t, _ in prep], [e for _, e in prep]
    rows = []
    base_row = {"streams": ns, "secs": a.secs, "piece_samples": piece, "gpu": gpu, "setup": "VBR q0.5 stereo 44.1 kHz"}
    small = max(2, min(ns, 8))                    # warm-up of every shape at a small size
    resume_pass(ctx, tls, eofs, small, piece)
    pcm_pass(ctx, pcms, small, piece)
    for rep in range(a.reps):
        for arm in ("resume on oracle timelines", "pcm_packets"):
            t0 = time.perf_counter()
            pk, times = (resume_pass(ctx, tls, eofs, ns, piece) if arm.startswith("resume") else
                         pcm_pass(ctx, pcms, ns, piece))
            wall = time.perf_counter() - t0
            if arm.startswith("resume"):
                want = pk
            else:
                assert pk == want, "the arms' packets differ"
            r = dict(base_row, arm=arm, rep=rep, calls=len(times), call_ms_median=float(np.median(times)) * 1e3,
                     calls_s=float(sum(times)), pass_s=wall)
            rows.append(r)
            print(json.dumps(r), flush=True)
    whole = None
    for rep in range(a.reps):
        pk, times = pcm_pass(ctx, pcms, ns, n)
        if whole is None:
            whole = pk
            assert all(pk[s] and pk[s][-1] for s in range(ns))
        r = dict(base_row, arm="pcm_packets, whole file in the first write", rep=rep, calls=len(times),
                 first_call_ms=times[0] * 1e3, calls_s=float(sum(times)), piece_samples=n)
        rows.append(r)
        print(json.dumps(r), flush=True)
    for label, p in (("1 s pieces", piece), ("whole file in the first write", n)):
        ms = lpc_kernel_ms(lambda: pcm_pass(ctx, pcms, ns, p))
        r = dict(base_row, arm="LPC kernels alone (profiled pass), " + label, kernel_ms=ms, piece_samples=p)
        rows.append(r)
        print(json.dumps(r), flush=True)
    d.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pcm_packets_bench.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
