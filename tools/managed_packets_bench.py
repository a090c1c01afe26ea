#!/usr/bin/env python
"""Cost of the bitrate-managed device entropy coder (all 15 packets of every block).

First part: `--blocks` independent long stereo blocks (44.1 kHz, q 0.5, bench.py's synthetic PCM), timed with CUDA
events as
  A: vb200_encode_dsp_managed_dev alone
  B: vb200_encode_dsp_managed_dev + vb200_encode_entropy_managed_dev (the packets stay on the device)
alternating A and B in one process, `--reps` measurements of each.  A sample of blocks is checked against the
reference's own coder on every curve (oracle/encode_packets.py checker a).  The bytes per block that a host caller
copies back are counted from shapes and packet lengths: the 15 curves' posts, nonzero flags and int32 residue plus
ampmax (vb200_encode_dsp_managed) against the packets, their bit counts and offsets plus ampmax
(vb200_encode_packets_managed).

Second part, 128 kbit/s nominal stereo: `--driver-streams` streams of `--driver-secs` seconds (noise, tones and bursts)
through the managed multi-stream driver with the device coder and with the host path forced (vb200ms_set_host_entropy),
alternating, `--driver-reps` runs of each, then once through the stock reference encoder (one CPU thread, one stream
after another); wall clock, blocks per second, launches per round, and the streams whose packets differ from the
stock encoder's.

Prints one JSON line with the card's name and power limit read in the same run.  Needs a GPU and oracle/_ref.

usage: python tools/managed_packets_bench.py [--blocks 20000] [--reps 5] [--sample 200]
                                             [--driver-streams 16] [--driver-secs 4] [--driver-reps 2]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def device_part(a, torch):
    from bench import make_desc, synth_pcm_torch
    from oracle import encode_packets as ep
    from vorbis_b200 import abi
    NB = abi.PACKETBLOBS
    ch, rate, q, W = 2, 44100, 0.5, 1
    d = ep.Driver(ch, rate, q)
    ctx = d.ctx
    dev = torch.device("cuda", 0)
    N = ctx.bs[W]
    n, nb = N // 2, a.blocks
    pcm = synth_pcm_torch(torch, nb, ch, N, rate, dev, seed=1000)
    desc_np = make_desc(nb)
    desc = torch.from_numpy(desc_np.view(np.uint8).reshape(nb, 16).copy()).to(dev)
    posts = torch.empty((NB, nb, ch, abi.FLOOR1_STRIDE), device=dev, dtype=torch.int32)
    nonzero = torch.empty((NB, nb, ch), device=dev, dtype=torch.int32)
    iwork = torch.empty((NB, nb, ch, n), device=dev, dtype=torch.int32)
    amp = torch.empty(nb, device=dev, dtype=torch.float32)
    io = abi.EncodeIO()
    io.pcm, io.pcm_fmt, io.desc, io.independent = pcm.data_ptr(), 0, desc.data_ptr(), 1
    io.posts, io.nonzero, io.iwork, io.ampmax_out = posts.data_ptr(), nonzero.data_ptr(), iwork.data_ptr(), amp.data_ptr()
    stride = ctx.packet_bound(W)
    bits = torch.empty(NB * nb, device=dev, dtype=torch.int32)
    data = torch.empty(NB * nb * stride, device=dev, dtype=torch.uint8)
    sptr = torch.cuda.current_stream().cuda_stream
    import ctypes as C

    def dsp():
        ctx._chk(ctx.L.vb200_encode_dsp_managed_dev(ctx.h, W, nb, 1, C.byref(io), sptr))

    def both():
        dsp()
        ctx.encode_entropy_managed_dev(W, nb, nb, desc.data_ptr(), posts.data_ptr(), nonzero.data_ptr(),
                                       iwork.data_ptr(), stride, bits.data_ptr(), data.data_ptr(), stream=sptr)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(2):
        timed(dsp), timed(both)
    ta, tb = [], []
    for _ in range(a.reps):
        ta.append(timed(dsp))
        tb.append(timed(both))
    b = bits.cpu().numpy().reshape(NB, nb)
    k = min(a.sample, nb)
    dd = data.view(NB, nb, stride)[:, :k].cpu().numpy()
    want, _, _ = ep.ref_packets(ch, rate, q, W, np.concatenate([desc_np[:k]] * NB),
                                posts[:, :k].cpu().numpy().reshape(NB * k, ch, abi.FLOOR1_STRIDE),
                                nonzero[:, :k].cpu().numpy().reshape(NB * k, ch),
                                iwork[:, :k].cpu().numpy().reshape(NB * k, ch, n))
    same = all(bytes(dd[c, i, :(b[c, i] + 7) // 8]) == want[c * k + i] for c in range(NB) for i in range(k))
    pkt_bytes = float(np.mean(((b + 7) // 8).sum(0)))
    d.close()
    return {"blocks": nb, "reps": a.reps, "dsp_managed_ms": stats(ta), "dsp_managed_entropy_ms": stats(tb),
            "entropy_ms_median": float(np.median(tb) - np.median(ta)),
            "packet_bytes_per_block_15_curves_mean": pkt_bytes, "packet_bound": stride,
            "d2h_bytes_per_block": {
                "vb200_encode_dsp_managed": NB * 4 * ch * (abi.FLOOR1_STRIDE + 1 + n) + 4,
                "vb200_encode_packets_managed": pkt_bytes + NB * (4 + 8) + 4},
            "sample_blocks": k, "sample_identical_to_reference": bool(same)}


def driver_part(a):
    from oracle import encode_managed, managed
    if not (managed.available() and encode_managed.available()):
        return "not measured (oracle/_ref not built)"
    ch, rate, nominal = 2, 44100, 128000
    n = int(rate * a.driver_secs)
    rng = np.random.default_rng(5)
    t = np.arange(n) / rate
    pcm = np.empty((a.driver_streams, ch, n), np.float32)
    for s in range(a.driver_streams):
        x = 0.05 * rng.standard_normal((ch, n)) + 0.3 * np.sin(2 * np.pi * rng.uniform(100, 4000) * t)
        for b in rng.integers(0, n - 2000, 6):
            x[:, b:b + 2000] += rng.uniform(0.3, 0.8) * rng.standard_normal((ch, 2000))
        pcm[s] = np.clip(x, -1, 1)
    runs = {"device": [], "host": []}
    out = {}
    for _ in range(a.driver_reps):
        for host in (False, True):
            t0 = time.perf_counter()
            blocks, rounds, launches, got, on = encode_managed.ms_encode(ch, rate, -1, nominal, -1, pcm,
                                                                         host_entropy=host)
            runs["host" if host else "device"].append(time.perf_counter() - t0)
            out["host" if host else "device"] = (blocks, rounds, launches, got, on)
    t0 = time.perf_counter()
    stock = [managed.stock_summary(ch, rate, -1, nominal, -1, pcm[s])[1:] for s in range(a.driver_streams)]
    t_stock = time.perf_counter() - t0
    res = {"streams": a.driver_streams, "seconds_per_stream": a.driver_secs, "stock_s": t_stock}
    for k, (blocks, rounds, launches, got, on) in out.items():
        res[k] = {"on_device": on, "blocks": blocks, "rounds": rounds, "launches_per_round": launches / rounds,
                  "wall_s": runs[k], "blocks_per_s_best": blocks / min(runs[k]),
                  "streams_differing_from_stock": [i for i in range(len(stock)) if tuple(got[i]) != tuple(stock[i])]}
    res["stock_blocks_per_s"] = out["device"][0] / t_stock
    return res


def main():
    import torch
    from bench import gpu_identity
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=200)
    ap.add_argument("--driver-streams", type=int, default=16)
    ap.add_argument("--driver-secs", type=float, default=4.0)
    ap.add_argument("--driver-reps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    res = {"gpu": gpu_identity(0), "device_calls": device_part(a, torch), "drop_in": driver_part(a)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
