#!/usr/bin/env python
"""Full-rate against half-rate decode (vb200_synthesis_halfrate) on the workload of bench.py's
decode_dsp_4096streams_x33blocks_mixed_s16 leg: 44.1 kHz stereo q 0.5 (256/2048-sample blocks), 4096 streams x 33
blocks with one run of 8 short blocks per stream, random residue, random floor posts, int16 interleaved output.
One vb200_decode_dsp_dev call per launch (de-coupling + floor multiply + IMDCT + overlap-add); the copy that
restores the in-place residue before every launch is timed on its own and subtracted, as bench.py does.

The two modes alternate on one context, `--reps` measurements of each, every measurement the mean of
`--launches` launches between CUDA events.  Prints one JSON line: the card's name and power limit (read in the
same run), every measurement and the spread per mode.

usage:  python tools/halfrate_bench.py [--reps 7] [--launches 10] [--device 0]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import GOLD, gpu_identity  # noqa: E402
from vorbis_b200 import abi, lib  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream().cuda_stream
    setup = abi.SetupHolder.load(os.path.join(GOLD, "setup_44k_stereo_q5.npz"))
    ctx = lib.Context(setup, device=args.device)
    ch, bs = setup.channels, [setup.blocksize(0), setup.blocksize(1)]
    ns, nblk = 4096, 33
    Wrow = np.ones(nblk, np.int32)
    Wrow[12:20] = 0
    Wseq = np.tile(Wrow, (ns, 1))
    g = torch.Generator(device=dev)
    g.manual_seed(12345)
    modes = {}
    for hs in (0, 1):
        coef_off, pcm_off, coef_len, pcm_len = lib.synthesis_layout(Wseq, bs, ch, halfrate=bool(hs))
        modes[hs] = {"co": torch.from_numpy(coef_off).to(dev), "po": torch.from_numpy(pcm_off).to(dev),
                     "len": pcm_len, "pcm": torch.zeros((ns, pcm_len, ch), dtype=torch.int16, device=dev)}
    dW = torch.from_numpy(Wseq).to(dev)
    res0 = (torch.rand(coef_len, generator=g, device=dev) * 2 - 1) * 1e-2
    res = res0.clone()
    posts = torch.randint(0, 120, (ns * nblk * ch, abi.FLOOR1_STRIDE), generator=g, device=dev, dtype=torch.int32)
    present = torch.ones(ns * nblk * ch, dtype=torch.int32, device=dev)

    def launch(hs):
        m = modes[hs]
        res.copy_(res0)                               # the chain works in place on the residue
        ctx._chk(ctx.L.vb200_decode_dsp_dev(ctx.h, ns, nblk, dW.data_ptr(), m["co"].data_ptr(), res.data_ptr(),
                                            posts.data_ptr(), present.data_ptr(), m["po"].data_ptr(),
                                            m["pcm"].data_ptr(), 1, m["len"], stream))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.launches

    def mode(hs):
        ctx.synthesis_halfrate(hs, None)              # closed-form windows: the timing does not depend on them
        return timed(lambda: launch(hs)) - timed(lambda: res.copy_(res0))

    for hs in (0, 1, 0, 1):                           # warm-up: module load, table upload, scratch growth
        mode(hs)
    ms = {0: [], 1: []}
    for _ in range(args.reps):
        for hs in (0, 1):
            ms[hs].append(mode(hs))
    ctx.synthesis_halfrate(0)

    def spread(v):
        return {"min": min(v), "median": float(np.median(v)), "max": max(v)}

    full, half = ms[0], ms[1]
    out = {"tool": "halfrate_bench", "gpu": gpu_identity(args.device), "device_name": torch.cuda.get_device_name(dev),
           "workload": "decode_dsp_4096streams_x33blocks_mixed_s16", "streams": ns, "blocks_per_stream": nblk,
           "launches_per_measurement": args.launches, "reps": args.reps,
           "full_rate_ms": full, "half_rate_ms": half,
           "full_rate": spread(full), "half_rate": spread(half),
           "stereo_blocks_per_s": {"full_rate_median": ns * nblk / float(np.median(full)) * 1e3,
                                   "half_rate_median": ns * nblk / float(np.median(half)) * 1e3},
           "speedup_median": float(np.median(full) / np.median(half)),
           "speedup_range": [min(full) / max(half), max(full) / min(half)]}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
