#!/usr/bin/env python
"""Cost of the device entropy coder on bench.py's workload: 100 000 independent long stereo blocks (44.1 kHz, q 0.5,
bench.py's synthetic PCM), timed with CUDA events as
  A: vb200_encode_dsp_dev alone
  B: vb200_encode_dsp_dev + vb200_encode_entropy_dev (the packets stay on the device, strided by the packet bound)
alternating A and B in one process.  Also reports the packet sizes and, on a sample of blocks run through the
reference's own coder (oracle/encode_packets.py checker a), how many stage-0 residue vectors land on an unused
lattice entry, i.e. how often local_book_besterror's serial fallback search runs at stage 0.  Prints one JSON line
with the card's name and power limit read in the same run.  Needs a GPU and oracle/_ref (the setup comes from the
multi-stream driver, which builds it from the stock encoder).

usage: python tools/encode_packets_bench.py [--blocks 100000] [--reps 10] [--sample 2000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from bench import make_desc, synth_pcm_torch
    from oracle import encode_packets as ep
    from vorbis_b200 import abi
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample", type=int, default=2000)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    ch, rate, q, W = 2, 44100, 0.5, 1
    d = ep.Driver(ch, rate, q)
    ctx = d.ctx
    dev = torch.device("cuda", 0)
    N = ctx.bs[W]
    n, nb = N // 2, a.blocks
    pcm = synth_pcm_torch(torch, nb, ch, N, rate, dev, seed=1000)
    desc_np = make_desc(nb)
    desc = torch.from_numpy(desc_np.view(np.uint8).reshape(nb, 16).copy()).to(dev)
    posts = torch.empty((nb, ch, abi.FLOOR1_STRIDE), device=dev, dtype=torch.int32)
    nonzero = torch.empty((nb, ch), device=dev, dtype=torch.int32)
    iwork = torch.empty((nb, ch, n), device=dev, dtype=torch.int32)
    amp = torch.empty(nb, device=dev, dtype=torch.float32)
    io = abi.EncodeIO()
    io.pcm, io.pcm_fmt, io.desc, io.independent = pcm.data_ptr(), 0, desc.data_ptr(), 1
    io.posts, io.nonzero, io.iwork, io.ampmax_out = posts.data_ptr(), nonzero.data_ptr(), iwork.data_ptr(), amp.data_ptr()
    stride = ctx.packet_bound(W)
    bits = torch.empty(nb, device=dev, dtype=torch.int32)
    data = torch.empty(nb * stride, device=dev, dtype=torch.uint8)
    sptr = torch.cuda.current_stream().cuda_stream

    def dsp():
        ctx.encode_dsp_dev(W, nb, 1, io, blobno=7, stream=sptr)

    def both():
        dsp()
        ctx.encode_entropy_dev(W, nb, desc.data_ptr(), posts.data_ptr(), nonzero.data_ptr(), iwork.data_ptr(), stride,
                               bits.data_ptr(), data.data_ptr(), stream=sptr)

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
    b = bits.cpu().numpy()
    k = min(a.sample, nb)
    want, _, hits = ep.ref_packets(ch, rate, q, W, desc_np[:k], posts[:k].cpu().numpy(), nonzero[:k].cpu().numpy(),
                                   iwork[:k].cpu().numpy())
    dd = data.view(nb, stride)[:k].cpu().numpy()
    same = all(bytes(dd[i, :(b[i] + 7) // 8]) == want[i] for i in range(k))
    res = {"gpu": gpu, "blocks": nb, "reps": a.reps,
           "dsp_ms": {"median": float(np.median(ta)), "min": float(np.min(ta)), "max": float(np.max(ta))},
           "dsp_entropy_ms": {"median": float(np.median(tb)), "min": float(np.min(tb)), "max": float(np.max(tb))},
           "entropy_share_of_median": float(1 - np.median(ta) / np.median(tb)),
           "packet_bytes_mean": float(np.mean((b + 7) // 8)), "packet_bound": stride,
           "sample_blocks": k, "sample_identical_to_reference": bool(same),
           "stage0_unused_lattice_hits_per_block": hits / k}
    print(json.dumps(res))
    d.close()


if __name__ == "__main__":
    main()
