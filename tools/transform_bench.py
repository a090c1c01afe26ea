#!/usr/bin/env python
"""Time k_phaseA_transform alone, two builds of the library alternating in one process.

usage: tools/transform_bench.py OLD.so NEW.so [--rounds 6] [--steps 10] [--blocks 100000]

Both libraries run bench.py's workload (one vb200_encode_dsp_dev call on --blocks long stereo blocks of the
44.1 kHz q5 setup, the same PCM and block descriptors) on cuda:0.  Each round runs --steps calls of one library
with the library's per-kernel CUDA events on, then the same for the other; the order of the two alternates from
round to round.  Printed per round and library: the transform kernel's mean time, and the whole chain's (the sum
of the six kernel times).  The card's name, power limit and SM clock are printed beside the numbers.  Nothing is
written to the tree: the libraries are loaded from copies in a temporary directory."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload: setup, PCM and descriptors of bench.py)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def open_ctx(lib, path, setup):
    """a Context bound to the library at `path` (vorbis_b200.lib keeps one loaded library: swap it per build)"""
    lib._lib = None
    lib.LIB_PATH = path
    return lib.Context(setup, device=0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=100000)
    args = ap.parse_args()
    import torch
    from vorbis_b200 import abi, lib
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool times kernels on the GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    setup = abi.SetupHolder.load(os.path.join(bench.GOLD, "setup_44k_stereo_q5.npz"))
    tmp = tempfile.mkdtemp(prefix="transform_bench_")
    try:
        ctxs = {}
        for tag in ("old", "new"):
            p = os.path.join(tmp, "lib%s.so" % tag)
            shutil.copy(getattr(args, tag), p)
            ctxs[tag] = open_ctx(lib, p, setup)
        N, ch, nb = setup.blocksize(bench.W_LONG), setup.channels, args.blocks
        n = N // 2
        pcm = bench.synth_pcm_torch(torch, nb, ch, N, setup.rate, dev, seed=1000)
        desc_np = bench.make_desc(nb)
        desc = torch.from_numpy(desc_np.view(np.uint8).reshape(nb, 16).copy()).to(dev)
        outs = {}
        for tag in ctxs:
            o = {"posts": torch.empty((nb, ch, abi.FLOOR1_STRIDE), device=dev, dtype=torch.int32),
                 "nonzero": torch.empty((nb, ch), device=dev, dtype=torch.int32),
                 "iwork": torch.empty((nb, ch, n), device=dev, dtype=torch.int32),
                 "amp": torch.empty(nb, device=dev, dtype=torch.float32)}
            io = abi.EncodeIO()
            io.pcm, io.pcm_fmt, io.desc, io.independent = pcm.data_ptr(), 0, desc.data_ptr(), 1
            io.posts, io.nonzero, io.iwork = o["posts"].data_ptr(), o["nonzero"].data_ptr(), o["iwork"].data_ptr()
            io.ampmax_out = o["amp"].data_ptr()
            outs[tag] = (o, io)
        sptr = torch.cuda.current_stream().cuda_stream

        def run(tag, steps):
            ctx, (o, io) = ctxs[tag], outs[tag]
            ctx.set_profiling(True)
            kms = np.zeros(6)
            for _ in range(steps):
                ctx.encode_dsp_dev(bench.W_LONG, nb, 1, io, blobno=7, stream=sptr)
                torch.cuda.synchronize()
                kms += np.array(ctx.encode_dsp_kernel_ms())
            ctx.set_profiling(False)
            return kms / steps

        print("card: %s" % card())
        print("workload: %d long stereo blocks (N=%d), %d rows per call; %d calls per round and build"
              % (nb, N, nb * ch, args.steps))
        for tag in ctxs:
            run(tag, args.warmup)
        same = all(torch.equal(outs["old"][0][k], outs["new"][0][k]) for k in outs["old"][0])
        print("outputs of the two builds identical: %s" % same)
        res = {"old": [], "new": []}
        for r in range(args.rounds):
            order = ("old", "new") if r % 2 == 0 else ("new", "old")
            for tag in order:
                kms = run(tag, args.steps)
                res[tag].append(kms)
                print("round %d %-3s transform %.3f ms   chain %.3f ms   kernels %s"
                      % (r, tag, kms[0], kms.sum(), " ".join("%.3f" % v for v in kms)))
        for tag in ("old", "new"):
            t = np.array([k[0] for k in res[tag]])
            c = np.array([k.sum() for k in res[tag]])
            print("%-3s transform ms: min %.3f median %.3f max %.3f   chain ms: min %.3f median %.3f max %.3f"
                  % (tag, t.min(), np.median(t), t.max(), c.min(), np.median(c), c.max()))
        to = np.array([k[0] for k in res["old"]])
        tn = np.array([k[0] for k in res["new"]])
        print("transform: slowest new round %.3f ms vs fastest old round %.3f ms; median change %+.1f %%"
              % (tn.max(), to.min(), 100.0 * (np.median(tn) / np.median(to) - 1.0)))
        print("card after: %s" % card())
        for c in ctxs.values():
            c.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
