"""Where k_floor1_fit's time goes: runs bench.py's workload (the same synthetic signal, setup and
vb200_encode_dsp_dev call) with VB200_FLOOR1_TIMING set, so that the fit launches its DBG instance, and
prints the per-phase SM cycles per row and the per-row counters.  The marks are clock64() deltas summed
over every warp, so a phase's share is of the warps' latency, not of the kernel's wall time.

    python tools/floor1_phase_timing.py [--blocks 100000] [--reps 5]
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["VB200_FLOOR1_TIMING"] = "1"

import torch  # noqa: E402

import bench  # noqa: E402
from vorbis_b200 import abi, lib  # noqa: E402

# slot layout of k_floor1_fit<true> (F1_T_* / F1_C_* in vorbis_b200/csrc/vb200_floor1.cuh)
PHASES = ["q build", "accumulate_fit", "terms", "fit_line (row)", "split: inspect", "split: fit_line",
          "split: rest", "prediction+store"]
COUNTS = ["inspects", "fits", "NULL rows", "rows"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    setup = abi.SetupHolder.load(os.path.join(bench.GOLD, "setup_44k_stereo_q5.npz"))
    ctx = lib.Context(setup, device=0)
    N, ch = setup.blocksize(bench.W_LONG), setup.channels
    nb = args.blocks
    dev = torch.device("cuda", 0)
    pcm = bench.synth_pcm_torch(torch, nb, ch, N, setup.rate, dev, seed=1000)
    desc_np = bench.make_desc(nb)
    desc = torch.from_numpy(desc_np.view(np.uint8).reshape(nb, 16).copy()).to(dev)
    posts = torch.empty((nb, ch, abi.FLOOR1_STRIDE), device=dev, dtype=torch.int32)
    nonzero = torch.empty((nb, ch), device=dev, dtype=torch.int32)
    iwork = torch.empty((nb, ch, N // 2), device=dev, dtype=torch.int32)
    amp = torch.empty(nb, device=dev, dtype=torch.float32)
    io = abi.EncodeIO()
    io.pcm, io.pcm_fmt, io.desc, io.independent = pcm.data_ptr(), 0, desc.data_ptr(), 1
    io.posts, io.nonzero, io.iwork, io.ampmax_out = posts.data_ptr(), nonzero.data_ptr(), iwork.data_ptr(), amp.data_ptr()
    sptr = torch.cuda.current_stream().cuda_stream
    for _ in range(2):
        ctx.encode_dsp_dev(bench.W_LONG, nb, 1, io, blobno=7, stream=sptr)
    ctx.debug_phase_cycles(True)
    for _ in range(args.reps):
        ctx.encode_dsp_dev(bench.W_LONG, nb, 1, io, blobno=7, stream=sptr)
    cyc = np.array(ctx.debug_phase_cycles(True), dtype=np.float64)
    t, c = cyc[:len(PHASES)], cyc[len(PHASES):len(PHASES) + len(COUNTS)]
    rows = c[3]
    assert rows == nb * ch * args.reps, (rows, nb * ch * args.reps)
    p = torch.cuda.get_device_properties(0)
    ghz = p.clock_rate / 1e6                     # the device's maximum SM clock: the us figures are lower bounds
    print("%s, %d rows x %d reps" % (p.name, nb * ch, args.reps))
    for name, v in zip(PHASES, t):
        print("%-18s %8.0f cycles/row  %5.1f%%  (%.2f us @%.3f GHz)" % (name, v / rows, 100 * v / t.sum(),
                                                                        v / rows / ghz / 1e3, ghz))
    print("total              %8.0f cycles/row = %.2f us" % (t.sum() / rows, t.sum() / rows / ghz / 1e3))
    print("per row: %.2f inspects, %.2f split fits, %.4f NULL rows" % (c[0] / rows, c[1] / rows, c[2] / rows))
    if c[1]:
        print("per call: inspect %.0f cycles, split fit_line %.0f cycles" % (t[4] / c[0], t[5] / c[1]))


if __name__ == "__main__":
    main()
