#!/usr/bin/env python
"""Random crops from many resident streams: (a) vb200_decode_streams_packets_dev of every stream a batch touches, then
one gather of the crops, against (b) vb200_decode_ranges_dev, alternating in one process.  Workload of
tools/decode_streams_bench.py: 44.1 kHz stereo at q = 0.5, 8 distinct encoded streams of 20 s repeated (default 500
resident streams), every packet resident on the device in one table.  Each batch is 256 seeded crops of 5 s: a
stream drawn uniformly, a start drawn uniformly below length[s] - L from vb200_decode_streams_index's lengths (run
once).  A second run keeps 10x more streams resident and asks for the same crops.

Reports per arm: crops/s and samples/s from CUDA events around the batch's calls (a: the decode and the gather;
b: the one call), ms per batch, launches per batch, device scratch bytes; and, from a separate torch.profiler pass,
the share of (b)'s kernel time spent in the plan kernel k_dr_plan.  Both arms' crops are checked equal on the first
batch before timing.  Prints one JSON line per measurement with the GPU's name and power limit read in the same run.

usage: python tools/decode_ranges_bench.py [--streams 500] [--seconds 20] [--crop 5] [--batch 256] [--batches 8]
       [--repeat 3] [--out DIR]
Needs oracle/_ref (built by __graft_entry__.build() where the reference sources exist) and a GPU.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import decode  # noqa: E402
from oracle import decode_packets as dp  # noqa: E402
from vorbis_b200 import abi  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_throughput import gpu_identity, signal  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=500)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--crop", type=float, default=5.0)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--repeat", type=int, default=3, help="alternations of the two arms")
    ap.add_argument("--resident-scale", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not (decode.available() and dp.available()):
        sys.exit("oracle/_ref decode libraries not built")
    import torch
    ch, rate, q = 2, 44100, 0.5
    L = int(a.crop * rate)
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i)) for i in range(a.distinct)]
    bufs, metas, off = [], [], 0
    for p in enc:
        m = p.audio.copy()
        m[:, 0] += off
        bufs.append(p.buf)
        metas.append(m)
        off += len(p.buf)
    buf = np.concatenate(bufs)
    mp = max(len(m) for m in metas)
    drv = dp.Driver(enc[0])
    ctx = drv.ctx
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    ident = gpu_identity()
    lines = []

    def table(n):
        npkt = np.array([len(metas[s % a.distinct]) for s in range(n)], np.int32)
        info = np.zeros((n, mp), abi.PACKET_INFO_DTYPE)
        for s in range(n):
            m = metas[s % a.distinct]
            info["offset"][s, :len(m)], info["bytes"][s, :len(m)] = m[:, 0], m[:, 1]
            info["granulepos"][s, :len(m)], info["e_o_s"][s, :len(m)], info["packetno"][s, :len(m)] = m[:, 2], m[:, 3], m[:, 4]
        return npkt, info

    npkt, info = table(a.streams)
    length = ctx.decode_streams_index(npkt, info, buf)["length"]
    rng = np.random.default_rng(2026)
    batches = []
    for _ in range(a.batches):
        s = rng.integers(0, a.streams, a.batch)
        start = (rng.random(a.batch) * (length[s] - L)).astype(np.int64)
        batches.append(np.array(list(zip(start, s, [L] * a.batch)), abi.PCM_RANGE_DTYPE))
    d_data = t(buf)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def resident(n):
        npkt_, info_ = table(n)
        return t(npkt_), t(info_.view(np.uint8)).view(-1, mp * abi.PACKET_INFO_DTYPE.itemsize), info_

    def arm_a(res, req, out):
        """decode every touched stream whole from fresh carries, then copy each crop out"""
        d_npkt, d_info, _ = res
        touched = np.unique(req["stream"])
        slot = {int(s): i for i, s in enumerate(touched)}
        n = len(touched)
        cap = int(length[touched].sum()) * ch
        carry = ctx.decode_streams_carry(n)
        sel = t(touched.astype(np.int64))
        pcm = torch.empty(cap, dtype=torch.float32, device=dev)
        base = torch.empty(n + 1, dtype=torch.int64, device=dev)
        dout = torch.empty(n * mp * abi.DECODED_PACKET_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        hb = np.concatenate([[0], np.cumsum(length[touched])])
        torch.cuda.synchronize()
        ev[0].record()
        sn, si = d_npkt.index_select(0, sel), d_info.index_select(0, sel)
        ctx.decode_streams_packets_dev(n, mp, sn.data_ptr(), si.data_ptr(), d_data.data_ptr(), carry.ptr, 0,
                                       pcm.data_ptr(), cap, base.data_ptr(), dout.data_ptr(), st)
        # one gather of every crop: element (r, c, j) of the batch is pcm[first[r][c] + j]
        first = np.array([[int(hb[slot[s]]) * ch + c * int(hb[slot[s] + 1] - hb[slot[s]]) + s0 for c in range(ch)]
                          for s0, s, _ in req.tolist()], np.int64)
        idx = t(first)[:, :, None] + ar
        torch.index_select(pcm, 0, idx.view(-1), out=out.view(-1))
        ev[1].record()
        torch.cuda.synchronize()
        carry.close()
        del idx
        # residue strided by packet slot (ch * blocksizes[1]/2 floats) + 40 B of tables per slot, 80 B per stream,
        # the packed PCM and the gather's int64 indices
        scratch = n * mp * (ch * (ctx.bs[1] // 2) * 4 + 40) + n * 80 + cap * 4 + len(req) * ch * L * 8
        # launches: 2 table gathers, 5 of the call, the index add and the crop gather
        return ev[0].elapsed_time(ev[1]), 2 + 5 + 2, scratch

    def arm_b(res, req, out, got):
        d_npkt, d_info, info_ = res
        d_req = t(req.view(np.uint8))
        l0 = ctx.launch_count()
        torch.cuda.synchronize()
        ev[0].record()
        ctx.decode_ranges_dev(len(info_), mp, d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(), len(req),
                              d_req.data_ptr(), 0, out.data_ptr(), L, got.data_ptr(), st)
        ev[1].record()
        torch.cuda.synchronize()
        nblk = (L // (ctx.bs[0] // 2)) + 3
        nres = ch * (2 * L + 3 * (ctx.bs[1] // 2))
        scratch = len(req) * (nblk * 40 + 12 + 4 * nres)
        return ev[0].elapsed_time(ev[1]), ctx.launch_count() - l0, scratch

    ar = torch.arange(L, dtype=torch.int64, device=dev)
    out_a = torch.empty((a.batch, ch, L), dtype=torch.float32, device=dev)
    out_b = torch.empty((a.batch, ch, L), dtype=torch.float32, device=dev)
    got = torch.empty(a.batch, dtype=torch.int32, device=dev)
    res = resident(a.streams)
    # both arms' crops equal on the first batch
    arm_a(res, batches[0], out_a)
    arm_b(res, batches[0], out_b, got)
    assert (got.cpu().numpy() == L).all()
    assert torch.equal(out_a.view(torch.int32), out_b.view(torch.int32)), "arms differ"
    for scale in (1, a.resident_scale):
        res = resident(a.streams * scale)
        for rep in range(a.repeat):
            for arm in ("a", "b"):
                ms = []
                for req in batches:
                    if arm == "a":
                        m, launches, scratch = arm_a(res, req, out_a)
                    else:
                        m, launches, scratch = arm_b(res, req, out_b, got)
                    ms.append(m)
                sec = sum(ms) / 1e3
                crops = a.batch * a.batches
                lines.append(dict(ident, arm="a: decode touched streams + gather" if arm == "a"
                                  else "b: vb200_decode_ranges_dev", resident_streams=a.streams * scale, run=rep,
                                  batches=a.batches, crops_per_batch=a.batch, crop_samples=L,
                                  crops_per_s=crops / sec, samples_per_s=crops * L / sec,
                                  ms_per_batch=float(np.mean(ms)), launches_per_batch=launches,
                                  scratch_bytes=scratch))
    # the plan kernel's share of (b)'s kernel time, in a profiled pass of its own
    from torch.profiler import ProfilerActivity, profile
    res = resident(a.streams)
    arm_b(res, batches[0], out_b, got)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for req in batches[:4]:
            arm_b(res, req, out_b, got)
    tot = plan = 0.0
    names = {}
    for e in prof.key_averages():
        if not str(getattr(e, "device_type", "")).endswith("CUDA"):
            continue
        dt = e.device_time_total
        tot += dt
        names[e.key[:60]] = dt
        if "k_dr_plan" in e.key:
            plan += dt
    lines.append(dict(ident, arm="b: profiled kernel time (torch.profiler, 4 batches)", plan_kernel_us=plan,
                      kernels_us=tot, plan_share=plan / tot if tot else None, kernels=names))
    drv.close()
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "decode_ranges_bench.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
