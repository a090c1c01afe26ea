#!/usr/bin/env python
"""Whole streams to stream-ordered packets: vb200_encode_streams_packets[_managed] against what a caller had to do
before it existed.

Job: `--streams` stereo streams of `--secs` seconds at 44.1 kHz (noise, a tone and loud bursts, seeded), each on a
timeline of a zero preamble, the PCM and a zero tail, with EOF set.  The context is a managed multi-stream driver's
(vb200ms_open_managed, 128 kbit/s nominal), which carries the managed encoder's setup and entropy setup; the bitrate
manager is its ci->bi (128 kbit/s average, 256 000 reservoir bits, bias 0.1, damping 1.5).

Managed, alternating, `--reps` times each:
  (a) before: H2D of the timelines, vb200_encode_streams_managed_dev, the plan back to the host to build the batches'
      lW / nW, vb200_encode_entropy_managed_dev per size, all 15 packets of every block back (bit counts, then the
      strided packet buffer), and on the host the bitrate manager along every stream (the CPU oracle's restatement of
      lib/bitrate.c, one C call per stream) and the packing of the kept packets in stream order
  (b) vb200_encode_streams_packets_managed
Un-managed (blob 7), the same pair with vb200_encode_streams_dev + vb200_encode_entropy_dev and a host reorder.
Wall time (host clock around work that ends in a synchronise), device-to-host bytes per block and kernel launches per
call; the packets of (a) and (b) are compared.  Prints one JSON line with the card's name and power limit read in the
same run.  Needs a GPU and oracle/_ref.

usage: python tools/stream_packets_bench.py [--streams 100] [--secs 12] [--reps 3]
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


def signals(ns, ch, rate, secs, half1):
    rng = np.random.default_rng(7)
    n = int(rate * secs)
    t = np.arange(n) / rate
    stride = (half1 + n + 4 * half1 + 3) & ~3
    tl = np.zeros((ns, ch, stride), np.float32)
    for s in range(ns):
        x = 0.05 * rng.standard_normal((ch, n)) + 0.3 * np.sin(2 * np.pi * rng.uniform(100, 4000) * t)
        for b in rng.integers(0, n - 2000, int(secs * 2)):
            x[:, b:b + 2000] += rng.uniform(0.3, 0.8) * rng.standard_normal((ch, 2000))
        tl[s, :, half1:half1 + n] = np.clip(x, -1, 1)
    pcm_len = np.full(ns, stride, np.int64)
    eof = np.full(ns, half1 + n, np.int64)
    return tl, pcm_len, eof


def arm_before(ctx, torch, tl, pcm_len, eof, cap, managed, info, count_out):
    """(a): the separate calls, all packets back, the choice and the packing on the host; returns (per-stream packet
    lists, D2H bytes)"""
    from oracle import bitrate as B
    from vorbis_b200 import abi
    NB = abi.PACKETBLOBS
    curves = NB if managed else 1
    ns, ch, stride = tl.shape
    dev = torch.device("cuda", 0)
    sptr = torch.cuda.current_stream().cuda_stream
    max_blocks = stride // (ctx.bs[0] // 2) + 8
    d2h = 0
    g = {"pcm": torch.from_numpy(tl).to(dev), "len": torch.from_numpy(pcm_len).to(dev), "eof": torch.from_numpy(eof).to(dev),
         "plan": torch.zeros(ns * max_blocks * 6, dtype=torch.int32, device=dev),
         "nb": torch.zeros(ns, dtype=torch.int32, device=dev)}
    io = abi.StreamsIO()
    io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = g["pcm"].data_ptr(), 1, max_blocks, stride
    io.pcm_len, io.eof, io.plan, io.nblocks = g["len"].data_ptr(), g["eof"].data_ptr(), g["plan"].data_ptr(), g["nb"].data_ptr()
    for w in range(2):
        n = ctx.bs[w] // 2
        io.cap[w] = cap[w]
        for k, shape in (("posts", (curves, cap[w], ch, abi.FLOOR1_STRIDE)), ("nonzero", (curves, cap[w], ch)),
                         ("iwork", (curves, cap[w], ch, n))):
            g[k + str(w)] = torch.empty(shape, dtype=torch.int32, device=dev)
        g["amp" + str(w)] = torch.empty(cap[w], dtype=torch.float32, device=dev)
        io.posts[w], io.nonzero[w] = g["posts%d" % w].data_ptr(), g["nonzero%d" % w].data_ptr()
        io.iwork[w], io.ampmax_out[w] = g["iwork%d" % w].data_ptr(), g["amp%d" % w].data_ptr()
    if managed:
        ctx._chk(ctx.L.vb200_encode_streams_managed_dev(ctx.h, ns, C.byref(io), sptr))
    else:
        ctx._chk(ctx.L.vb200_encode_streams_dev(ctx.h, ns, 7, C.byref(io), sptr))
    count = [io.count[0], io.count[1]]
    count_out[:] = count
    plan = g["plan"].cpu().numpy().view(abi.STREAM_BLOCK_DTYPE).reshape(ns, max_blocks)
    nblocks = g["nb"].cpu().numpy()
    d2h += plan.nbytes + nblocks.nbytes
    bits, data = {}, {}
    for w in range(2):
        cnt = count[w]
        if not cnt:
            continue
        desc = np.zeros(cnt, abi.BLOCKDESC_DTYPE)
        for s in range(ns):
            p = plan[s, :nblocks[s]]
            p = p[p["W"] == w]
            desc["lW"][p["slot"]], desc["nW"][p["slot"]] = p["lW"], p["nW"]
        dd = torch.from_numpy(desc.view(np.uint8).copy()).to(dev)
        bound = ctx.packet_bound(w)
        db = torch.empty(curves * cnt, dtype=torch.int32, device=dev)
        ds = torch.empty(curves * cnt * bound, dtype=torch.uint8, device=dev)
        if managed:
            ctx.encode_entropy_managed_dev(w, cnt, cap[w], dd.data_ptr(), g["posts%d" % w].data_ptr(),
                                           g["nonzero%d" % w].data_ptr(), g["iwork%d" % w].data_ptr(), bound,
                                           db.data_ptr(), ds.data_ptr(), stream=sptr)
        else:
            ctx.encode_entropy_dev(w, cnt, dd.data_ptr(), g["posts%d" % w].data_ptr(), g["nonzero%d" % w].data_ptr(),
                                   g["iwork%d" % w].data_ptr(), bound, db.data_ptr(), ds.data_ptr(), stream=sptr)
        bits[w] = db.cpu().numpy().reshape(curves, cnt)
        data[w] = ds.cpu().numpy().reshape(curves, cnt, bound)
        d2h += bits[w].nbytes + data[w].nbytes
    out = []
    for s in range(ns):
        p = plan[s, :nblocks[s]]
        Ws, slots = p["W"], p["slot"]
        if managed:
            pb = np.zeros((len(p), NB), np.int32)
            for w in (0, 1):
                sel = Ws == w
                if sel.any():
                    pb[sel] = bits[w][:, slots[sel]].T
            choice, nbytes, _ = B.vbo_bitrate_addblock(info, 44100, ctx.bs, Ws, pb)
        else:
            choice = np.zeros(len(p), np.int32)
            nbytes = np.array([(bits[int(w)][0, sl] + 7) // 8 for w, sl in zip(Ws, slots)], np.int64)
        pk = []
        for w, sl, c, nbt in zip(Ws, slots, choice, nbytes):
            nat = (int(bits[int(w)][c, sl]) + 7) // 8
            raw = data[int(w)][c, sl, :min(nat, nbt)].tobytes()
            pk.append(raw + bytes(int(nbt) - len(raw)))
        out.append(pk)
    return out, d2h


def main():
    import torch
    from bench import gpu_identity
    from oracle import bitrate as B
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=100)
    ap.add_argument("--secs", type=float, default=12.0)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    if not B.ref_available(True):
        sys.exit("oracle/_ref not built")
    ch, rate = 2, 44100
    d = B.ManagedDriver(ch, rate, -1, 128000, -1)
    ctx = d.ctx
    info, _ = B.ref_bitrate_info(B.managed(ch, rate, nominal_br=128000))
    ctx.bitrate_setup(info)
    tl, pcm_len, eof = signals(a.streams, ch, rate, a.secs, ctx.bs[1] // 2)
    need = ctx.encode_streams_packets(tl[:, :, :], pcm_len, eof, cap=[1, 1], data_cap=1, check=False)["count"]
    cap = [max(need[0], 1), max(need[1], 1)]
    res = {"gpu": gpu_identity(0), "streams": a.streams, "secs": a.secs, "reps": a.reps, "count": need}
    for managed in (True, False):
        data_cap = a.streams * (tl.shape[2] // 64) * 64 + (1 << 20)
        wall = {"a": [], "b": []}
        launches, d2h = {}, {}
        same = True
        for rep in range(a.reps + 1):                   # the first round warms both arms up
            for arm in ("a", "b"):
                torch.cuda.synchronize()
                l0 = ctx.launch_count()
                t0 = time.perf_counter()
                if arm == "a":
                    cnt = [0, 0]
                    pk, nbytes = arm_before(ctx, torch, tl, pcm_len, eof, cap, managed, info, cnt)
                else:
                    got = ctx.encode_streams_packets(tl, pcm_len, eof, cap=cap, managed=managed, data_cap=data_cap)
                    pk = got["packets"]
                    nbytes = (int(got["info"]["bytes"].sum()) + got["info"].nbytes + got["plan"].nbytes +
                              got["nblocks"].nbytes)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if rep:
                    wall[arm].append(dt)
                launches[arm] = ctx.launch_count() - l0
                d2h[arm] = nbytes
                if arm == "a":
                    ref_pk = pk
                else:
                    same = same and pk == ref_pk
        blocks = sum(need)
        res["managed" if managed else "unmanaged"] = {
            "blocks": blocks,
            "a_before_s": {"median": float(np.median(wall["a"])), "min": float(np.min(wall["a"]))},
            "b_streams_packets_s": {"median": float(np.median(wall["b"])), "min": float(np.min(wall["b"]))},
            "d2h_bytes_per_block": {k: v / blocks for k, v in d2h.items()},
            "launches": launches, "packets_identical": bool(same)}
    d.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
