#!/usr/bin/env python
"""Whole streams from packets: the multi-stream decode driver's device path (vb200md, vorbis_b200/host/vb200_decode.c:
host header parse and blockin bookkeeping around vb200_decode_packets_resume_dev) against vb200_decode_streams_packets
(host form) on the same packets, fed 1, 4 and 16 packets per stream per call, alternating in one process.  Workload of
tools/decode_throughput.py: 44.1 kHz stereo at q = 0.5, 8 distinct encoded streams repeated (default 500 streams of
20 s).  Reports packets/s, samples/s, bytes copied device -> host per call and launches per call, and the kernel time of
the _dev form on device-resident packets from CUDA events.  Before timing, both arms' PCM is checked equal on the first
16 streams.  Prints one JSON line per measurement with the GPU's name and power limit read in the same run.

The per-call packet tables and packed packet bytes of the new call are built before timing: they are what a demuxer
hands over.  vb200md builds its own tables inside its rounds, which is part of what it costs.

usage: python tools/decode_streams_bench.py [--streams 500] [--seconds 20] [--distinct 8] [--repeat 2] [--out DIR]
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
from oracle import decode_packets as dp  # noqa: E402
from oracle import decode_streams as ds  # noqa: E402
from vorbis_b200 import abi  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_throughput import gpu_identity, signal  # noqa: E402


def calls_for(metas, pick, per, buf):
    """per-call (npkt, info, data) with `per` packets of every stream, the call's packets packed back to back"""
    n = [len(metas[i]) for i in pick]
    out = []
    for a in range(0, max(n), per):
        npkt = np.array([max(0, min(per, k - a)) for k in n], np.int32)
        info = np.zeros((len(pick), per), abi.PACKET_INFO_DTYPE)
        chunks, off = [], 0
        for s, i in enumerate(pick):
            m = metas[i][a:a + npkt[s]]
            for k, r in enumerate(m):
                chunks.append(buf[r[0]:r[0] + r[1]])
                info[s, k] = (off, r[2], r[1], r[3], r[4], 0)
                off += int(r[1])
        data = np.concatenate(chunks) if chunks else np.zeros(1, np.uint8)
        out.append((npkt, info, data))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=500)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--repeat", type=int, default=2, help="alternations of the two arms per packets-per-call")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not (decode.available() and dp.available()):
        sys.exit("oracle/_ref decode libraries not built")
    import torch
    ch, rate, q = 2, 44100, 0.5
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i)) for i in range(a.distinct)]
    bufs, metas, off = [], [], 0
    for p in enc:
        m = p.audio.copy()
        m[:, 0] += off
        bufs.append(p.buf)
        metas.append(m)
        off += len(p.buf)
    buf = np.concatenate(bufs)
    hdr = np.ascontiguousarray(enc[0].meta[:3])
    rows = np.cumsum([0] + [len(m) for m in metas])
    meta = np.concatenate(metas)
    drv = dp.Driver(enc[0])
    ctx = drv.ctx
    # the finished samples of every packet (the plan's fin), for vb200md's strided copy-back per round
    fin = []
    for i in range(a.distinct):
        ident = enc[0].buf[int(hdr[0, 0]):int(hdr[0, 0] + hdr[0, 1])]
        plan = ds.Plan([1 << int(ident[28] & 15), 1 << int(ident[28] >> 4)], 1)
        fin.append(plan.run(buf, metas[i])[:, 10])
    ident = gpu_identity()
    lines = []

    def joined_for(pick):
        return (buf, hdr, meta, rows[pick].astype(np.int64), np.array([len(metas[i]) for i in pick], np.int64))

    def run_new(calls, ns, keep=False):
        carry = ctx.decode_streams_carry(ns)
        pcm = [[] for _ in range(ns)] if keep else None
        n = d2h = 0
        for npkt, info, data in calls:
            r = ctx.decode_streams_packets(npkt, info, data, carry)
            n += int(r["pcm_base"][-1])
            d2h += 8 * (ns + 1) + abi.DECODED_PACKET_DTYPE.itemsize * info.size + 4 * ch * int(r["pcm_base"][-1])
            if keep:
                for s in range(ns):
                    pcm[s].append(r["pcm"][s])
        carry.close()
        return n, d2h, ([np.concatenate(p, axis=1) for p in pcm] if keep else None)

    # both arms' PCM equal on the first 16 streams, 4 packets per call
    pick = np.arange(min(16, a.streams)) % a.distinct
    sched = np.full((int(np.ceil(max(len(m) for m in metas) / 4)) + 1, len(pick)), 4, np.int32)
    want, _ = dp.md_run(joined_for(pick), sched, ch)
    _, _, got = run_new(calls_for(metas, pick, 4, buf), len(pick), keep=True)
    for s in range(len(pick)):
        assert np.array_equal(got[s].view(np.uint32), want[s].view(np.uint32)), "arms differ on stream %d" % s

    pick = np.arange(a.streams) % a.distinct
    joined = joined_for(pick)
    packets = int(joined[4].sum())
    for per in (1, 4, 16):
        calls = calls_for(metas, pick, per, buf)
        rounds = len(calls)
        sched = np.full((rounds + 1, a.streams), per, np.int32)
        md_d2h = 0
        for c in range(rounds):
            md_d2h += 4 * a.streams * ch * max(1, max(int(fin[i][c * per:(c + 1) * per].sum()) for i in range(a.distinct)))
        for rep in range(a.repeat):
            t0 = time.perf_counter()
            _, st = dp.md_run(joined, sched, ch, keep=False)
            dt = time.perf_counter() - t0
            n = int(st["samples"].sum())
            lines.append(dict(ident, arm="a: vb200md device path", packets_per_call=per, run=rep, streams=a.streams,
                              packets=packets, seconds=dt, packets_per_s=packets / dt, samples_per_s=n / dt,
                              calls=st["rounds"], d2h_bytes_per_call=md_d2h / rounds,
                              launches_per_call=st["launches"] / st["rounds"]))
            l0 = ctx.launch_count()
            t0 = time.perf_counter()
            n2, d2h, _ = run_new(calls, a.streams)
            dt = time.perf_counter() - t0
            assert n2 == n, "samples %d != %d" % (n2, n)
            lines.append(dict(ident, arm="b: vb200_decode_streams_packets host form", packets_per_call=per, run=rep,
                              streams=a.streams, packets=packets, seconds=dt, packets_per_s=packets / dt,
                              samples_per_s=n2 / dt, calls=rounds, d2h_bytes_per_call=d2h / rounds,
                              launches_per_call=(ctx.launch_count() - l0) / rounds))
        # the _dev form's kernel time on device-resident packets, CUDA events around every call
        dev = torch.device("cuda", 0)
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
        dcalls = [(t(npkt), t(info.view(np.uint8)), t(data), info.shape[1]) for npkt, info, data in calls]
        cap = a.streams * per * 1024 * ch
        d_pcm = torch.empty(cap, dtype=torch.float32, device=dev)
        d_base = torch.empty(a.streams + 1, dtype=torch.int64, device=dev)
        d_out = torch.empty(a.streams * per * abi.DECODED_PACKET_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        carry = ctx.decode_streams_carry(a.streams)
        st = torch.cuda.current_stream().cuda_stream
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        for d_npkt, d_info, d_data, mp in dcalls:
            ctx.decode_streams_packets_dev(a.streams, mp, d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(),
                                           carry.ptr, 0, d_pcm.data_ptr(), cap, d_base.data_ptr(), d_out.data_ptr(), st)
        ev[1].record()
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1])
        carry.close()
        lines.append(dict(ident, arm="b: _dev form, device-resident packets, CUDA events", packets_per_call=per,
                          streams=a.streams, packets=packets, seconds=ms / 1e3, packets_per_s=packets / (ms / 1e3),
                          samples_per_s=n / (ms / 1e3), calls=rounds, ms_per_call=ms / rounds))
        del dcalls
    drv.close()
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "decode_streams_bench.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
