#!/usr/bin/env python
"""Grouping demuxed Ogg files by setup: the host way against one vb200_ogg_group_dev call.

Workload: --files Ogg files (default 500 and 5000) of --setups distinct stock setups (default 6, in 4-8), interleaved
in a seeded order; every file has its own comment header (a title tag with its index), so no two files share all
three header packets.  The files are resident on the device and demuxed once (vb200_ogg_demux_dev); each arm starts
from the demux's device tables and ends with each group a contiguous run of the packet tables:
  (a) host: streams back, every file's header packets (identification, comment, setup: one byte range per file) copied
      back into pinned memory, grouped by (identification, setup) bytes in a dict, the order sent up, and the npkt and
      info rows permuted with index_select;
  (b) device: one vb200_ogg_group_dev call (status, order, permuted tables, groups).
Both arms give the same order and groups (checked).  Times are wall clock around work that ends in a device
synchronise, the two arms alternated over --repeat runs; (b) also by CUDA events.  Prints one JSON line per file
count with the GPU's name and power limit read in the same run.

usage: python tools/ogg_group_bench.py [--files 500 5000] [--setups 6] [--seconds 2] [--repeat 7] [--out DIR]
Needs oracle/_ref (built by __graft_entry__.build() where the reference sources exist) for the stock encoder, and a GPU.
"""
import argparse
import json
import os
import struct
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import decode  # noqa: E402
from oracle import ogg  # noqa: E402
from vorbis_b200 import abi, lib  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_throughput import gpu_identity, signal  # noqa: E402

SETUPS = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2), (2, 44100, -0.1), (2, 48000, 0.9), (1, 44100, 0.4),
          (2, 32000, 0.0), (4, 48000, 0.1)]


def comment_packet(tag):
    vendor = b"ogg_group_bench"
    return (b"\x03vorbis" + struct.pack("<I", len(vendor)) + vendor + struct.pack("<I", 1) +
            struct.pack("<I", len(tag)) + tag + b"\x01")


def with_comment(p, comment):
    pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
    pk[1] = comment
    meta = p.meta.copy()
    meta[:, 1] = [len(x) for x in pk]
    meta[:, 0] = np.concatenate([[0], np.cumsum(meta[:-1, 1])])
    return decode.Packets(np.frombuffer(b"".join(pk), np.uint8).copy(), meta)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, nargs="+", default=[500, 5000])
    ap.add_argument("--setups", type=int, default=6)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--repeat", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not decode.available():
        sys.exit("oracle/_ref decode libraries not built")
    assert 4 <= a.setups <= len(SETUPS)
    import torch
    dev = torch.device("cuda", 0)
    st_cuda = torch.cuda.current_stream().cuda_stream
    ident = gpu_identity()
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i))
           for i, (ch, rate, q) in enumerate(SETUPS[:a.setups])]
    lines = []
    for nfiles in a.files:
        rng = np.random.default_rng(nfiles)
        which = rng.integers(0, a.setups, nfiles)
        files = [b"".join(ogg.file_of(with_comment(enc[s], comment_packet(b"TITLE=file %d" % f)), rng,
                                      max_segs=16, min_segs=16)) for f, s in enumerate(which)]
        off = np.zeros(nfiles + 1, np.int64)
        off[1:] = np.cumsum([len(f) for f in files])
        mp = max(len(p.audio) for p in enc)
        d_bytes = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
        d_off = torch.from_numpy(off).to(dev)
        d_info = torch.empty((nfiles, mp * abi.PACKET_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        d_npkt = torch.empty(nfiles, dtype=torch.int32, device=dev)
        d_data = torch.zeros_like(d_bytes)
        d_st = torch.empty((nfiles, abi.OGG_STREAM_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        lib.ogg_demux_dev(nfiles, d_bytes.data_ptr(), d_off.data_ptr(), mp, d_info.data_ptr(), d_npkt.data_ptr(),
                          d_data.data_ptr(), d_st.data_ptr(), st_cuda)
        torch.cuda.synchronize()
        # arm (b) buffers
        d_status, d_order, d_npkt_g = (torch.empty(nfiles, dtype=torch.int32, device=dev) for _ in range(3))
        d_info_g = torch.empty_like(d_info)
        d_groups = torch.empty(nfiles * abi.FILE_GROUP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        d_ng = torch.empty(1, dtype=torch.int32, device=dev)
        sb = lib.ogg_group_scratch_bytes(nfiles, mp)
        d_scr = torch.empty(sb, dtype=torch.uint8, device=dev)
        pinned = torch.empty(int(off[-1]), dtype=torch.uint8).pin_memory()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def arm_a():
            sts = d_st.cpu().numpy().view(abi.OGG_STREAM_DTYPE).reshape(-1)
            lo = sts["hdr_offset"][:, 0]
            hi = sts["hdr_offset"][:, 2] + sts["hdr_bytes"][:, 2]
            for f in range(nfiles):
                if sts["status"][f] == 0:
                    pinned[int(lo[f]):int(hi[f])].copy_(d_data[int(lo[f]):int(hi[f])], non_blocking=True)
            torch.cuda.synchronize()
            host = pinned.numpy()
            reps, members = {}, {}
            for f in range(nfiles):
                if sts["status"][f] != 0:
                    continue
                o, n = sts["hdr_offset"][f], sts["hdr_bytes"][f]
                key = (host[o[0]:o[0] + n[0]].tobytes(), host[o[2]:o[2] + n[2]].tobytes())
                members.setdefault(reps.setdefault(key, f), []).append(f)
            order = [f for r in sorted(members) for f in members[r]]
            groups, at = [], 0
            for r in sorted(members):
                groups.append((at, len(members[r]), r))
                at += len(members[r])
            d_ord = torch.tensor(order, dtype=torch.int64).to(dev, non_blocking=True)
            info_g = d_info.index_select(0, d_ord)
            npkt_g = d_npkt.index_select(0, d_ord)
            torch.cuda.synchronize()
            return order, groups, info_g, npkt_g

        def arm_b(events=False):
            if events:
                ev[0].record()
            lib.ogg_group_dev(nfiles, d_data.data_ptr(), d_st.data_ptr(), mp, d_npkt.data_ptr(), d_info.data_ptr(),
                              d_status.data_ptr(), d_order.data_ptr(), d_npkt_g.data_ptr(), d_info_g.data_ptr(),
                              d_groups.data_ptr(), d_ng.data_ptr(), d_scr.data_ptr(), sb, st_cuda)
            if events:
                ev[1].record()
            torch.cuda.synchronize()

        order, groups, info_g, npkt_g = arm_a()                  # warm up both and check they agree
        arm_b()
        ng = int(d_ng.item())
        got = d_groups.cpu().numpy()[:ng * abi.FILE_GROUP_DTYPE.itemsize].view(abi.FILE_GROUP_DTYPE)
        assert [tuple(int(x) for x in g) for g in got] == groups and ng == len(set(which.tolist()))
        assert d_order.cpu().numpy().tolist() == order
        assert torch.equal(d_npkt_g, npkt_g)
        ta, tb, tbe = [], [], []
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            arm_a()
            ta.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            arm_b(events=True)
            tb.append((time.perf_counter() - t0) * 1e3)
            tbe.append(ev[0].elapsed_time(ev[1]))
        hdr_bytes = int(sum(int(s["hdr_bytes"][0]) + int(s["hdr_bytes"][1]) + int(s["hdr_bytes"][2])
                            for s in d_st.cpu().numpy().view(abi.OGG_STREAM_DTYPE).reshape(-1)))
        lines.append(dict(ident, what="group demuxed Ogg files by setup: host (a) against vb200_ogg_group_dev (b)",
                          files=nfiles, setups=a.setups, groups=ng, max_packets=mp, header_bytes=hdr_bytes,
                          host_ms=ta, host_ms_median=float(np.median(ta)), host_ms_spread=float(max(ta) - min(ta)),
                          dev_wall_ms=tb, dev_wall_ms_median=float(np.median(tb)),
                          dev_event_ms=tbe, dev_event_ms_median=float(np.median(tbe)),
                          dev_event_ms_spread=float(max(tbe) - min(tbe)),
                          host_over_dev=float(np.median(ta)) / float(np.median(tb))))
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ogg_group_bench.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
