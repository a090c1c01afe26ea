#!/usr/bin/env python
"""Chained Ogg files resident on the device: vb200_ogg_links_dev, each timing alternated with vb200_ogg_demux_dev on
the same bytes.

1. The workload of tools/ogg_demux_bench.py (44.1 kHz stereo at q = 0.5, 8 distinct encoded streams of 20 s repeated
   over 500 files, 16 lacing segments per page): every file is one link, so this is what link-awareness costs on
   ordinary files.  Times one links call and one demux call of the whole files.
2. A capture-like workload: 64 files of 60 links of 10 s each, one setup, every link with its own comment header (8
   distinct encoded streams, each link's comment page rewritten).  Times links + demux on link_off + group, against one
   demux of the whole files, and checks that the links form one group.

The tables are checked against oracle/ogg_links.py on a few files first.  Reports, from CUDA events, the median and spread of
--repeat alternated runs of --calls calls each; prints one JSON line per measurement with the GPU's name and power
limit read in the same run.

usage: python tools/ogg_links_bench.py [--files 500] [--seconds 20] [--chains 64] [--links 60] [--link-seconds 10]
                                       [--calls 10] [--repeat 5] [--out DIR]
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
from oracle import ogg  # noqa: E402
from oracle import ogg_links  # noqa: E402
from vorbis_b200 import abi, lib  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_throughput import gpu_identity, signal  # noqa: E402


def _comment(text):
    import struct
    vendor = b"vb200 bench"
    tag = b"TITLE=" + text
    return b"\x03vorbis" + struct.pack("<I", len(vendor)) + vendor + struct.pack("<II", 1, len(tag)) + tag + b"\x01"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=500)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--chains", type=int, default=64)
    ap.add_argument("--links", type=int, default=60)
    ap.add_argument("--link-seconds", type=float, default=10.0)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--segs", type=int, default=16, help="lacing segments per page")
    ap.add_argument("--calls", type=int, default=10, help="calls per timed window")
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not decode.available():
        sys.exit("oracle/_ref decode libraries not built")
    import torch
    ch, rate, q = 2, 44100, 0.5
    rng = np.random.default_rng(2026)
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    ident = gpu_identity()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    lines = []

    def resident(files, mp):
        n = len(files)
        off = np.zeros(n + 1, np.int64)
        off[1:] = np.cumsum([len(f) for f in files])
        d = dict(n=n, bytes=int(off[-1]), mp=mp)
        d["d_bytes"] = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
        d["d_off"] = torch.from_numpy(off).to(dev)
        return d

    def demux_bufs(n, mp, nbytes):
        return dict(info=torch.empty((n, mp * abi.PACKET_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev),
                    npkt=torch.empty(n, dtype=torch.int32, device=dev),
                    data=torch.empty(nbytes, dtype=torch.uint8, device=dev),
                    st=torch.empty((n, abi.OGG_STREAM_DTYPE.itemsize), dtype=torch.uint8, device=dev))

    def demux(n, d_bytes, d_off, mp, b):
        lib.ogg_demux_dev(n, d_bytes.data_ptr(), d_off.data_ptr(), mp, b["info"].data_ptr(), b["npkt"].data_ptr(),
                          b["data"].data_ptr(), b["st"].data_ptr(), st)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(a.calls):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / a.calls

    def alternate(f1, f2):
        t1, t2 = [], []
        for _ in range(a.repeat):
            t1.append(timed(f1))
            t2.append(timed(f2))
        return t1, t2

    def stats(name, ts):
        return {name + "_ms": ts, name + "_ms_median": float(np.median(ts)), name + "_ms_spread": float(max(ts) - min(ts))}

    # ---- 1. single-link files ------------------------------------------------------------------------------------
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i)) for i in range(a.distinct)]
    distinct = [b"".join(ogg.file_of(p, rng, min_segs=a.segs, max_segs=a.segs)) for p in enc]
    files = [distinct[i % a.distinct] for i in range(a.files)]
    mp = max(len(p.audio) for p in enc)
    d = resident(files, mp)
    first = torch.empty(d["n"] + 1, dtype=torch.int64, device=dev)
    links = torch.empty(d["n"] + 1, dtype=torch.int64, device=dev)
    b = demux_bufs(d["n"], mp, d["bytes"])

    def links1():
        lib.ogg_links_dev(d["n"], d["d_bytes"].data_ptr(), d["d_off"].data_ptr(), first.data_ptr(), links.data_ptr(),
                          d["n"], st)
    links1()
    torch.cuda.synchronize()
    assert np.array_equal(links.cpu().numpy(), d["d_off"].cpu().numpy()), "one link per file"
    tl, td = alternate(links1, lambda: demux(d["n"], d["d_bytes"], d["d_off"], mp, b))
    ml = float(np.median(tl))
    lines.append(dict(ident, what="vb200_ogg_links_dev on single-link files, alternated with vb200_ogg_demux_dev",
                      files=a.files, file_bytes=d["bytes"], seconds_per_file=a.seconds, **stats("links", tl),
                      **stats("demux", td), links_GB_per_s=d["bytes"] / ml / 1e6,
                      links_over_demux=ml / float(np.median(td))))
    del d, b, first, links
    torch.cuda.empty_cache()

    # ---- 2. capture-like chains ----------------------------------------------------------------------------------
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.link_seconds, seed=100 + i)) for i in range(a.distinct)]
    base = [ogg.file_of(p, rng, serial=1000 + i, min_segs=a.segs, max_segs=a.segs) for i, p in enumerate(enc)]
    hdr = [[bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:3, :2]] for p in enc]
    chains = []
    for c in range(a.chains):
        parts = []
        for k in range(a.links):
            i = (c + k) % a.distinct
            pg = base[i]
            comment = _comment(b"chain %d track %d" % (c, k))
            assert pg[1][26] == (len(hdr[i][1]) // 255 + 1)       # the comment header alone on page 1
            com = ogg.page(0, 0, 1000 + i, 1, [255] * (len(comment) // 255) + [len(comment) % 255], comment)
            parts.append(pg[0] + com + b"".join(pg[2:]))
        chains.append(b"".join(parts))
    for c in range(2):                                    # the oracle's links on two chains
        assert len(ogg_links.links(chains[c])) == a.links + 1
    mp = max(len(p.audio) for p in enc)
    d = resident(chains, mp)
    total = a.chains * a.links
    first = torch.empty(a.chains + 1, dtype=torch.int64, device=dev)
    links = torch.empty(total + 1, dtype=torch.int64, device=dev)
    b = demux_bufs(total, mp, d["bytes"])
    bw = demux_bufs(a.chains, mp, d["bytes"])
    g = dict(status=torch.empty(total, dtype=torch.int32, device=dev), order=torch.empty(total, dtype=torch.int32,
                                                                                        device=dev),
             npkt=torch.empty(total, dtype=torch.int32, device=dev),
             info=torch.empty((total, mp * abi.PACKET_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev),
             groups=torch.empty((total, abi.FILE_GROUP_DTYPE.itemsize), dtype=torch.uint8, device=dev),
             ngroups=torch.empty(1, dtype=torch.int32, device=dev))
    sbytes = lib.ogg_group_scratch_bytes(total, mp)
    scratch = torch.empty(max(sbytes, 8), dtype=torch.uint8, device=dev)

    def chained():
        lib.ogg_links_dev(a.chains, d["d_bytes"].data_ptr(), d["d_off"].data_ptr(), first.data_ptr(), links.data_ptr(),
                          total, st)
        demux(total, d["d_bytes"], links, mp, b)
        lib.ogg_group_dev(total, b["data"].data_ptr(), b["st"].data_ptr(), mp, b["npkt"].data_ptr(),
                          b["info"].data_ptr(), g["status"].data_ptr(), g["order"].data_ptr(), g["npkt"].data_ptr(),
                          g["info"].data_ptr(), g["groups"].data_ptr(), g["ngroups"].data_ptr(), scratch.data_ptr(),
                          sbytes, st)
    chained()
    torch.cuda.synchronize()
    assert int(first[-1]) == total and int(g["ngroups"][0]) == 1, "one group"
    assert (b["st"].cpu().numpy().view(abi.OGG_STREAM_DTYPE)["status"] == 0).all()
    tc, td = alternate(chained, lambda: demux(a.chains, d["d_bytes"], d["d_off"], mp, bw))
    mc = float(np.median(tc))
    lines.append(dict(ident, what="links + demux on link_off + group on chains, alternated with one demux of the "
                                  "whole files (first link only)", files=a.chains, links_per_file=a.links,
                      seconds_per_link=a.link_seconds, file_bytes=d["bytes"], groups=1, **stats("chained", tc),
                      **stats("demux_whole", td), chained_GB_per_s=d["bytes"] / mc / 1e6))
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ogg_links_bench.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
