#!/usr/bin/env python
"""Ogg files resident on the device: vb200_ogg_demux_dev against one vb200_decode_ranges_dev batch on its output.
Workload of tools/decode_ranges_bench.py: 44.1 kHz stereo at q = 0.5, 8 distinct encoded streams of 20 s repeated
(default 500 files), here written as Ogg files with 16 lacing segments per page (about 4 KB bodies, near what libogg's
ogg_stream_pageout emits for these packets).  The demux output tables go straight into decode_ranges: 256 seeded crops
of 5 s, a file drawn uniformly, a start drawn uniformly below its length - L.

Reports, from CUDA events: the demux time per call (GB/s of file bytes, pages/s) and the ranges batch time, alternated
over --repeat runs, with their median and spread; then the demux alone at smaller and larger file counts, where one
warp per file leaves the GPU underfilled.  The first demux output is checked against oracle/ogg.py on the 8 distinct
files.  Prints one JSON line per measurement with the GPU's name and power limit read in the same run.

usage: python tools/ogg_demux_bench.py [--files 500] [--seconds 20] [--calls 20] [--repeat 5] [--out DIR]
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
from oracle import ogg  # noqa: E402
from vorbis_b200 import abi, lib  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_throughput import gpu_identity, signal  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=500)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--segs", type=int, default=16, help="lacing segments per page")
    ap.add_argument("--crop", type=float, default=5.0)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--calls", type=int, default=20, help="demux calls per timed window")
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not (decode.available() and dp.available()):
        sys.exit("oracle/_ref decode libraries not built")
    import torch
    ch, rate, q = 2, 44100, 0.5
    L = int(a.crop * rate)
    rng = np.random.default_rng(2026)
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i)) for i in range(a.distinct)]
    distinct = [ogg.file_of(p, rng, min_segs=a.segs, max_segs=a.segs) for p in enc]
    pages_of = [len(pg) for pg in distinct]
    distinct = [b"".join(pg) for pg in distinct]
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    ident = gpu_identity()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    mp = max(len(p.audio) for p in enc)
    lines = []

    def resident(n):
        files = [distinct[i % a.distinct] for i in range(n)]
        off = np.zeros(n + 1, np.int64)
        off[1:] = np.cumsum([len(f) for f in files])
        d = dict(n=n, bytes=int(off[-1]), pages=sum(pages_of[i % a.distinct] for i in range(n)))
        d["d_bytes"] = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
        d["d_off"] = torch.from_numpy(off).to(dev)
        d["d_info"] = torch.empty((n, mp * abi.PACKET_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        d["d_npkt"] = torch.empty(n, dtype=torch.int32, device=dev)
        d["d_data"] = torch.empty_like(d["d_bytes"])
        d["d_st"] = torch.empty((n, abi.OGG_STREAM_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        return d

    def demux(d):
        lib.ogg_demux_dev(d["n"], d["d_bytes"].data_ptr(), d["d_off"].data_ptr(), mp, d["d_info"].data_ptr(),
                          d["d_npkt"].data_ptr(), d["d_data"].data_ptr(), d["d_st"].data_ptr(), st)

    def time_demux(d):
        demux(d)
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(a.calls):
            demux(d)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / a.calls

    res = resident(a.files)
    demux(res)
    torch.cuda.synchronize()
    sts = res["d_st"].cpu().numpy().view(abi.OGG_STREAM_DTYPE).reshape(-1)
    npkt = res["d_npkt"].cpu().numpy()
    info = res["d_info"].cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(a.files, mp)
    for i in range(a.distinct):                       # the device tables equal the oracle's on the distinct files
        r = ogg.demux(distinct[i], mp)
        assert sts[i]["status"] == 0 and sts[i]["pages"] == r["pages"] and npkt[i] == len(r["packets"])
        t = ogg.packet_table(r)
        assert (info[i, :npkt[i]]["offset"] - int(res["d_off"][i]) == t[:, 0]).all()
    hdr = np.array([[sts[0]["hdr_offset"][k], sts[0]["hdr_bytes"][k], 0, 0, k] for k in range(3)], np.int64)
    drv = dp.Driver(decode.Packets(res["d_data"].cpu().numpy(), np.concatenate([hdr, hdr[:1]])))
    ctx = drv.ctx
    length = ctx.decode_streams_index(npkt, info, res["d_data"].cpu().numpy())["length"]
    s = rng.integers(0, a.files, a.batch)
    start = (rng.random(a.batch) * (length[s] - L)).astype(np.int64)
    d_req = torch.from_numpy(np.array(list(zip(start, s, [L] * a.batch)), abi.PCM_RANGE_DTYPE).view(np.uint8)).to(dev)
    out = torch.empty((a.batch, ch, L), dtype=torch.float32, device=dev)
    got = torch.empty(a.batch, dtype=torch.int32, device=dev)

    def ranges():
        ctx.decode_ranges_dev(a.files, mp, res["d_npkt"].data_ptr(), res["d_info"].data_ptr(),
                              res["d_data"].data_ptr(), a.batch, d_req.data_ptr(), 0, out.data_ptr(), L,
                              got.data_ptr(), st)

    ranges()
    torch.cuda.synchronize()
    assert (got.cpu().numpy() == L).all()
    dm, rg = [], []
    for _ in range(a.repeat):
        dm.append(time_demux(res))
        torch.cuda.synchronize()
        ev[0].record()
        ranges()
        ev[1].record()
        torch.cuda.synchronize()
        rg.append(ev[0].elapsed_time(ev[1]))
    med = float(np.median(dm))
    lines.append(dict(ident, what="vb200_ogg_demux_dev, alternated with one ranges batch", files=a.files,
                      file_bytes=res["bytes"], pages=res["pages"], seconds_per_file=a.seconds,
                      demux_ms=dm, demux_ms_median=med, demux_ms_spread=float(max(dm) - min(dm)),
                      demux_GB_per_s=res["bytes"] / med / 1e6, demux_pages_per_s=res["pages"] / med * 1e3,
                      ranges_ms=rg, ranges_ms_median=float(np.median(rg)), ranges_crops=a.batch, crop_samples=L,
                      demux_over_ranges=med / float(np.median(rg))))
    del res
    for n in (1, 8, 64, 132 * 4, 2000, 4000):
        d = resident(n)
        ms = [time_demux(d) for _ in range(3)]
        m = float(np.median(ms))
        lines.append(dict(ident, what="vb200_ogg_demux_dev by file count", files=n, file_bytes=d["bytes"],
                          pages=d["pages"], demux_ms=ms, demux_ms_median=m, demux_GB_per_s=d["bytes"] / m / 1e6,
                          demux_pages_per_s=d["pages"] / m * 1e3))
        del d
    drv.close()
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ogg_demux_bench.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
