#!/usr/bin/env python
"""Ogg files written on the device: vb200_ogg_mux_dev over packet tables resident on the device.
Workload of tools/ogg_demux_bench.py: 44.1 kHz stereo at q = 0.5, 8 distinct encoded streams of 20 s repeated (500
streams in the main line), written as Ogg files with 16 lacing segments per page and demuxed on the device; the
demux's tables (data, info, npkt and the header rows of vb200_ogg_stream) are what the mux reads.  Each call starts
from fresh carries (copied in before its timed window) and writes whole files: the headers, every audio page, the EOS
page.

Reports, from CUDA events around each call after a warm-up: the mux time per call at 1, 8, 64, 500, 2000 and 4000
streams, alternated over --repeat rounds, with its median and spread; output GB/s and pages/s; and the output bytes
per second as a share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), named as such (the kernel also reads the
packets and reads each page back for its CRC, so this is not its share of the memory traffic).  Then the output of
the 500-stream call is demuxed on the device and its packets checked against the input tables.  Prints one JSON
line per measurement with the GPU's name and power limit read in the same run.

usage: python tools/ogg_mux_bench.py [--seconds 20] [--repeat 5] [--out DIR]
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
from vorbis_b200 import abi, lib  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_throughput import gpu_identity, signal  # noqa: E402

HBM_TB_S = 3.35          # H100 SXM data sheet, HBM3
COUNTS = (1, 8, 64, 500, 2000, 4000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--segs", type=int, default=16, help="lacing segments per page of the input files")
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not decode.available():
        sys.exit("oracle/_ref decode libraries not built")
    import torch
    ch, rate, q = 2, 44100, 0.5
    rng = np.random.default_rng(2026)
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i)) for i in range(a.distinct)]
    distinct = [b"".join(ogg.file_of(p, rng, min_segs=a.segs, max_segs=a.segs)) for p in enc]
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    ident = gpu_identity()
    mp = max(len(p.audio) for p in enc)
    PI, CI = abi.PACKET_INFO_DTYPE.itemsize, abi.OGG_MUX_CARRY_DTYPE.itemsize

    def resident(n):
        """the device demux of n files, and the mux's inputs and outputs on its tables"""
        files = [distinct[i % a.distinct] for i in range(n)]
        off = np.zeros(n + 1, np.int64)
        off[1:] = np.cumsum([len(f) for f in files])
        d = dict(n=n)
        d_bytes = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
        d_off = torch.from_numpy(off).to(dev)
        d["info"] = torch.empty((n, mp * PI), dtype=torch.uint8, device=dev)
        d["npkt"] = torch.empty(n, dtype=torch.int32, device=dev)
        d["data"] = torch.empty_like(d_bytes)
        d_st = torch.empty((n, abi.OGG_STREAM_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        lib.ogg_demux_dev(n, d_bytes.data_ptr(), d_off.data_ptr(), mp, d["info"].data_ptr(), d["npkt"].data_ptr(),
                          d["data"].data_ptr(), d_st.data_ptr(), st)
        torch.cuda.synchronize()
        del d_bytes
        sts = d_st.cpu().numpy().view(abi.OGG_STREAM_DTYPE).reshape(-1)
        assert (sts["status"] == 0).all()
        hdr = np.zeros((n, 3), abi.PACKET_INFO_DTYPE)
        hdr["offset"], hdr["bytes"] = sts["hdr_offset"], sts["hdr_bytes"]
        hdr["packetno"] = np.arange(3)
        d["hdr"] = torch.from_numpy(hdr.view(np.uint8).reshape(n, -1).copy()).to(dev)
        fresh = np.zeros(n, abi.OGG_MUX_CARRY_DTYPE)
        fresh["serial"] = np.arange(n) + 1
        d["fresh"] = torch.from_numpy(fresh.view(np.uint8).copy()).to(dev)
        d["carry"] = d["fresh"].clone()
        d["off"] = torch.empty(n + 1, dtype=torch.int64, device=dev)
        d["status"] = torch.empty(n, dtype=torch.int32, device=dev)
        d["out"] = None
        mux(d, 0)                                          # the sizing call
        torch.cuda.synchronize()
        d["bytes"] = int(d["off"][-1])
        d["out"] = torch.empty(d["bytes"], dtype=torch.uint8, device=dev)
        return d

    def mux(d, cap):
        d["carry"].copy_(d["fresh"])
        lib.ogg_mux_dev(d["n"], d["data"].data_ptr(), d["data"].numel(), d["hdr"].data_ptr(), mp, d["npkt"].data_ptr(),
                        d["info"].data_ptr(), d["carry"].data_ptr(), d["out"].data_ptr() if cap else None, cap,
                        d["off"].data_ptr(), d["status"].data_ptr(), st)

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(d):
        d["carry"].copy_(d["fresh"])
        ev[0].record()
        lib.ogg_mux_dev(d["n"], d["data"].data_ptr(), d["data"].numel(), d["hdr"].data_ptr(), mp, d["npkt"].data_ptr(),
                        d["info"].data_ptr(), d["carry"].data_ptr(), d["out"].data_ptr(), d["bytes"],
                        d["off"].data_ptr(), d["status"].data_ptr(), st)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1])

    res = {n: resident(n) for n in COUNTS}
    for d in res.values():                                 # warm-up, and the page count of every workload
        for _ in range(3):
            timed(d)
        out = d["out"].cpu().numpy()
        assert not d["status"].cpu().numpy().any()
        d["pages"] = 0
        at = 0
        while at < out.size:                               # every page's header gives its length
            nseg = int(out[at + 26])
            at += 27 + nseg + int(out[at + 27:at + 27 + nseg].sum())
            d["pages"] += 1
        assert at == out.size
    ms = {n: [] for n in COUNTS}
    for _ in range(a.repeat):
        for n in COUNTS:
            ms[n].append(float(np.median([timed(res[n]) for _ in range(5)])))
    lines = []
    for n in COUNTS:
        d, m = res[n], float(np.median(ms[n]))
        lines.append(dict(ident, what="vb200_ogg_mux_dev, whole files from fresh carries", streams=n,
                          seconds_per_stream=a.seconds, out_bytes=d["bytes"], pages=d["pages"], mux_ms=ms[n],
                          mux_ms_median=m, mux_ms_spread=float(max(ms[n]) - min(ms[n])),
                          out_GB_per_s=d["bytes"] / m / 1e6, pages_per_s=d["pages"] / m * 1e3,
                          out_bytes_share_of_hbm3_datasheet=d["bytes"] / m / 1e9 / HBM_TB_S))
    # the 500-stream output demuxed on the device gives back the input packets
    d = res[500]
    timed(d)
    off = d["off"].cpu().numpy()
    back = lib.ogg_demux([d["out"][int(off[i]):int(off[i + 1])].cpu().numpy() for i in range(a.distinct)],
                         max_packets=mp)
    npkt = d["npkt"].cpu().numpy()
    info = d["info"].cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(d["n"], mp)
    data = d["data"].cpu().numpy()
    for i in range(a.distinct):
        n = int(npkt[i])
        assert back["streams"][i]["status"] == 0 and back["npkt"][i] == n
        for k in range(n):
            r, s = back["info"][i, k], info[i, k]
            assert r["bytes"] == s["bytes"] and (r["e_o_s"] == s["e_o_s"])
            assert back["data"][r["offset"]:r["offset"] + r["bytes"]].tobytes() == \
                data[s["offset"]:s["offset"] + s["bytes"]].tobytes()
        assert back["info"][i, n - 1]["granulepos"] == info[i, n - 1]["granulepos"]
    lines.append(dict(ident, what="demux of the mux output", streams_checked=a.distinct, packets_equal=True))
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ogg_mux_bench.jsonl"), "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
