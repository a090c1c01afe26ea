"""Random crops straight from Ogg files: (a) vb200_ogg_demux_dev of every file, then vb200_decode_ranges_dev on its
tables, against (b) one vb200_ogg_ranges_dev call, alternating in one process on one GPU.

Workloads (44.1 kHz stereo, q = 0.5; every batch is 256 seeded crops of 5 s, a file drawn uniformly and a start
drawn uniformly below its length):
  short  INTEGRATION §2f's: 500 files of 20 s (4 distinct encodes, each file muxed by vb200_ogg_mux under its own
         serial)
  long   --long-files files of --long-minutes minutes: one 20 s encode's audio packets repeated with running
         granulepos, muxed once by vb200_ogg_mux, the file copied --long-files times on the device
Reports per arm and workload: ms per batch and crops/s from CUDA events around the batch's calls, the bytes each arm
keeps resident besides the files (a: the demux's packet copy and tables; b: the packet scratch), and, from a separate
torch.profiler pass, each kernel's share of the arm's kernel time (the plan kernels k_dr_plan and k_or_plan, and the
demux).  Both arms' got and crops are checked equal on the first batch before timing.  One JSON line per measurement
with the GPU's name and power limit read in the same run.

usage: python tools/ogg_ranges_bench.py [--files 500] [--long-files 64] [--long-minutes 60] [--batches 6]
       [--repeat 3] [--pkt-cap 262144] [--out DIR]
Needs oracle/_ref (the stock encoder, built by __graft_entry__.build() where the reference sources exist) and a GPU.
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
from oracle.decode_ranges import packet_header  # noqa: E402
from vorbis_b200 import abi, lib  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from decode_throughput import gpu_identity, signal  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=500)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--distinct", type=int, default=4)
    ap.add_argument("--long-files", type=int, default=64)
    ap.add_argument("--long-minutes", type=float, default=60.0)
    ap.add_argument("--crop", type=float, default=5.0)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--repeat", type=int, default=3, help="alternations of the two arms")
    ap.add_argument("--pkt-cap", type=int, default=1 << 18)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not (decode.available() and dp.available()):
        sys.exit("oracle/_ref decode libraries not built")
    import torch
    from torch.profiler import ProfilerActivity, profile
    ch, rate, q = 2, 44100, 0.5
    L = int(a.crop * rate)
    enc = [decode.encode(ch, rate, q, signal(ch, rate, a.seconds, seed=i)) for i in range(a.distinct)]
    pks = [[bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]] for p in enc]
    drv = dp.Driver(enc[0])
    ctx = drv.ctx
    bs = ctx.bs
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    ident = gpu_identity()
    lines = []

    def emit(d):
        d.update(ident)
        print(json.dumps(d), flush=True)
        lines.append(d)

    def short_files():
        n = a.files
        m = lib.ogg_mux([pks[f % a.distinct][3:] for f in range(n)],
                        [[int(g) for g in enc[f % a.distinct].meta[3:, 2]] for f in range(n)],
                        headers=[pks[f % a.distinct][:3] for f in range(n)], serials=list(range(1, n + 1)))
        sizes = [len(x) for x in m["pages"]]
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        return t(np.frombuffer(b"".join(m["pages"]), np.uint8)), off, max(len(p) for p in pks) - 3

    def long_files():
        audio = pks[0][3:]
        W = [packet_header(np.frombuffer(x, np.uint8), 0, len(x), 1) for x in audio]
        reps = int(round(a.long_minutes * 60 / a.seconds))
        Ws = W * reps
        g, gr = 0, []
        for k, w in enumerate(Ws):
            if k:
                g += bs[Ws[k - 1]] // 4 + bs[w] // 4
            gr.append(g)
        m = lib.ogg_mux([audio * reps], [gr], headers=[pks[0][:3]], serials=[7])
        one = t(np.frombuffer(m["pages"][0], np.uint8))
        n = a.long_files
        off = np.arange(n + 1, dtype=np.int64) * one.numel()
        return one.repeat(n), off, len(audio) * reps

    def run(name, d_bytes, off, max_audio):
        nfiles = len(off) - 1
        mp = max_audio + 1
        d_off = t(off)
        # lengths from the packet-table index of one demux
        d_info = torch.zeros(nfiles * mp * abi.PACKET_INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        d_npkt = torch.zeros(nfiles, dtype=torch.int32, device=dev)
        d_data = torch.zeros_like(d_bytes)
        d_st = torch.zeros(nfiles * abi.OGG_STREAM_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        lib.ogg_demux_dev(nfiles, d_bytes.data_ptr(), d_off.data_ptr(), mp, d_info.data_ptr(), d_npkt.data_ptr(),
                          d_data.data_ptr(), d_st.data_ptr(), st)
        d_len = torch.zeros(nfiles, dtype=torch.int64, device=dev)
        d_out = torch.zeros(nfiles * mp * abi.DECODED_PACKET_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        ctx.decode_streams_index_dev(nfiles, mp, d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(),
                                     d_len.data_ptr(), d_out.data_ptr(), st)
        length = d_len.cpu().numpy()
        status = d_st.cpu().numpy().view(abi.OGG_STREAM_DTYPE)["status"]
        assert (status == 0).all(), "demux status"
        del d_out
        rng = np.random.default_rng(2026)
        batches = []
        for _ in range(a.batches):
            f = rng.integers(0, nfiles, a.batch)
            start = (rng.random(a.batch) * (length[f] - L)).astype(np.int64)
            batches.append(t(np.array(list(zip(start, f, [L] * a.batch)), abi.PCM_RANGE_DTYPE).view(np.uint8)))
        out_a = torch.empty((a.batch, ch, L), dtype=torch.float32, device=dev)
        out_b = torch.empty((a.batch, ch, L), dtype=torch.float32, device=dev)
        got_a = torch.empty(a.batch, dtype=torch.int32, device=dev)
        got_b = torch.empty(a.batch, dtype=torch.int32, device=dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def arm_a(req):
            lib.ogg_demux_dev(nfiles, d_bytes.data_ptr(), d_off.data_ptr(), mp, d_info.data_ptr(), d_npkt.data_ptr(),
                              d_data.data_ptr(), d_st.data_ptr(), st)
            ctx.decode_ranges_dev(nfiles, mp, d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(), a.batch,
                                  req.data_ptr(), 0, out_a.data_ptr(), L, got_a.data_ptr(), st)

        def arm_b(req):
            ctx.ogg_ranges_dev(nfiles, d_bytes.data_ptr(), d_off.data_ptr(), a.batch, req.data_ptr(), 0,
                               out_b.data_ptr(), L, a.pkt_cap, got_b.data_ptr(), st)

        arms = {"a": arm_a, "b": arm_b}
        for req in batches[:2]:
            arm_a(req)
            arm_b(req)
            torch.cuda.synchronize()
            assert (got_a.cpu().numpy() == L).all() and torch.equal(got_a, got_b), "got differs"
            assert torch.equal(out_a.view(torch.int32), out_b.view(torch.int32)), "arms differ"
        resident = {"a": int(d_bytes.numel()) + nfiles * mp * abi.PACKET_INFO_DTYPE.itemsize + nfiles * 76,
                    "b": a.batch * a.pkt_cap}
        ms = {"a": [], "b": []}
        for _ in range(a.repeat):
            for arm in ("a", "b"):
                torch.cuda.synchronize()
                ev[0].record()
                for req in batches:
                    arms[arm](req)
                ev[1].record()
                torch.cuda.synchronize()
                ms[arm].append(ev[0].elapsed_time(ev[1]) / len(batches))
        for arm in ("a", "b"):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for req in batches:
                    arms[arm](req)
                torch.cuda.synchronize()
            k = {}
            for e in prof.events():
                if e.device_type.name == "CUDA" and not e.name.startswith(("Memcpy", "Memset")):
                    key = e.name.split("(")[0].split("<")[0].replace("void ", "")
                    k[key] = k.get(key, 0.0) + e.device_time_total
            tot = sum(k.values())
            best = min(ms[arm])
            emit({"workload": name, "arm": arm, "files": nfiles, "file_bytes": int(d_bytes.numel()),
                  "crops_per_batch": a.batch, "crop_s": a.crop, "ms_per_batch": round(best, 3),
                  "ms_per_batch_all": [round(x, 3) for x in ms[arm]], "crops_per_s": round(a.batch / best * 1e3, 1),
                  "resident_bytes_besides_files": resident[arm],
                  "kernel_share": {n: round(v / tot, 4) for n, v in sorted(k.items(), key=lambda x: -x[1])[:6]}})
        del d_data, d_info

    b, off, mx = short_files()
    run("short: %d files of %g s" % (a.files, a.seconds), b, off, mx)
    del b
    torch.cuda.empty_cache()
    b, off, mx = long_files()
    run("long: %d files of %g min" % (a.long_files, a.long_minutes), b, off, mx)
    drv.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ogg_ranges_bench.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
