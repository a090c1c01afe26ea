"""Raw PCM to packets from host memory against device memory: vb200_encode_pcm_packets on pinned host PCM (each call
copies its rows in) against vb200_encode_pcm_packets_dev on PCM resident on the GPU (the whole clips in one tensor,
first = 0 on every call), N stereo 44.1 kHz VBR q0.5 streams fed in 1 s writes, then the end; a third arm adds
vb200_decode_streams_packets_dev on the _dev call's packets, left on the device.  The arms alternate.  Per call:
CUDA-event time on the stream, the host time spent inside the call, launches.  One JSON line per arm and repetition, with the card's name and power limit read in the same run.

    python tools/pcm_packets_dev_bench.py --streams 500 --secs 20 --reps 2"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=500)
    ap.add_argument("--secs", type=float, default=20.0)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from oracle import decode, decode_packets as dp
    from test_gpu_encode_packets import _driver
    from test_plan_vs_ref import burst_signal
    from vorbis_b200 import abi, lib
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rate, piece, ns, ch = 44100, 44100, a.streams, 2
    n = int(rate * a.secs)
    d = _driver(ch, rate, 0.5)
    ctx = d.ctx
    bs0, bs1 = ctx.bs
    sig = [burst_signal(ch, rate, a.secs, 1 + i)[:, :n] for i in range(8)]
    clip = np.stack([sig[s % 8] for s in range(ns)]).astype(np.float32)
    stage = torch.zeros((ns, ch, 4 * piece), dtype=torch.float32).pin_memory().numpy()   # the host arm's rows, pinned
    dclip = torch.from_numpy(clip).cuda()
    dec = dp.Driver(decode.Packets(*(lambda p: (p.buf, p.meta))(decode.encode(ch, rate, 0.5, sig[0][:, :rate]))))
    mb = piece // (bs0 // 2) + 4 * bs1 // (bs0 // 2) + 8
    cap = [ns * mb, ns * (piece + 4 * bs1) // (bs1 // 2) + 8 * ns]
    data_cap = ns * mb * max(ctx.packet_bound(0), ctx.packet_bound(1))
    z = lambda k, t=torch.uint8: torch.zeros(k, dtype=t, device="cuda")  # noqa: E731
    plan, nb = z(ns * mb * abi.STREAM_BLOCK_DTYPE.itemsize), z(ns, torch.int32)
    info, data, status, res = z(ns * mb * abi.PACKET_INFO_DTYPE.itemsize), z(data_cap), z(ns, torch.int32), z(24)
    first, dlen, dend = z(ns, torch.int64), z(ns, torch.int64), z(ns, torch.int32)
    pcm_cap = ns * mb * (bs1 // 2) * ch
    d_pcm, d_base = z(pcm_cap, torch.float32), z(ns + 1, torch.int64)
    d_out = z(ns * mb * abi.DECODED_PACKET_DTYPE.itemsize)
    st = torch.cuda.current_stream()

    def writes():
        w = 0
        while w < n:
            w = min(w + piece, n)
            yield w, None
        yield w, 1

    def host_arm():
        carry = ctx.encode_pcm_carry_init(ns)
        out = []
        for w, end in writes():
            raw = ctx.encode_pcm_carry_head(carry)["raw_base"]
            lens = (w - raw).astype(np.int64)
            buf = stage[:, :, :int(lens.max())]
            for s in range(ns):
                buf[s, :, :lens[s]] = clip[s, :, raw[s]:w]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0 = ctx.launch_count()
            e0.record(st)
            t0 = time.perf_counter()
            got = ctx.encode_pcm_packets(buf, lens, carry, None if end is None else np.ones(ns, np.int32),
                                         max_blocks=mb, cap=cap, data_cap=data_cap)
            host = time.perf_counter() - t0
            e1.record(st)
            e1.synchronize()
            out.append((e0.elapsed_time(e1), host * 1e3, ctx.launch_count() - l0))
            pk = got["packets"]
        return out, pk

    def dev_arm(decode_too):
        carry = torch.from_numpy(ctx.encode_pcm_carry_init(ns)).cuda()
        dcarry = dec.ctx.decode_streams_carry(ns) if decode_too else None
        out = []
        for w, end in writes():
            dlen.fill_(w)
            dend.fill_(1 if end else 0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0 = ctx.launch_count()
            e0.record(st)
            t0 = time.perf_counter()
            ctx.encode_pcm_packets_dev(ns, dclip.data_ptr(), lib.PCM_F32_PLANAR, n, dlen.data_ptr(), carry.data_ptr(),
                                       plan.data_ptr(), nb.data_ptr(), mb, cap, info.data_ptr(), data.data_ptr(),
                                       data_cap, status.data_ptr(), res.data_ptr(), d_end=dend.data_ptr(),
                                       d_first=first.data_ptr(), stream=st.cuda_stream)
            if decode_too:
                dec.ctx.decode_streams_packets_dev(ns, mb, nb.data_ptr(), info.data_ptr(), data.data_ptr(), dcarry.ptr,
                                                   0, d_pcm.data_ptr(), pcm_cap, d_base.data_ptr(), d_out.data_ptr(),
                                                   st.cuda_stream)
            host = time.perf_counter() - t0
            e1.record(st)
            e1.synchronize()
            r = res.cpu().numpy().view(abi.ENCODE_RESULT_DTYPE)[0]
            assert r["rc"] == 0, r
            out.append((e0.elapsed_time(e1), host * 1e3, ctx.launch_count() - l0))
        got_info = info.cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(ns, mb)
        got_nb, got_data = nb.cpu().numpy(), data.cpu().numpy()
        pk = [[bytes(got_data[i["offset"]:i["offset"] + i["bytes"]]) for i in got_info[s, :got_nb[s]]]
              for s in range(ns)]
        return out, pk

    arms = (("host form, pinned host PCM", lambda: host_arm()), ("_dev form, resident PCM", lambda: dev_arm(False)),
            ("_dev encode + _dev decode", lambda: dev_arm(True)))
    for _, f in arms:                                                # warm-up of every shape
        f()
    for rep in range(a.reps):
        last = {}
        for name, f in arms:
            calls, pk = f()
            last[name] = pk
            ev, host, launches = (np.array([c[i] for c in calls]) for i in range(3))
            print(json.dumps({"arm": name, "rep": rep, "streams": ns, "secs": a.secs, "calls": len(calls),
                              "event_ms_per_call": float(ev.mean()), "event_ms_total": float(ev.sum()),
                              "host_ms_in_call": float(host.mean()), "launches_per_call": float(launches.mean()),
                              "gpu": gpu}), flush=True)
        assert last["host form, pinned host PCM"] == last["_dev form, resident PCM"], "the last call's packets differ"
    dec.close()
    d.close()


if __name__ == "__main__":
    main()
