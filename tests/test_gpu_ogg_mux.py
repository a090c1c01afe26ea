"""Ogg Vorbis files out on the device (vb200_ogg_mux[_dev]) against oracle/ogg_mux.py, the demux and the stock decoder:
- the seven hand-worked cases of tests/test_ogg_mux_oracle.py give their literal pages, and case D cut after packet 4
  keeps one packet with 18 of its values on pages;
- stock-encoder streams of the four setups of test_gpu_ogg.py equal oracle.ogg_mux.mux byte for byte; the device
  demux of the files gives the oracle demux's tables and the packets back, and demux -> group -> header parse ->
  vb200_decode_streams_packets gives the stock decoder's PCM bit for bit;
- raw PCM fed to vb200_encode_pcm_packets in seeded writes, each call's packets (with the carry's kept tail) muxed
  call by call, gives the file encoder_example.c writes for the same writes;
- 1000 seeded packet streams in one call (0-byte packets, multiples of 255 and their neighbours, sizes around 4096,
  65025 and beyond, streams without e_o_s) equal the oracle, and seeded cuts equal one call in bytes and carries;
- shared identification and setup rows with per-stream comment headers (one of 100 000 bytes) over a mix of setups
  group by setup after the demux;
- every per-stream refusal leaves the other streams' bytes as they were; a short out_cap writes nothing and leaves the
  carries; out_cap = 0 sizes the call;
- the _dev form equals the host form, and one call is three kernel launches at 1 and at 1000 streams (counted with
  torch.profiler in a process of its own)."""
import numpy as np
import pytest

from oracle import decode
from oracle import decode_packets as dp
from oracle import decode_streams as ds
from oracle import ogg
from oracle import ogg_mux
from test_gpu_ogg import launched_kernels
from test_ogg_mux_oracle import CASES as HAND, SERIAL, hand_case, seeded_cuts, seeded_stream
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
EINVAL = -131
STOCK = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2), (2, 44100, -0.1)]   # the CASES of test_gpu_ogg.py


def _need():
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def _oracle_call(carries, headers, packets, granules, eos):
    """oracle.ogg_mux.mux_call per stream: (status, pages bytes, carries)"""
    st, pages, out = [], [], []
    for s in range(len(packets)):
        c = {k: int(carries[s][k]) for k in ("serial", "pageno", "state", "kept", "kept_segs")}
        r, pg, nc = ogg_mux.mux_call(c, headers[s] if headers is not None else None, packets[s], granules[s], eos[s])
        st.append(r)
        pages.append(b"".join(pg))
        out.append(nc)
    return st, pages, out


def _carry_rows(carries):
    return [{k: int(c[k]) for k in ("serial", "pageno", "state", "kept", "kept_segs")} for c in carries]


def test_literal_cases(cuda_ok):
    cs = [hand_case(n) for n in HAND]
    r = lib.ogg_mux([c[1] for c in cs], [c[2] for c in cs], [c[3] for c in cs], headers=[c[0] for c in cs],
                    serials=[SERIAL] * len(cs))
    for name, c, got in zip(HAND, cs, r["pages"]):
        assert got == b"".join(c[4]), "case %s" % name
    assert (r["carry"]["state"] == 2).all() and list(r["carry"]["pageno"]) == [len(c[4]) for c in cs]
    hdr, pk, gr, eos, want = hand_case("D")
    a = lib.ogg_mux([pk[:4]], [gr[:4]], [eos[:4]], headers=[hdr], serials=[SERIAL])
    assert a["pages"][0] == b"".join(want[:3])
    assert _carry_rows(a["carry"]) == [dict(serial=SERIAL, pageno=3, state=1, kept=1, kept_segs=18)]
    b = lib.ogg_mux([pk[3:]], [gr[3:]], [eos[3:]], carries=a["carry"])
    assert b["pages"][0] == want[3] and b["pages"][0][5] == 5


_enc = {}


def _stock(ch, rate, q):
    if (ch, rate, q) not in _enc:
        from conftest import probe_signal
        p = decode.encode(ch, rate, q, probe_signal(ch, rate, 0.7, seed=31))
        pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
        _enc[(ch, rate, q)] = (pk[:3], pk[3:], [int(g) for g in p.meta[3:, 2]], [bool(e) for e in p.meta[3:, 3]])
    return _enc[(ch, rate, q)]


def _hdr_rows(st):
    return np.array([[st["hdr_offset"][k], st["hdr_bytes"][k], 0, 0, k] for k in range(3)], np.int64)


def _audio_rows(info):
    return np.stack([info["offset"], info["bytes"], info["granulepos"], info["e_o_s"], info["packetno"]], 1)


def test_stock_streams(cuda_ok):
    _need()
    src = [_stock(*c) for c in STOCK]
    r = lib.ogg_mux([s[1] for s in src], [s[2] for s in src], [s[3] for s in src], headers=[s[0] for s in src],
                    serials=[11 * (i + 1) for i in range(len(src))])
    files = r["pages"]
    for i, s in enumerate(src):
        assert files[i] == b"".join(ogg_mux.mux(s[0], s[1], s[2], s[3], 11 * (i + 1))), "stock %s" % (STOCK[i],)
    res = lib.ogg_demux(files)
    for f, s in enumerate(src):
        o = ogg.demux(files[f], res["info"].shape[1])
        assert o["status"] == 0 and o["hdr_data"] == s[0] and o["pkt_data"] == s[1]
        n, base = int(res["npkt"][f]), int(res["file_off"][f])
        assert n == len(s[1]) and res["streams"][f]["status"] == 0
        t = ogg.packet_table(o)
        info = res["info"][f, :n]
        assert np.array_equal(_audio_rows(info) - [base, 0, 0, 0, 0], t), "demux %s" % (STOCK[f],)
        gp = info["granulepos"]
        assert ((gp == -1) | (gp == s[2])).all() and gp[-1] == s[2][-1] and info["e_o_s"][-1] == 1
    g = lib.ogg_group(res)
    assert len(g["groups"]) == len(src)
    for first, nf, rep in g["groups"].tolist():
        st = res["streams"][rep]
        hb = [bytes(res["data"][int(st["hdr_offset"][k]):int(st["hdr_offset"][k] + st["hdr_bytes"][k])])
              for k in range(3)]
        h = lib.vorbis_headers(*hb)
        ctx = h.context()
        try:
            npkt, info = g["npkt"][first:first + nf], g["info"][first:first + nf]
            want = [ds.ref_decode(res["data"], _hdr_rows(st), _audio_rows(info[k, :npkt[k]]), h.channels)
                    for k in range(nf)]
            got = ctx.decode_streams_packets(npkt, info, res["data"], ctx.decode_streams_carry(nf))
            from test_gpu_decode_streams import _check
            _check(got, want, h.channels, False, "file %d" % rep)
        finally:
            ctx.close()


def test_raw_pcm_to_file(cuda_ok):
    """vb200_encode_pcm_packets call by call into vb200_ogg_mux with the mux carries: the file encoder_example.c
    writes for the same writes (oracle.ogg_mux.mux of the stock encoder's packets)"""
    from oracle import bitrate as B
    from test_gpu_encode_packets import _driver
    from test_gpu_pcm_packets import Feed, _sched
    from test_gpu_stream_packets import _need_ref, _streams
    _need_ref()
    ch, rate, q = 2, 44100, 0.5
    hdr = _stock(ch, rate, q)[0]
    d = _driver(ch, rate, q)
    try:
        sig = _streams(ch, rate, 0.6)
        rng = np.random.default_rng(17)
        ws = [int(w) for w in rng.integers(64, 9000, len(sig))]
        f = Feed(d.ctx, sig, [_sched(p.shape[1], w) for p, w in zip(sig, ws)])
        ns = len(sig)
        carry = np.zeros(ns, abi.OGG_MUX_CARRY_DTYPE)
        carry["serial"] = np.arange(ns) + 500
        files = [b""] * ns
        seen = [0] * ns                                  # packets of each stream muxed or kept so far
        for _ in range(100000):
            head = d.ctx.encode_pcm_carry_head(f.carry)
            if head["enc"]["done"].all():
                break
            f.step()
            pk, gr, eo = [], [], []
            for s in range(ns):
                lo = seen[s] - int(carry[s]["kept"])
                pk.append(f.pk[s][lo:])
                gr.append([int(r["granulepos"]) for r in f.inf[s][lo:]])
                eo.append([bool(r["e_o_s"]) for r in f.inf[s][lo:]])
                seen[s] = len(f.pk[s])
            r = lib.ogg_mux(pk, gr, eo, headers=[hdr] * ns, carries=carry)
            carry = r["carry"]
            files = [a + b for a, b in zip(files, r["pages"])]
        assert (carry["state"] == 2).all()
        for s, p in enumerate(sig):
            cap = B.ref_stream_capture(B.vbr(ch, rate, q), p, chunk=ws[s])
            want = ogg_mux.mux(hdr, cap["packets"], [int(g) for g in cap["granulepos"]],
                               [bool(e) for e in cap["e_o_s"]], 500 + s)
            assert files[s] == b"".join(want), "stream %d (writes of %d)" % (s, ws[s])
    finally:
        d.close()


def _seeded(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n):
        m = int(rng.integers(0, 40)) if s % 10 else int(rng.integers(0, 400))
        out.append(seeded_stream(rng, m, eos=s % 7 != 3, big=s % 25 == 0))
    return out


def test_seeded_streams_and_cuts(cuda_ok):
    S = _seeded(1000, 2026)
    ns = len(S)
    r = lib.ogg_mux([s[1] for s in S], [s[2] for s in S], [s[3] for s in S], headers=[s[0] for s in S],
                    serials=list(range(ns)))
    fresh = np.zeros(ns, abi.OGG_MUX_CARRY_DTYPE)
    fresh["serial"] = np.arange(ns)
    st, pages, carries = _oracle_call(fresh, [s[0] for s in S], [s[1] for s in S], [s[2] for s in S],
                                      [s[3] for s in S])
    assert not any(st) and (r["status"] == 0).all()
    for s in range(ns):
        assert r["pages"][s] == pages[s], "stream %d" % s
    assert _carry_rows(r["carry"]) == carries
    # every stream cut by its own seeded cuts; each round is one call over all streams
    rng = np.random.default_rng(7)
    cuts = [seeded_cuts(rng, len(s[1]), int(rng.integers(1, 6))) + [len(s[1])] for s in S]
    rounds = max(len(c) for c in cuts)
    carry, at, got = fresh.copy(), [0] * ns, [b""] * ns
    for i in range(rounds):
        pk, gr, eo = [], [], []
        for s in range(ns):
            end = cuts[s][min(i, len(cuts[s]) - 1)]
            lo = at[s] - int(carry[s]["kept"])
            pk.append(S[s][1][lo:end])
            gr.append(S[s][2][lo:end])
            eo.append(S[s][3][lo:end])
            at[s] = end
        q = lib.ogg_mux(pk, gr, eo, headers=[s[0] for s in S], carries=carry)
        carry = q["carry"]
        got = [a + b for a, b in zip(got, q["pages"])]
    assert got == r["pages"]
    assert carry.tobytes() == r["carry"].tobytes()


def test_shared_and_per_stream_headers(cuda_ok):
    _need()
    from test_gpu_ogg_headers import comment_packet
    src = [_stock(*c) for c in STOCK]
    rng = np.random.default_rng(5)
    blobs, at = [], 0
    shared = []                                           # per setup: (id row, setup row) offsets
    for s in src:
        shared.append((at, at + len(s[0][0])))
        blobs += [s[0][0], s[0][2]]
        at += len(s[0][0]) + len(s[0][2])
    ns = 12
    setup_of = [int(x) for x in rng.integers(0, len(src), ns)]
    npk = [len(src[k][1]) for k in setup_of]
    mp = max(npk)
    hdr = np.zeros((ns, 3), abi.PACKET_INFO_DTYPE)
    info = np.zeros((ns, mp), abi.PACKET_INFO_DTYPE)
    comments = []
    for i, k in enumerate(setup_of):
        c = comment_packet([b"TITLE=" + (b"x" * 100_000 if i == 3 else b"stream %d" % i)])
        comments.append(c)
        hdr[i] = [(shared[k][0], 0, len(src[k][0][0]), 0, 0, 0), (at, 0, len(c), 0, 1, 0),
                  (shared[k][1], 0, len(src[k][0][2]), 0, 2, 0)]
        blobs.append(c)
        at += len(c)
        for j, p in enumerate(src[k][1]):
            info[i, j] = (at, src[k][2][j], len(p), int(src[k][3][j]), 0, 0)
            blobs.append(p)
            at += len(p)
    data = np.frombuffer(b"".join(blobs), np.uint8)
    carry = np.zeros(ns, abi.OGG_MUX_CARRY_DTYPE)
    carry["serial"] = np.arange(ns) * 3 + 1
    out_off = np.zeros(ns + 1, np.int64)
    status = np.zeros(ns, np.int32)
    npkt = np.array(npk, np.int32)
    L = lib.load()
    args = [ns, data.ctypes.data, data.size, hdr.ctypes.data, mp, npkt.ctypes.data, info.ctypes.data]
    assert L.vb200_ogg_mux(*args, carry.copy().ctypes.data, None, 0, out_off.ctypes.data, status.ctypes.data) == EINVAL
    out = np.zeros(int(out_off[-1]), np.uint8)
    assert L.vb200_ogg_mux(*args, carry.ctypes.data, out.ctypes.data, out.size, out_off.ctypes.data,
                           status.ctypes.data) == 0
    files = [out[out_off[i]:out_off[i + 1]].tobytes() for i in range(ns)]
    for i, k in enumerate(setup_of):
        s = src[k]
        assert files[i] == b"".join(ogg_mux.mux([s[0][0], comments[i], s[0][2]], s[1], s[2], s[3], 3 * i + 1))
    res = lib.ogg_demux(files)
    assert (res["streams"]["status"] == 0).all()
    g = lib.ogg_group(res)
    assert len(g["groups"]) == len(set(setup_of))
    for first, nf, rep in g["groups"].tolist():
        members = [int(f) for f in g["order"][first:first + nf]]
        assert members == [i for i in range(ns) if setup_of[i] == setup_of[rep]], "groups follow the setups"


def test_refusals(cuda_ok):
    S = _seeded(8, 99)
    S = [s for s in S if s[1] and s[3][-1]][:5]
    assert len(S) == 5
    hs, pks, grs, eos = [s[0] for s in S], [list(s[1]) for s in S], [list(s[2]) for s in S], [list(s[3]) for s in S]
    good = lib.ogg_mux(pks, grs, eos, headers=hs, serials=[1, 2, 3, 4, 5])
    assert good["rc"] == 0

    def refused(bad, **kw):
        """stream `bad` refused, the others' bytes as in the good call"""
        r = lib.ogg_mux(pks, grs, kw.get("eo", eos), headers=hs,
                        carries=kw.get("carry"), serials=None if "carry" in kw else [1, 2, 3, 4, 5], check=False,
                        out_cap=kw.get("out_cap"))
        assert r["rc"] == EINVAL
        assert list(np.nonzero(r["status"])[0]) == [bad] and r["status"][bad] == EINVAL
        assert r["out_off"][bad + 1] == r["out_off"][bad]
        for s in range(len(S)):
            if s != bad:
                assert r["pages"][s] == good["pages"][s]
        return r
    eo = [list(e) for e in eos]
    eo[1][0] = True                                       # e_o_s before the last row
    if len(eo[1]) > 1:
        refused(1, eo=eo)
    fresh = np.zeros(5, abi.OGG_MUX_CARRY_DTYPE)
    fresh["serial"] = [1, 2, 3, 4, 5]
    done = fresh.copy()
    done[2]["state"] = 2
    refused(2, carry=done)                                # packets on a done carry
    kept = fresh.copy()
    kept[3]["state"], kept[3]["kept"] = 1, len(pks[3]) + 1
    refused(3, carry=kept)                                # npkt below kept
    # rows: a negative size and a row past the end of data, through the raw call
    L = lib.load()
    n, mp = len(S), max(len(p) for p in pks)
    info = np.zeros((n, mp), abi.PACKET_INFO_DTYPE)
    hdr = np.zeros((n, 3), abi.PACKET_INFO_DTYPE)
    blobs, at = [], 0
    for s in range(n):
        for k, h in enumerate(hs[s]):
            hdr[s, k] = (at, 0, len(h), 0, k, 0)
            blobs.append(h)
            at += len(h)
        for k, p in enumerate(pks[s]):
            info[s, k] = (at, grs[s][k], len(p), int(eos[s][k]), 0, 0)
            blobs.append(p)
            at += len(p)
    data = np.frombuffer(b"".join(blobs), np.uint8)
    npkt = np.array([len(p) for p in pks], np.int32)
    total = int(good["out_off"][-1])

    def raw(info, hdr_ptr, carry, cap):
        out = np.zeros(max(cap, 1), np.uint8)
        off, st = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
        rc = L.vb200_ogg_mux(n, data.ctypes.data, data.size, hdr_ptr, mp, npkt.ctypes.data, info.ctypes.data,
                             carry.ctypes.data, out.ctypes.data if cap else None, cap, off.ctypes.data, st.ctypes.data)
        return rc, out, off, st
    for s, field, value in ((0, "bytes", -1), (4, "offset", data.size - int(info[4, 0]["bytes"]) + 1)):
        bad = info.copy()
        bad[s, 0][field] = value
        c = fresh.copy()
        rc, out, off, st = raw(bad, hdr.ctypes.data, c, total)
        assert rc == EINVAL and list(np.nonzero(st)[0]) == [s] and off[s + 1] == off[s]
        assert c.tobytes() == fresh.tobytes()
    rc, out, off, st = raw(info, None, fresh.copy(), total)         # fresh carries without header rows
    assert rc == EINVAL and (st == EINVAL).all() and off[-1] == 0
    # out_cap one byte short: nothing written, carries as they were, out_off filled; out_cap = 0 sizes the call
    for cap in (total - 1, 0):
        c = fresh.copy()
        rc, out, off, st = raw(info, hdr.ctypes.data, c, cap)
        assert rc == EINVAL and (st == 0).all() and np.array_equal(off, good["out_off"])
        assert not out.any() and c.tobytes() == fresh.tobytes()
    c = fresh.copy()
    rc, out, off, st = raw(info, hdr.ctypes.data, c, total)
    assert rc == 0 and out.tobytes() == b"".join(good["pages"]) and c.tobytes() == good["carry"].tobytes()
    assert L.vb200_ogg_mux_dev(1, None, 0, None, 1, None, None, None, None, 0, None, None, None) == EINVAL
    off0 = np.ones(1, np.int64)
    assert L.vb200_ogg_mux(0, None, 0, None, 1, None, None, None, None, 0, off0.ctypes.data, None) == 0 and off0[0] == 0


def _dev_call(ns, profiled=False):
    """vb200_ogg_mux_dev on ns seeded streams with fresh carries: (host form's result, device outputs, kernel names or
    None)"""
    import torch
    dev = torch.device("cuda", 0)
    base = _seeded(60, 4)
    S = [base[i % len(base)] for i in range(ns)]
    host = lib.ogg_mux([s[1] for s in S], [s[2] for s in S], [s[3] for s in S], headers=[s[0] for s in S],
                       serials=list(range(ns)))
    mp = max(1, max(len(s[1]) for s in S))
    info = np.zeros((ns, mp), abi.PACKET_INFO_DTYPE)
    hdr = np.zeros((ns, 3), abi.PACKET_INFO_DTYPE)
    blobs, at = [], 0
    for i, s in enumerate(S):
        for k, h in enumerate(s[0]):
            hdr[i, k] = (at, 0, len(h), 0, k, 0)
            blobs.append(h)
            at += len(h)
        for k, p in enumerate(s[1]):
            info[i, k] = (at, s[2][k], len(p), int(s[3][k]), 0, 0)
            blobs.append(p)
            at += len(p)
    total = int(host["out_off"][-1])
    t = {k: torch.from_numpy(v.reshape(-1).view(np.uint8).copy()).to(dev) for k, v in
         dict(data=np.frombuffer(b"".join(blobs), np.uint8), hdr=hdr, info=info,
              npkt=np.array([len(s[1]) for s in S], np.int32)).items()}
    carry = np.zeros(ns, abi.OGG_MUX_CARRY_DTYPE)
    carry["serial"] = np.arange(ns)
    d_carry = torch.from_numpy(carry.view(np.uint8).copy()).to(dev)
    d_out = torch.zeros(total, dtype=torch.uint8, device=dev)
    d_off = torch.zeros(ns + 1, dtype=torch.int64, device=dev)
    d_st = torch.zeros(ns, dtype=torch.int32, device=dev)

    def call():
        lib.ogg_mux_dev(ns, t["data"].data_ptr(), at, t["hdr"].data_ptr(), mp, t["npkt"].data_ptr(),
                        t["info"].data_ptr(), d_carry.data_ptr(), d_out.data_ptr(), total, d_off.data_ptr(),
                        d_st.data_ptr())
        torch.cuda.synchronize()
    torch.cuda.synchronize()
    kernels = None
    if profiled:
        kernels = launched_kernels(call)
    else:
        call()
    out = {"out_off": d_off.cpu().numpy(), "status": d_st.cpu().numpy(), "out": d_out.cpu().numpy(),
           "carry": d_carry.cpu().numpy().view(abi.OGG_MUX_CARRY_DTYPE)}
    return host, out, kernels


def test_dev_form(cuda_ok):
    for ns in (1, 1000):
        host, dev, _ = _dev_call(ns)
        assert np.array_equal(dev["out_off"], host["out_off"]) and not dev["status"].any(), "%d streams" % ns
        assert dev["out"].tobytes() == b"".join(host["pages"]), "%d streams: pages" % ns
        assert dev["carry"].tobytes() == host["carry"].tobytes(), "%d streams: carries" % ns


def test_launches(cuda_ok):
    """three kernels (count, offsets, write) at 1 and at 1000 streams, counted with torch.profiler in a process of its
    own (a profiler session of another test in the same process can lose the kernel records of a later one)"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_ogg_mux as T; "
            "print(json.dumps([T._dev_call(n, profiled=True)[2] for n in (1, 1000)]))" % (here, os.path.dirname(here)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=here)
    assert r.returncode == 0, r.stderr[-3000:]
    for kernels in json.loads(r.stdout.strip().splitlines()[-1]):
        assert len(kernels) == 3 and "k_ogg_mux_count" in kernels[0] and "k_ds_scan" in kernels[1] and \
            "k_ogg_mux_write" in kernels[2], kernels
