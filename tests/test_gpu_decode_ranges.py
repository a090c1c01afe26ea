"""Sample ranges of many streams on the device (vb200_decode_streams_index[_dev], vb200_decode_ranges[_dev]) against
the stock decoder, bit for bit, on the streams of tests/test_decode_streams_oracle.py make_streams (four setups, the
last one 512/4096; seven kinds of stream; granulepos on every packet and on page-final packets only):
- the index equals a fresh-carry vb200_decode_streams_packets call: out byte for byte, length = the pcm_base
  differences, at full and half rate;
- the ranges equal slices of the stock decoder's PCM, float and int16: start 0, inside the first returned block,
  across each kind's special packet and the trims, ending at and past the end, starting at and past it, length 0 and
  length = out_stride, several overlapping requests per stream in reverse stream order, and one request per stream
  for its whole length, which equals the whole vb200_decode_streams_packets output;
- half rate against the stock half-rate decoder; vb200_encode_streams_packets' info and data straight in;
- the capacity guard: interior blocks that return nothing give got = VB200_EINVAL and a zero row, the other requests
  of the call are unaffected, and a larger out_stride serves the request;
- the _dev forms on device-resident packets equal the host forms; three launches per ranges call and two per index
  call whatever nreq and nstreams are; every error code; the vb200_pcm_range layout."""
import ctypes as C

import numpy as np
import pytest

from oracle import decode
from oracle import decode_ranges as dr
from oracle import decode_streams as ds
from oracle import halfrate
from test_decode_streams_oracle import CASES, make_streams
from test_gpu_decode_streams import _ctx, _need, _table, drivers  # noqa: F401  (drivers: a fixture)
from vorbis_b200 import abi

pytestmark = pytest.mark.gpu
EINVAL = -131


def _requests(audios, whole, index, out_stride, rng):
    """the seeded requests of the module docstring, in reverse stream order"""
    req = []
    for s in reversed(range(len(audios))):
        n = whole[s].shape[1]
        o = index["out"][s, :len(audios[s])]
        first = next((int(x["pcm_offset"]) for x in o if x["samples"] > 0), 0)
        mid = int(o[len(audios[s]) // 2]["pcm_offset"])
        trim = int(o[min(3, len(o) - 1)]["pcm_offset"])
        for start, length in [(0, 1500), (first + 5, 700), (max(mid - 900, 0), 2000), (max(mid - 200, 0), 3000),
                              (max(trim - 500, 0), 1200), (max(n - 1500, 0), 1500), (max(n - 300, 0), 1000),
                              (n, 100), (n + 77, 5), (10, 0), (3, out_stride), (0, min(n, out_stride))]:
            req.append((start, s, length))
        for _ in range(3):
            req.append((int(rng.integers(0, max(n, 1))), s, int(rng.integers(1, out_stride + 1))))
    return np.array(req, abi.PCM_RANGE_DTYPE)


def _check_ranges(r, req, whole, s16, what):
    for i, (start, s, length) in enumerate(req.tolist()):
        n = whole[s].shape[1]
        got = min(length, max(0, n - start))
        assert r["got"][i] == got, "%s request %d %s: got %d, want %d" % (what, i, (start, s, length), r["got"][i], got)
        want = whole[s][:, start:start + got]
        if s16:
            g = r["pcm"][i]
            assert np.array_equal(g[:got], ds.s16_of(want)), "%s request %d: int16" % (what, i)
            assert not g[got:].any(), "%s request %d: tail not zero" % (what, i)
        else:
            g = r["pcm"][i]
            assert np.array_equal(g[:, :got].view(np.uint32), want.view(np.uint32)), "%s request %d" % (what, i)
            assert not g[:, got:].view(np.uint32).any(), "%s request %d: tail not zero" % (what, i)


def _stock(buf, hdr, audios, ch, half=False):
    return [ds.ref_decode(buf, hdr, a, ch, halfrate=half)[0] for a in audios]


def _index_equals_streams(ctx, buf, audios, what):
    npkt, info = _table(audios)
    idx = ctx.decode_streams_index(npkt, info, buf)
    full = ctx.decode_streams_packets(npkt, info, buf, ctx.decode_streams_carry(len(audios)))
    assert (idx["length"] == np.diff(full["pcm_base"])).all(), what
    for s in range(len(audios)):
        assert idx["out"][s, :npkt[s]].tobytes() == full["out"][s, :npkt[s]].tobytes(), "%s stream %d" % (what, s)
    return idx, full


@pytest.mark.parametrize("ch,rate,q", CASES)
@pytest.mark.parametrize("page_final", [False, True])
def test_index_and_ranges_equal_stock_decoder(cuda_ok, drivers, ch, rate, q, page_final):  # noqa: F811
    _need()
    buf, hdr, audios = make_streams(ch, rate, q, page_final)
    ctx = _ctx(drivers, buf, hdr)
    whole = _stock(buf, hdr, audios, ch)
    idx, full = _index_equals_streams(ctx, buf, audios, "index")
    assert (idx["length"] == [w.shape[1] for w in whole]).all()
    out_stride = int(idx["length"].max()) + 64
    req = _requests(audios, whole, idx, out_stride, np.random.default_rng(rate + ch + page_final))
    npkt, info = _table(audios)
    for s16 in (False, True):
        r = ctx.decode_ranges(npkt, info, buf, req, out_stride, s16=s16)
        _check_ranges(r, req, whole, s16, "s16=%s" % s16)
    # one request per stream for its whole length is the whole decode_streams_packets output
    one = np.array([(0, s, out_stride) for s in range(len(audios))], abi.PCM_RANGE_DTYPE)
    r = ctx.decode_ranges(npkt, info, buf, one, out_stride)
    for s in range(len(audios)):
        n = full["pcm"][s].shape[1]
        assert r["got"][s] == n
        assert np.array_equal(r["pcm"][s][:, :n].view(np.uint32), full["pcm"][s].view(np.uint32)), "whole %d" % s


@pytest.mark.parametrize("ch,rate,q", [CASES[0], CASES[3]])
def test_halfrate_equals_stock_halfrate_decoder(cuda_ok, drivers, ch, rate, q):  # noqa: F811
    _need()
    buf, hdr, audios = make_streams(ch, rate, q, page_final=True)
    ctx = _ctx(drivers, buf, hdr)
    enc = decode.encode(ch, rate, q, np.zeros((ch, 4096), np.float32))
    win = halfrate.ref_decode((enc.buf, enc.meta[:, 1].copy()), ctx.bs, ch, 8192, halfrate=True)
    ctx.synthesis_halfrate(True, [win["window0"], win["window1"]])
    try:
        whole = _stock(buf, hdr, audios, ch, half=True)
        idx, _ = _index_equals_streams(ctx, buf, audios, "half-rate index")
        assert (idx["length"] == [w.shape[1] for w in whole]).all()
        out_stride = int(idx["length"].max()) + 32
        req = _requests(audios, whole, idx, out_stride, np.random.default_rng(11))
        npkt, info = _table(audios)
        for s16 in (False, True):
            _check_ranges(ctx.decode_ranges(npkt, info, buf, req, out_stride, s16=s16), req, whole, s16, "half rate")
    finally:
        ctx.synthesis_halfrate(False)


def test_encoder_packets_straight_in(cuda_ok, drivers):  # noqa: F811
    """vb200_encode_streams_packets' info and data, unchanged: ranges equal slices of the stock decoder's PCM"""
    _need()
    from oracle import bitrate as B
    from test_gpu_encode_packets import _driver
    from test_gpu_stream_packets import _streams, _timelines
    if not B.ref_available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ch, rate, q = 2, 44100, 0.5
    enc = _driver(ch, rate, q)
    try:
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p) for p in _streams(ch, rate, 0.6)]
        tl, pcm_len, eof = _timelines(caps, ch)
        e = enc.ctx.encode_streams_packets(tl, pcm_len, eof)
    finally:
        enc.close()
    stock = decode.encode(ch, rate, q, np.zeros((ch, 4096), np.float32))
    ctx = _ctx(drivers, stock.buf, stock.hdr)
    info, data = e["info"], e["data"]
    buf = np.concatenate([stock.buf, data])
    whole = []
    for s in range(len(caps)):
        r = info[s, :e["nblocks"][s]]
        rows = np.stack([r["offset"] + len(stock.buf), r["bytes"], r["granulepos"], r["e_o_s"], r["packetno"]], 1)
        whole.append(ds.ref_decode(buf, stock.hdr, rows.astype(np.int64), ch)[0])
    idx = ctx.decode_streams_index(e["nblocks"], info, data)
    assert (idx["length"] == [w.shape[1] for w in whole]).all()
    rng = np.random.default_rng(3)
    req = np.array([(int(rng.integers(0, max(w.shape[1], 1))), s, 4410) for s, w in enumerate(whole) for _ in range(4)],
                   abi.PCM_RANGE_DTYPE)
    _check_ranges(ctx.decode_ranges(e["nblocks"], info, data, req, 4410), req, whole, False, "encoder output")
    assert sum(w.shape[1] for w in whole) > 0


@pytest.mark.parametrize("out_stride", [11025, 4097])
def test_odd_channels_and_odd_out_stride(cuda_ok, drivers, out_stride):  # noqa: F811
    """mono with an odd out_stride: every request's residue region (and so every block in it) stays 16-byte aligned
    for the synthesis' vector loads; many requests, so that odd-numbered ones are covered"""
    _need()
    ch, rate, q = CASES[1]
    assert ch == 1
    buf, hdr, audios = make_streams(ch, rate, q)
    ctx = _ctx(drivers, buf, hdr)
    whole = _stock(buf, hdr, audios, ch)
    idx = ctx.decode_streams_index(*_table(audios), buf)
    req = _requests(audios, whole, idx, out_stride, np.random.default_rng(out_stride))
    assert len(req) > 20
    npkt, info = _table(audios)
    for s16 in (False, True):
        _check_ranges(ctx.decode_ranges(npkt, info, buf, req, out_stride, s16=s16), req, whole, s16,
                      "mono out_stride %d s16=%s" % (out_stride, s16))


@pytest.mark.parametrize("seed", range(4))
def test_fuzzed_bookkeeping_equals_streams(cuda_ok, drivers, seed):  # noqa: F811
    """k_dr_plan runs blockin's bookkeeping as its own copy of k_ds_plan's step: on seeded packet metadata (granulepos
    on random packets, some behind the count, packetno gaps, e_o_s flags, dropped and empty packets) the ranges of a
    stream equal the matching slices of a fresh-carry vb200_decode_streams_packets call, and got follows its lengths"""
    _need()
    ch, rate, q = CASES[0]
    buf, hdr, audios = make_streams(ch, rate, q)
    ctx = _ctx(drivers, buf, hdr)
    rng = np.random.default_rng(100 + seed)
    fuzzed = []
    for a in audios:
        a = a.copy()
        n = len(a)
        a[:, 4] += np.cumsum(rng.random(n) < 0.1)               # packetno gaps
        gp = np.where(rng.random(n) < 0.3, a[:, 2] - rng.integers(-3000, 3000, n), -1)
        a[:, 2] = np.where(gp < -1, -1, gp)
        a[:, 3] = rng.random(n) < 0.05                          # e_o_s on a few packets, not only the last
        a[rng.random(n) < 0.05, 1] = 0                          # dropped as empty
        fuzzed.append(a)
    npkt, info = _table(fuzzed)
    full = ctx.decode_streams_packets(npkt, info, buf, ctx.decode_streams_carry(len(fuzzed)))
    idx = ctx.decode_streams_index(npkt, info, buf)
    length = np.diff(full["pcm_base"])
    assert (idx["length"] == length).all()
    out_stride = int(npkt.max()) * (ctx.bs[1] // 2) + 64       # holds even a stream whose blocks return nothing
    req = []
    for s in range(len(fuzzed)):
        req.append((0, s, out_stride))
        for _ in range(6):
            req.append((int(rng.integers(0, max(int(length[s]), 1) + 50)), s, int(rng.integers(0, 4000))))
    req = np.array(req, abi.PCM_RANGE_DTYPE)
    r = ctx.decode_ranges(npkt, info, buf, req, out_stride)
    for i, (start, s, n) in enumerate(req.tolist()):
        got = min(n, max(0, int(length[s]) - start))
        assert r["got"][i] == got, (seed, i, start, s, n)
        want = full["pcm"][s][:, start:start + got]
        assert np.array_equal(r["pcm"][i][:, :got].view(np.uint32), want.view(np.uint32)), (seed, i)


def test_capacity_guard(cuda_ok, drivers):  # noqa: F811
    """eight packets in the middle of a stream, each after a packetno gap and with a granulepos far behind the count,
    return nothing: a short range across them needs more blocks than its out_stride gives"""
    _need()
    buf, hdr, audios = make_streams(2, 44100, 0.5)
    ctx = _ctx(drivers, buf, hdr)
    a = audios[1].copy()
    m = len(a) // 2
    for k in range(m, m + 8):
        a[k:, 4] += 1
    a[m:m + 8, 2] = -(1 << 20)            # behind by more than any block, but by less than 2^31: the reference's
                                          # pcm_returned is an int
    crafted = [audios[0], a, audios[2]]
    whole = _stock(buf, hdr, crafted, 2)
    idx = ctx.decode_streams_index(*_table(crafted), buf)
    o = idx["out"][1]
    assert (o["samples"][m:m + 8] == 0).all() and o["samples"][m - 1] > 0 and o["samples"][m + 8] > 0
    start = int(o[m]["pcm_offset"]) - 250
    stride = 512
    nblk, _ = dr.capacity(stride, ctx.bs, 2)
    assert nblk < 11                                        # priming, m - 1, the eight, m + 8
    req = np.array([(0, 0, 500), (start, 1, 500), (100, 2, stride)], abi.PCM_RANGE_DTYPE)
    npkt, info = _table(crafted)
    r = ctx.decode_ranges(npkt, info, buf, req, stride)
    assert r["got"][1] == EINVAL and not r["pcm"][1].view(np.uint32).any()
    ok = req[[0, 2]]
    _check_ranges({"got": r["got"][[0, 2]], "pcm": r["pcm"][[0, 2]]}, ok, whole, False, "beside the guard")
    big = 1 << 16
    r2 = ctx.decode_ranges(npkt, info, buf, req, big)
    _check_ranges(r2, req, whole, False, "retry")


def test_dev_forms_launches_and_errors(cuda_ok, drivers):  # noqa: F811
    import torch
    _need()
    buf, hdr, audios = make_streams(2, 44100, 0.5)
    ctx = _ctx(drivers, buf, hdr)
    ns, ch = len(audios), 2
    npkt, info = _table(audios)
    whole = _stock(buf, hdr, audios, ch)
    idx = ctx.decode_streams_index(npkt, info, buf)
    stride = 3000
    req = _requests(audios, whole, idx, stride, np.random.default_rng(1))
    want = ctx.decode_ranges(npkt, info, buf, req, stride, s16=True)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_npkt, d_info, d_data = t(npkt), t(info.view(np.uint8)), t(buf)
    # _dev index
    d_len = torch.zeros(ns, dtype=torch.int64, device=dev)
    d_out = torch.zeros(info.size * abi.DECODED_PACKET_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    ctx.decode_streams_index_dev(ns, info.shape[1], d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(),
                                 d_len.data_ptr(), d_out.data_ptr())
    torch.cuda.synchronize()
    assert (d_len.cpu().numpy() == idx["length"]).all()
    dout = d_out.cpu().numpy().view(abi.DECODED_PACKET_DTYPE).reshape(info.shape)
    for s in range(ns):                                     # entries past npkt[s] are not written
        assert dout[s, :npkt[s]].tobytes() == idx["out"][s, :npkt[s]].tobytes()
    # _dev ranges, int16, with bad requests appended: per-request VB200_EINVAL
    bad = np.array([(0, ns, 10), (-1, 0, 10), (0, 0, -1), (0, 0, stride + 1), (0, -1, 5)], abi.PCM_RANGE_DTYPE)
    allreq = np.concatenate([req, bad])
    d_req = t(allreq.view(np.uint8))
    d_pcm = torch.full((len(allreq) * stride * ch,), 7, dtype=torch.int16, device=dev)
    d_got = torch.zeros(len(allreq), dtype=torch.int32, device=dev)
    ctx.decode_ranges_dev(ns, info.shape[1], d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(), len(allreq),
                          d_req.data_ptr(), 1, d_pcm.data_ptr(), stride, d_got.data_ptr())
    torch.cuda.synchronize()
    got = d_got.cpu().numpy()
    pcm = d_pcm.cpu().numpy().reshape(len(allreq), stride, ch)
    assert (got[:len(req)] == want["got"]).all() and (got[len(req):] == EINVAL).all()
    assert np.array_equal(pcm[:len(req)], want["pcm"]) and not pcm[len(req):].any()
    # a fixed number of launches, whatever nreq and nstreams
    counts = []
    for n, nr in ((2, 2), (12, 40)):
        sel = [audios[i % ns] for i in range(n)]
        q = np.array([(100 * i, i % n, 2000) for i in range(nr)], abi.PCM_RANGE_DTYPE)
        l0 = ctx.launch_count()
        ctx.decode_streams_index(*_table(sel), buf)
        l1 = ctx.launch_count()
        ctx.decode_ranges(*_table(sel), buf, q, 2000)
        counts.append((l1 - l0, ctx.launch_count() - l1))
    assert counts == [(2, 3), (2, 3)]
    # errors of the host forms
    L, h = ctx.L, ctx.h
    g = np.zeros(len(req), np.int32)
    host = np.zeros(len(req) * ch * stride, np.float32)
    length = np.zeros(ns, np.int64)
    outs = np.zeros(info.shape, abi.DECODED_PACKET_DTYPE)

    def call(npkt_=npkt, info_=info, data=buf, nbytes=None, req_=req, nreq=None, pcm=host, mp=info.shape[1],
             stride_=stride, got=g):
        p = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        return L.vb200_decode_ranges(h, ns, mp, p(npkt_), p(info_), p(data), buf.size if nbytes is None else nbytes,
                                     len(req) if nreq is None else nreq, p(req_), 0, p(pcm), stride_, p(got))

    def index(npkt_=npkt, info_=info, data=buf, nbytes=None, mp=info.shape[1], length_=length):
        p = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        return L.vb200_decode_streams_index(h, ns, mp, p(npkt_), p(info_), p(data),
                                            buf.size if nbytes is None else nbytes, p(length_), outs.ctypes.data)
    assert call() == 0 and index() == 0
    for kw in ({"npkt_": None}, {"info_": None}, {"data": None}, {"req_": None}, {"pcm": None}, {"got": None},
               {"nreq": -1}, {"mp": 0}, {"nbytes": buf.size - 1}, {"npkt_": npkt + np.int32(info.shape[1])},
               {"npkt_": npkt - np.int32(1000)}):
        assert call(**kw) == EINVAL, kw
    for b in bad:
        assert call(req_=np.array([b] * len(req), abi.PCM_RANGE_DTYPE)) == EINVAL, b
    badinfo = info.copy()
    badinfo["offset"][0, 0] = -1
    assert call(info_=badinfo) == EINVAL and index(info_=badinfo) == EINVAL
    for kw in ({"npkt_": None}, {"info_": None}, {"data": None}, {"length_": None}, {"mp": 0},
               {"nbytes": buf.size - 1}, {"npkt_": npkt + np.int32(info.shape[1])}):
        assert index(**kw) == EINVAL, kw
    assert L.vb200_decode_ranges_dev(h, ns, info.shape[1], d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(),
                                     len(req), None, 0, d_pcm.data_ptr(), stride, d_got.data_ptr(), None) == EINVAL
    assert L.vb200_decode_streams_index_dev(h, ns, info.shape[1], None, d_info.data_ptr(), d_data.data_ptr(),
                                            d_len.data_ptr(), d_out.data_ptr(), None) == EINVAL
    # no entropy setup registered
    import os
    from conftest import ROOT
    from vorbis_b200 import lib
    setup = abi.SetupHolder.load(os.path.join(ROOT, "tests", "golden", "setup_44k_stereo_q5.npz"))
    bare = lib.Context(setup, device=0)
    with pytest.raises(lib.VB200Error, match="entropy_setup"):
        bare.decode_ranges(npkt, info, buf, req, stride)
    with pytest.raises(lib.VB200Error, match="entropy_setup"):
        bare.decode_streams_index(npkt, info, buf)


def test_pcm_range_layout():
    class R(C.Structure):
        _fields_ = [("start", C.c_int64), ("stream", C.c_int32), ("length", C.c_int32)]
    assert C.sizeof(R) == abi.PCM_RANGE_DTYPE.itemsize
    for name, _ in R._fields_:
        assert getattr(R, name).offset == abi.PCM_RANGE_DTYPE.fields[name][1]
