"""Whole streams from packets on the device (vb200_decode_streams_packets[_dev]) against the stock decoder:
- on four setups (the last one 512/4096), seven streams each (tests/test_decode_streams_oracle.py make_streams: a
  stream shorter than a long block, a partial last packet, a non-audio packet, a truncated packet, a zero-byte packet,
  a packetno gap, a beginning trim), granulepos on every packet and on page-final packets only: float PCM bit for bit
  as the stock pcmout loop returns it, int16 as decoder_example converts it, and each packet's status, samples and
  granulepos;
- a seeded schedule of 0-5 packets per stream per call, and one packet per call, equal one call; restarting one
  stream's carry mid-way and feeding it again reproduces it;
- half rate against the stock half-rate decoder, and a full-rate carry refused in half-rate mode;
- vb200_encode_streams_packets' info and data passed straight in;
- pcm_cap one sample short: VB200_EINVAL with pcm_base filled and the carries unchanged, then the retry;
- bad arguments give error codes; the _dev form on device-resident packets equals the host form; the launch count
  does not grow with the stream count."""
import numpy as np
import pytest

from oracle import decode
from oracle import decode_packets as dp
from oracle import decode_streams as ds
from oracle import halfrate
from test_decode_streams_oracle import CASES, make_streams
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
EINVAL = -131


def _need():
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


_drivers = {}


@pytest.fixture(scope="module")
def drivers():
    yield _drivers
    for d in _drivers.values():
        d.close()
    _drivers.clear()


def _ctx(drivers, buf, hdr):
    key = bytes(buf[int(hdr[0, 0]):int(hdr[2, 0] + hdr[2, 1])])
    if key not in drivers:
        rows = np.array(hdr, np.int64).copy()
        meta = np.concatenate([rows, rows[:1]])              # Packets wants at least one audio row; it is not read
        drivers[key] = dp.Driver(decode.Packets(buf, meta))
        assert drivers[key].on_device
    return drivers[key].ctx


def _table(audios, ranges=None):
    """audio rows of each stream (rows [a, b) of stream s where ranges is given) -> (npkt, info)"""
    ranges = ranges or [(0, len(a)) for a in audios]
    npkt = np.array([b - a for a, b in ranges], np.int32)
    info = np.zeros((len(audios), max(1, int(npkt.max()))), abi.PACKET_INFO_DTYPE)
    for s, (a, b) in enumerate(ranges):
        m = audios[s][a:b]
        info["offset"][s, :b - a], info["bytes"][s, :b - a] = m[:, 0], m[:, 1]
        info["granulepos"][s, :b - a], info["e_o_s"][s, :b - a], info["packetno"][s, :b - a] = m[:, 2], m[:, 3], m[:, 4]
    return npkt, info


def _stock(buf, hdr, audios, ch, half=False):
    return [ds.ref_decode(buf, hdr, a, ch, halfrate=half) for a in audios]


def _check(got, want, ch, s16, what):
    for s, (pcm, rec, _) in enumerate(want):
        n = len(rec)
        o = got["out"][s, :n]
        assert (o["status"] == rec[:, 0]).all(), "%s stream %d: status" % (what, s)
        assert (o["samples"] == rec[:, 2]).all(), "%s stream %d: samples" % (what, s)
        assert (o["granulepos"] == rec[:, 3]).all(), "%s stream %d: granulepos" % (what, s)
        assert (o["pcm_offset"] == np.cumsum(rec[:, 2]) - rec[:, 2]).all(), "%s stream %d: pcm_offset" % (what, s)
        g = got["pcm"][s]
        if s16:
            assert np.array_equal(g, ds.s16_of(pcm)), "%s stream %d: int16 PCM" % (what, s)
        else:
            assert g.shape == pcm.shape and np.array_equal(g.view(np.uint32), pcm.view(np.uint32)), \
                "%s stream %d: PCM" % (what, s)


def _schedule_run(ctx, buf, audios, sched, s16=False, carry=None):
    """the streams fed in calls of sched[i][s] packets each: (concatenated per-stream PCM, out rows per stream)"""
    ns = len(audios)
    carry = carry or ctx.decode_streams_carry(ns)
    pos = [0] * ns
    pcm = [[] for _ in range(ns)]
    outs = [[] for _ in range(ns)]
    for row in sched:
        ranges = [(pos[s], min(len(audios[s]), pos[s] + int(row[s]))) for s in range(ns)]
        npkt, info = _table(audios, ranges)
        r = ctx.decode_streams_packets(npkt, info, buf, carry, s16=s16)
        for s in range(ns):
            pcm[s].append(r["pcm"][s])
            outs[s].append(r["out"][s, :npkt[s]])
            pos[s] = ranges[s][1]
        if all(pos[s] == len(audios[s]) for s in range(ns)):
            break
    assert all(pos[s] == len(audios[s]) for s in range(ns))
    cat = [np.concatenate(p, axis=0 if s16 else 1) for p in pcm]
    return cat, [np.concatenate(o) for o in outs]


@pytest.mark.parametrize("ch,rate,q", CASES)
@pytest.mark.parametrize("page_final", [False, True])
def test_streams_equal_stock_decoder(cuda_ok, drivers, ch, rate, q, page_final):
    _need()
    buf, hdr, audios = make_streams(ch, rate, q, page_final)
    ctx = _ctx(drivers, buf, hdr)
    want = _stock(buf, hdr, audios, ch)
    npkt, info = _table(audios)
    for s16 in (False, True):
        got = ctx.decode_streams_packets(npkt, info, buf, ctx.decode_streams_carry(len(audios)), s16=s16)
        assert (np.diff(got["pcm_base"]) == [p.shape[1] for p, _, _ in want]).all()
        _check(got, want, ch, s16, "one call s16=%s" % s16)
    # pieces: a seeded schedule of 0-5 packets per stream per call, and one packet per call
    one = ctx.decode_streams_packets(npkt, info, buf, ctx.decode_streams_carry(len(audios)))
    rng = np.random.default_rng(rate + ch + int(10 * q) + page_final)
    longest = max(len(a) for a in audios)
    for sched in (rng.integers(0, 6, (8 * longest, len(audios))), np.ones((longest, len(audios)), np.int32)):
        pcm, outs = _schedule_run(ctx, buf, audios, sched)
        for s in range(len(audios)):
            assert np.array_equal(pcm[s].view(np.uint32), one["pcm"][s].view(np.uint32)), "pieces: stream %d" % s
            o, w = outs[s], one["out"][s, :len(audios[s])]
            for f in ("granulepos", "samples", "status"):
                assert (o[f] == w[f]).all(), "pieces: stream %d %s" % (s, f)


@pytest.mark.parametrize("ch,rate,q", CASES[:2])
def test_restart_one_stream(cuda_ok, drivers, ch, rate, q):
    """carry_init on one stream's slot mid-way (vorbis_synthesis_restart): fed again from its first packet, that stream
    reproduces its one-call output while the others continue"""
    _need()
    buf, hdr, audios = make_streams(ch, rate, q)
    ctx = _ctx(drivers, buf, hdr)
    ns = len(audios)
    npkt, info = _table(audios)
    one = ctx.decode_streams_packets(npkt, info, buf, ctx.decode_streams_carry(ns))
    carry = ctx.decode_streams_carry(ns)
    half = [len(a) // 2 for a in audios]
    first = ctx.decode_streams_packets(*_table(audios, [(0, h) for h in half]), buf, carry)
    ctx.decode_streams_carry_init(carry, stream=1)
    ranges = [(h, len(a)) for h, a in zip(half, audios)]
    ranges[1] = (0, len(audios[1]))
    second = ctx.decode_streams_packets(*_table(audios, ranges), buf, carry)
    assert np.array_equal(second["pcm"][1].view(np.uint32), one["pcm"][1].view(np.uint32))
    for s in (0, 2, 5):
        cat = np.concatenate([first["pcm"][s], second["pcm"][s]], axis=1)
        assert np.array_equal(cat.view(np.uint32), one["pcm"][s].view(np.uint32)), "stream %d" % s


@pytest.mark.parametrize("ch,rate,q", [CASES[0], CASES[3]])
def test_halfrate_equals_stock_halfrate_decoder(cuda_ok, drivers, ch, rate, q):
    _need()
    buf, hdr, audios = make_streams(ch, rate, q, page_final=True)
    ctx = _ctx(drivers, buf, hdr)
    enc = decode.encode(ch, rate, q, np.zeros((ch, 4096), np.float32))
    win = halfrate.ref_decode((enc.buf, enc.meta[:, 1].copy()), ctx.bs, ch, 8192, halfrate=True)
    full_carry = ctx.decode_streams_carry(len(audios))
    ctx.synthesis_halfrate(True, [win["window0"], win["window1"]])
    try:
        want = _stock(buf, hdr, audios, ch, half=True)
        npkt, info = _table(audios)
        got = ctx.decode_streams_packets(npkt, info, buf, ctx.decode_streams_carry(len(audios)))
        _check(got, want, ch, False, "half rate")
        rng = np.random.default_rng(5)
        pcm, _ = _schedule_run(ctx, buf, audios, rng.integers(0, 6, (400, len(audios))))
        for s in range(len(audios)):
            assert np.array_equal(pcm[s].view(np.uint32), got["pcm"][s].view(np.uint32)), "half rate pieces %d" % s
        r = ctx.decode_streams_packets(npkt, info, buf, full_carry, check=False)
        assert r["rc"] == EINVAL
    finally:
        ctx.synthesis_halfrate(False)


def test_encoder_packets_straight_in(cuda_ok, drivers):
    """vb200_encode_streams_packets' info and data, unchanged, decode as the stock decoder decodes those packets"""
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
    got = ctx.decode_streams_packets(e["nblocks"], info, data, ctx.decode_streams_carry(len(caps)))
    buf = np.concatenate([stock.buf, data])
    want = []
    for s in range(len(caps)):
        r = info[s, :e["nblocks"][s]]
        rows = np.stack([r["offset"] + len(stock.buf), r["bytes"], r["granulepos"], r["e_o_s"], r["packetno"]], 1)
        want.append(ds.ref_decode(buf, stock.hdr, rows.astype(np.int64), ch))
    _check(got, want, ch, False, "encoder output")
    assert sum(p.shape[1] for p, _, _ in want) > 0


def test_overflow_leaves_carries_and_retry_equals_one_call(cuda_ok, drivers):
    _need()
    buf, hdr, audios = make_streams(2, 44100, 0.5)
    ctx = _ctx(drivers, buf, hdr)
    ns, ch = len(audios), 2
    half = [len(a) // 2 for a in audios]
    one = ctx.decode_streams_packets(*_table(audios), buf, ctx.decode_streams_carry(ns))
    carry = ctx.decode_streams_carry(ns)
    a = ctx.decode_streams_packets(*_table(audios, [(0, h) for h in half]), buf, carry)
    before = carry.read()
    second = _table(audios, [(h, len(x)) for h, x in zip(half, audios)])
    need = ctx.decode_streams_packets(*second, buf, carry)
    total = int(need["pcm_base"][-1])
    carry.write(before)
    r = ctx.decode_streams_packets(*second, buf, carry, pcm_cap=total * ch - 1, check=False)
    assert r["rc"] == EINVAL
    assert r["pcm_base"][-1] == total and (r["out"]["samples"] >= 0).all()
    assert np.array_equal(carry.read(), before), "a call that does not fit changed the carries"
    b = ctx.decode_streams_packets(*second, buf, carry, pcm_cap=total * ch)
    assert (b["pcm_base"] == r["pcm_base"]).all()
    for s in range(ns):
        cat = np.concatenate([a["pcm"][s], b["pcm"][s]], axis=1)
        assert np.array_equal(cat.view(np.uint32), one["pcm"][s].view(np.uint32)), "retry stream %d" % s


def test_dev_form_launches_and_errors(cuda_ok, drivers):
    import torch
    _need()
    buf, hdr, audios = make_streams(2, 44100, 0.5)
    ctx = _ctx(drivers, buf, hdr)
    ns, ch = len(audios), 2
    npkt, info = _table(audios)
    want = ctx.decode_streams_packets(npkt, info, buf, ctx.decode_streams_carry(ns), s16=True)
    # the _dev form on device-resident packets, int16
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_npkt, d_info, d_data = t(npkt), t(info.view(np.uint8)), t(buf)
    cap = int(npkt.sum()) * (ctx.bs[1] // 2) * ch
    d_pcm = torch.zeros(cap, dtype=torch.int16, device=dev)
    d_base = torch.zeros(ns + 1, dtype=torch.int64, device=dev)
    d_out = torch.zeros(info.size * abi.DECODED_PACKET_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    carry = ctx.decode_streams_carry(ns)
    torch.cuda.synchronize()
    ctx.decode_streams_packets_dev(ns, info.shape[1], d_npkt.data_ptr(), d_info.data_ptr(), d_data.data_ptr(), carry.ptr,
                                   1, d_pcm.data_ptr(), cap, d_base.data_ptr(), d_out.data_ptr())
    torch.cuda.synchronize()
    base = d_base.cpu().numpy()
    assert (base == want["pcm_base"]).all()
    pcm = d_pcm.cpu().numpy()
    for s in range(ns):
        assert np.array_equal(pcm[base[s] * ch:base[s + 1] * ch].reshape(-1, ch), want["pcm"][s])
    out = d_out.cpu().numpy().view(abi.DECODED_PACKET_DTYPE).reshape(info.shape)
    for s in range(ns):
        assert (out[s, :npkt[s]] == want["out"][s, :npkt[s]]).all()
    # a fixed number of launches, whatever the stream count
    counts = []
    for n in (2, 12):
        sel = [audios[i % ns] for i in range(n)]
        k = ctx.decode_streams_carry(n)
        l0 = ctx.launch_count()
        ctx.decode_streams_packets(*_table(sel), buf, k)
        counts.append(ctx.launch_count() - l0)
    assert counts == [5, 5]
    # errors
    L, h = ctx.L, ctx.h
    base = np.zeros(ns + 1, np.int64)
    outs = np.zeros(info.shape, abi.DECODED_PACKET_DTYPE)
    host = np.zeros(cap, np.float32)

    def call(npkt_=npkt, info_=info, data=buf, nbytes=None, carry_ptr=carry.ptr, pcm=host, mp=info.shape[1]):
        return L.vb200_decode_streams_packets(h, ns, mp, None if npkt_ is None else npkt_.ctypes.data,
                                              None if info_ is None else info_.ctypes.data,
                                              None if data is None else data.ctypes.data,
                                              buf.size if nbytes is None else nbytes, carry_ptr, 0,
                                              None if pcm is None else pcm.ctypes.data, cap, base.ctypes.data,
                                              outs.ctypes.data)
    assert call() == 0
    assert call(npkt_=None) == EINVAL and call(info_=None) == EINVAL and call(data=None) == EINVAL
    assert call(carry_ptr=None) == EINVAL and call(pcm=None) == EINVAL and call(mp=0) == EINVAL
    assert call(nbytes=buf.size - 1) == EINVAL                           # the last packet ends past data
    bad = info.copy()
    bad["offset"][0, 0] = -1
    assert call(info_=bad) == EINVAL
    assert call(npkt_=npkt + np.int32(info.shape[1])) == EINVAL         # npkt > max_packets
    assert call(npkt_=npkt - np.int32(1000)) == EINVAL                  # npkt < 0
    assert L.vb200_decode_streams_packets_dev(h, ns, info.shape[1], None, d_info.data_ptr(), d_data.data_ptr(),
                                              carry.ptr, 0, d_pcm.data_ptr(), cap, d_base.data_ptr(),
                                              d_out.data_ptr(), None) == EINVAL
    assert L.vb200_decode_streams_carry_init(h, 1, None) == EINVAL
    # no entropy setup registered
    import os
    from conftest import ROOT
    setup = abi.SetupHolder.load(os.path.join(ROOT, "tests", "golden", "setup_44k_stereo_q5.npz"))
    bare = lib.Context(setup, device=0)
    k = bare.decode_streams_carry(ns)
    with pytest.raises(lib.VB200Error, match="entropy_setup"):
        bare.decode_streams_packets(npkt, info, buf, k)
