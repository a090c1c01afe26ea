"""Whole streams to packets in pieces (vb200_encode_streams_packets[_managed]_resume): a fresh carry with the whole
timeline in one call equals vb200_encode_streams_packets[_managed]; any cut of a stream's timeline into calls that pass
the carry along gives the packets and infos of one call; fed the timeline of a stock encoder written in chunks, the
calls give that encoder's packets.  The stock-encoder comparisons need oracle/_ref (built where the reference sources
exist; the libraries travel)."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_setup, probe_signal
from oracle import bitrate as B
from test_gpu_encode_packets import SETUPS, _driver
from test_gpu_stream_packets import MANAGED, _need_ref, _noise_and_silence, _streams, _timelines
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

VB200_EINVAL = -131
INFO_FIELDS = ("granulepos", "bytes", "e_o_s", "packetno", "choice")


def _cuts(rng, eof, length):
    """increasing buffer ends of one stream's calls: random points up to its EOF sample (some equal: calls with no new
    samples; some a few samples apart: cuts inside a 64-sample step), then the whole timeline with its EOF"""
    k = int(rng.integers(1, 7))
    ends = list(rng.integers(0, eof + 1, k))
    a = int(rng.integers(0, max(eof - 200, 1)))
    ends += [a, a, a + int(rng.integers(1, 64))]
    return sorted(min(e, eof) for e in ends) + [length]


def _feed(ctx, tls, eofs, ends, managed=False, max_blocks=None, mark_steps=0, carry=None, offset=None, rounds=None):
    """Stream s's calls end at ends[s][r] in round r (its last end repeats), eof given with the whole timeline.
    offset[s] is added to the timeline sample of every buffer start (a carry whose base was raised).  Returns per
    stream the packets, info rows and absolute block positions, and the carry."""
    ns, ch = len(tls), tls[0].shape[0]
    bs1 = ctx.bs[1]
    carry = ctx.encode_carry_init(ns, mark_steps) if carry is None else carry
    off = np.zeros(ns, np.int64) if offset is None else np.asarray(offset, np.int64)
    pk, inf, pos = [[] for _ in range(ns)], [[] for _ in range(ns)], [[] for _ in range(ns)]
    rounds = rounds or max(len(e) for e in ends) + 400
    for r in range(rounds):
        head = ctx.encode_carry_head(carry)
        if head["done"].all():
            break
        base = head["base"] - off
        end = np.array([e[min(r, len(e) - 1)] for e in ends], np.int64)
        lens = np.maximum(end - base, 0)                # done streams pass anything
        stride = max(int(lens.max()), bs1) + 3 & ~3
        pcm = np.zeros((ns, ch, stride), np.float32)
        for s in range(ns):
            pcm[s, :, :lens[s]] = tls[s][:, base[s]:end[s]]
        eof = np.array([eofs[s] + off[s] if end[s] == tls[s].shape[1] else 0 for s in range(ns)], np.int64)
        got = ctx.encode_streams_packets_resume(pcm, lens, carry, eof, managed=managed, max_blocks=max_blocks)
        for s in range(ns):
            n = int(got["nblocks"][s])
            assert not head["done"][s] or n == 0, "a done stream emitted packets"
            pk[s] += got["packets"][s]
            inf[s] += list(got["info"][s, :n])
            pos[s] += list(head["base"][s] + got["plan"][s, :n]["pos"].astype(np.int64))
    return pk, inf, pos, carry


def _check(pk, inf, pos, one, what, gshift=0):
    for s in range(len(pk)):
        n = int(one["nblocks"][s])
        assert pk[s] == one["packets"][s], "%s stream %d: packet bytes (%d vs %d packets)" % (what, s, len(pk[s]), n)
        for f in INFO_FIELDS:
            want = one["info"][s, :n][f] + (gshift if f == "granulepos" else 0)
            assert np.array_equal(np.array([r[f] for r in inf[s]]), want), "%s stream %d: %s" % (what, s, f)
        assert np.array_equal(np.array(pos[s]) - (gshift if gshift else 0), one["plan"][s, :n]["pos"]), what


def _vs_capture(pk, inf, caps, what):
    for s, c in enumerate(caps):
        assert pk[s] == c["packets"], "%s stream %d: packets" % (what, s)
        for f in ("granulepos", "e_o_s", "packetno"):
            assert np.array_equal(np.array([r[f] for r in inf[s]]), c[f]), "%s stream %d: %s" % (what, s, f)


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_fresh_carry_one_call_equals_packets_call(cuda_ok, ch, rate, q):
    """contract (a): a fresh carry with every whole timeline in one call gives the packets call's plan, infos and
    bytes; the carries end done, with packetno 3 + blocks and the last granulepos"""
    _need_ref()
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p) for p in _streams(ch, rate, 0.6)]
        tl, pcm_len, eof = _timelines(caps, ch)
        one = ctx.encode_streams_packets(tl, pcm_len, eof)
        carry = ctx.encode_carry_init(len(caps))
        got = ctx.encode_streams_packets_resume(tl, pcm_len, carry, eof)
        for k in ("plan", "nblocks", "info"):
            assert np.array_equal(got[k], one[k]), k
        assert got["packets"] == one["packets"] and got["count"] == one["count"]
        head = ctx.encode_carry_head(carry)
        assert head["done"].all()
        assert np.array_equal(head["packetno"], 3 + one["nblocks"])
        assert np.array_equal(head["granulepos"], [one["info"][s, n - 1]["granulepos"] for s, n in enumerate(one["nblocks"])])
    finally:
        d.close()


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_cuts_equal_one_call_unmanaged(cuda_ok, ch, rate, q):
    """contracts (b) and (c), un-managed: the timelines of stock encoders written in chunks of 64, 1000, 1024, 4410
    samples and all at once, fed in random per-stream cuts, give one call's packets and infos and the stock encoders'
    packets, granulepos, e_o_s and packetno.  The streams of one call are at different phases: some pass no new data,
    some are already done"""
    _need_ref()
    d = _driver(ch, rate, q)
    ctx = d.ctx
    rng = np.random.default_rng(int(rate + 10 * q))
    try:
        sig = _streams(ch, rate, 0.6)
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p, chunk=w or p.shape[1])
                for w in (64, 1000, 1024, 4410, None) for p in sig]
        tl, pcm_len, eof = _timelines(caps, ch)
        one = ctx.encode_streams_packets(tl, pcm_len, eof)
        tls = [c["timeline"] for c in caps]
        ends = [_cuts(rng, int(c["eof"]), c["timeline"].shape[1]) for c in caps]
        pk, inf, pos, carry = _feed(ctx, tls, eof, ends)
        _check(pk, inf, pos, one, "q=%g" % q)
        _vs_capture(pk, inf, caps, "q=%g" % q)
        assert ctx.encode_carry_head(carry)["done"].all()
    finally:
        d.close()


@pytest.mark.parametrize("name,ch,rate,max_br,nominal,min_br,rm2", MANAGED)
def test_cuts_equal_one_call_managed(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2):
    """contracts (a), (b) and (c), bitrate-managed (with truncated and padded packets in the small-reservoir CBR case):
    random per-stream cuts give one managed call's packets and the stock managed encoder's"""
    _need_ref()
    if not B.ref_available(True):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    cf = B.managed(ch, rate, max_br, nominal, min_br, *(rm2 or ()))
    info, _ = B.ref_bitrate_info(cf)
    d = B.ManagedDriver(ch, rate, max_br, nominal, min_br)
    ctx = d.ctx
    rng = np.random.default_rng(len(name))
    try:
        early = ctx.encode_carry_init(1)          # made before the bitrate setup: no bitrate state
        ctx.bitrate_setup(info)
        sig = _streams(ch, rate, 0.8)
        if rm2:
            sig = [_noise_and_silence(ch, rate, 1.5, 1), _noise_and_silence(ch, rate, 1.0, 2)] + sig
        caps = [B.ref_stream_capture(cf, p, chunk=w) for w in (1000, 4410) for p in sig]
        tl, pcm_len, eof = _timelines(caps, ch)
        one = ctx.encode_streams_packets(tl, pcm_len, eof, managed=True)
        assert ctx.encode_streams_packets_resume(tl[:1], pcm_len[:1], early, eof[:1], managed=True,
                                                 check=False)["rc"] == VB200_EINVAL
        fresh = ctx.encode_streams_packets_resume(tl, pcm_len, ctx.encode_carry_init(len(caps)), eof, managed=True)
        assert np.array_equal(fresh["info"], one["info"]) and fresh["packets"] == one["packets"]
        ends = [_cuts(rng, int(c["eof"]), c["timeline"].shape[1]) for c in caps]
        pk, inf, pos, _ = _feed(ctx, [c["timeline"] for c in caps], eof, ends, managed=True)
        _check(pk, inf, pos, one, name)
        _vs_capture(pk, inf, caps, name)
    finally:
        d.close()


def test_max_blocks_and_base_shift(cuda_ok):
    """max_blocks smaller than a call's blocks: follow-up calls finish the streams with one call's packets (the mark
    window sized for what a cut call keeps); a carry whose base is raised by 2^32 shifts every later granulepos by
    exactly 2^32 and changes no packet byte"""
    _need_ref()
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    rng = np.random.default_rng(5)
    try:
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p) for p in _streams(ch, rate, 0.6)]
        tl, pcm_len, eof = _timelines(caps, ch)
        one = ctx.encode_streams_packets(tl, pcm_len, eof)
        tls = [c["timeline"] for c in caps]
        ends = [_cuts(rng, int(c["eof"]), c["timeline"].shape[1]) for c in caps]
        steps = tl.shape[2] // 64 + 8
        pk, inf, pos, _ = _feed(ctx, tls, eof, ends, max_blocks=3, mark_steps=steps)
        _check(pk, inf, pos, one, "max_blocks=3")
        # one call into every stream, then the base raised by 2^32
        carry = ctx.encode_carry_init(len(caps))
        first = [[e[0]] for e in ends]
        pk0, inf0, pos0, carry = _feed(ctx, tls, eof, first, carry=carry, rounds=1)
        head = carry[:, :8].copy().view(np.int64)
        carry[:, :8] = (head + (1 << 32)).view(np.uint8)
        pk1, inf1, pos1, carry = _feed(ctx, tls, eof, [e[1:] for e in ends], carry=carry,
                                       offset=np.full(len(caps), 1 << 32, np.int64))
        for s in range(len(caps)):
            n0 = len(pk0[s])
            assert pk0[s] + pk1[s] == one["packets"][s]
            g = np.array([r["granulepos"] for r in inf1[s]], np.int64)
            assert np.array_equal(g - (1 << 32), one["info"][s, n0:one["nblocks"][s]]["granulepos"])
            assert np.array_equal(np.array([r["packetno"] for r in inf1[s]]), one["info"][s, n0:one["nblocks"][s]]["packetno"])
    finally:
        d.close()


def test_errors_and_launches(cuda_ok):
    """VB200_EINVAL for a null carry, pcm_len below what the carry kept, eof at or before base, a carry of another
    setup or mark capacity and a mark window overflow, each leaving the carry as it was; launches equal the packets
    call's and do not grow with the stream count"""
    _need_ref()
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    other = lib.Context(load_setup("44k_mono_q4"))
    try:
        cap = B.ref_stream_capture(B.vbr(ch, rate, q), probe_signal(ch, rate, 0.5, seed=2))
        tl, pcm_len, eof = _timelines([cap], ch)
        t = cap["timeline"]
        L = ctx.L
        # a valid io, info and data: only the carry is missing
        io = abi.StreamsIO()
        io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = tl.ctypes.data, lib.PCM_F32_PLANAR, 256, tl.shape[2]
        io.pcm_len, io.eof = pcm_len.ctypes.data, eof.ctypes.data
        plan, nbk = np.zeros((1, 256), abi.STREAM_BLOCK_DTYPE), np.zeros(1, np.int32)
        io.plan, io.nblocks = plan.ctypes.data, nbk.ctypes.data
        io.cap[0] = io.cap[1] = 256
        info, data = np.zeros(256, abi.PACKET_INFO_DTYPE), np.zeros(1 << 20, np.uint8)
        assert L.vb200_encode_streams_packets_resume(ctx.h, 1, 7, C.byref(io), None, info.ctypes.data,
                                                     data.ctypes.data, data.size) == VB200_EINVAL
        assert L.vb200_encode_streams_packets_resume(ctx.h, 1, 7, C.byref(io), ctx.encode_carry_init(1).ctypes.data,
                                                     info.ctypes.data, data.ctypes.data, data.size) == 0
        carry = ctx.encode_carry_init(1)
        half = np.array([pcm_len[0] // 2], np.int64)
        ctx.encode_streams_packets_resume(tl, half, carry, None)
        head = ctx.encode_carry_head(carry)
        assert head["base"][0] > 0 and head["packetno"][0] > 3 and not head["done"][0]
        kept = half[0] - head["base"][0]
        buf = np.zeros((1, ch, t.shape[1]), np.float32)
        buf[0, :, :t.shape[1] - head["base"][0]] = t[:, head["base"][0]:]
        before = carry.copy()

        def rc(pcm, n, e, c=carry, **kw):
            return ctx.encode_streams_packets_resume(pcm, np.array([n], np.int64), c, e, check=False, **kw)["rc"]
        assert rc(buf, kept - 1, None) == VB200_EINVAL
        assert rc(buf, kept + 64, np.array([head["base"][0]], np.int64)) == VB200_EINVAL
        assert rc(buf, kept + 64, None, c=other.encode_carry_init(1)) == VB200_EINVAL
        two = np.concatenate([carry, ctx.encode_carry_init(2, 99)[:1, :carry.shape[1]]])
        assert ctx.encode_streams_packets_resume(np.concatenate([buf, buf]), np.array([kept, kept], np.int64), two,
                                                 None, check=False)["rc"] == VB200_EINVAL
        # max_blocks=1 on the rest of the timeline with the default window: the analysed lookahead does not fit
        assert rc(buf, t.shape[1] - head["base"][0], np.array([eof[0]]), max_blocks=1) == VB200_EINVAL
        assert np.array_equal(carry, before)
        # launches: as the packets call, whatever the stream count
        l0 = ctx.launch_count()
        ctx.encode_streams_packets(tl, pcm_len, eof)
        fresh = ctx.launch_count() - l0
        for n in (1, 8):
            l0 = ctx.launch_count()
            ctx.encode_streams_packets_resume(np.concatenate([tl] * n), np.concatenate([pcm_len] * n),
                                              ctx.encode_carry_init(n), np.concatenate([eof] * n))
            assert ctx.launch_count() - l0 == fresh <= 40
    finally:
        other.close()
        d.close()
