"""vb200_decode_dsp_resume[_dev]: the decode chain continued across calls through a carry of the overlap state.
Cutting every stream's blocks into any sequence of calls that pass the carry along gives, bit for bit, the PCM of
one vb200_decode_dsp call over all of them, which equals the CPU oracle's; at full and half rate, in float and
int16, on the real streams of the decode fixtures and on random block sequences with all four overlap cases."""
import ctypes as C

import numpy as np
import pytest

from conftest import CONFIG_NAMES, assert_bits_equal, load_npz
from oracle import halfrate
from test_halfrate_oracle import halfrate_setup
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu

EINVAL = -131


@pytest.fixture(scope="module", params=CONFIG_NAMES)
def cfg(request, oracle_lib, cuda_ok):
    name = request.param
    setup, _ = halfrate_setup(name)
    full = vlib.Context(setup)
    half = vlib.Context(setup)
    half.synthesis_halfrate(1, setup.halfrate_windows())
    oracles = {"full": oracle_lib.Oracle(setup), "half": halfrate.Oracle.create(setup, setup.halfrate_windows())}
    return name, setup, {"full": full, "half": half}, oracles, load_npz("decode", name)


def _s16(x):
    """examples/decoder_example.c:250-262 on [ns][ch][len] float -> interleaved [ns][len][ch] int16"""
    return np.clip(np.floor(x * np.float32(32767.0) + np.float32(0.5)), -32768, 32767).astype(np.int16).transpose(0, 2, 1)


def _finished(prev, Ws, bs, hr):
    """samples a run of blocks Ws finishes after a block of flag prev (-1: nothing before it)"""
    n = 0
    for w in Ws:
        if prev >= 0:
            n += (bs[prev] // 4 + bs[w] // 4) >> hr
        prev = int(w)
    return n


class Stream:
    """the inputs of ns streams as vb200_decode_dsp takes them, and the cutting of them into resumed calls"""

    def __init__(self, ctx, Wseq, res, posts, present):
        self.ctx, self.Wseq = ctx, np.ascontiguousarray(Wseq, np.int32)
        self.ns, self.nblk = self.Wseq.shape
        self.hr = ctx.halfrate
        self.co, self.po, clen, self.plen = vlib.synthesis_layout(self.Wseq, ctx.bs, ctx.channels, halfrate=self.hr)
        assert res.size == clen
        self.res = np.ascontiguousarray(res, np.float32)
        self.posts = np.ascontiguousarray(posts, np.int32).reshape(self.ns, self.nblk, ctx.channels, abi.FLOOR1_STRIDE)
        self.present = np.ascontiguousarray(present, np.int32).reshape(self.ns, self.nblk, ctx.channels)

    def one_call(self, s16):
        return self.ctx.decode_dsp(self.Wseq, self.co, self.res, self.posts, self.present, self.po, self.plen, s16=s16)

    def piece(self, pos, counts, carry_W):
        """the arguments of one resumed call that decodes counts[s] blocks of stream s from block pos[s]"""
        ch, bs = self.ctx.channels, self.ctx.bs
        m = max(1, int(counts.max()))
        Wc = np.zeros((self.ns, m), np.int32)
        posts = np.zeros((self.ns, m, ch, abi.FLOOR1_STRIDE), np.int32)
        present = np.zeros((self.ns, m, ch), np.int32)
        for s in range(self.ns):
            Wc[s, :counts[s]] = self.Wseq[s, pos[s]:pos[s] + counts[s]]
            posts[s, :counts[s]] = self.posts[s, pos[s]:pos[s] + counts[s]]
            present[s, :counts[s]] = self.present[s, pos[s]:pos[s] + counts[s]]
        co, po, clen, plen = vlib.synthesis_layout(Wc, bs, ch, halfrate=self.hr, carry_W=carry_W, count=counts)
        res = np.zeros(max(clen, 1), np.float32)
        for s in range(self.ns):
            for k in range(counts[s]):
                n = ch * bs[Wc[s, k]] // 2
                src = self.co[s, pos[s] + k]
                res[co[s, k]:co[s, k] + n] = self.res[src:src + n]
        lens = [_finished(int(carry_W[s, 0]), Wc[s, :counts[s]], bs, self.hr) for s in range(self.ns)]
        assert max(lens) == plen
        return Wc, co, res, posts, present, po, max(plen, 1), lens

    def resumed(self, schedule, s16, call=None):
        """decode the streams in the calls of schedule (a list of per-stream block counts); returns every stream's
        concatenated PCM and the final carry.  Checks that a stream with count 0 leaves its carry as it was."""
        ctx = self.ctx
        call = call or (lambda args, carry, counts: ctx.decode_dsp_resume(*args, carry, count=counts, s16=s16))
        carry = ctx.new_decode_carry(self.ns)
        pos = np.zeros(self.ns, np.int64)
        out = [[] for _ in range(self.ns)]
        for counts in schedule:
            counts = np.asarray(counts, np.int32)
            Wc, co, res, posts, present, po, plen, lens = self.piece(pos, counts, carry[1])
            before = (carry[0].copy(), carry[1].copy())
            pcm = call((Wc, co, res, posts, present, po, plen), carry, counts)
            for s in range(self.ns):
                out[s].append(pcm[s][:lens[s]] if s16 else pcm[s][:, :lens[s]])
                if counts[s] == 0:
                    assert_bits_equal(carry[0][s], before[0][s], "idle stream's carried tail")
                    assert np.array_equal(carry[1][s], before[1][s]), "idle stream's carried W"
                else:
                    assert (carry[1][s] == Wc[s, counts[s] - 1]).all()
            pos += counts
        assert (pos == self.nblk).all()
        return [np.concatenate(o, axis=0 if s16 else 1) for o in out], carry


def _schedules(rng, ns, nblk):
    """whole in one call; 2 and 3 uneven pieces, cut differently per stream (some streams idle in a call);
    one block per call"""
    yield "one call", [[nblk] * ns]
    for parts in (2, 3):
        cuts = [np.sort(rng.choice(np.arange(0, nblk + 1), parts - 1, replace=True)) for _ in range(ns)]
        sched = [[int(np.diff(np.concatenate([[0], c, [nblk]]))[p]) for c in cuts] for p in range(parts)]
        yield "%d pieces" % parts, sched
    yield "one block per call", [[1] * ns] * nblk


def _check(st, oracle, rng, s16, what):
    whole = st.one_call(False)
    want = oracle.decode_dsp(st.Wseq, st.co, st.res, st.posts, st.present, st.po, st.plen)
    assert_bits_equal(whole, want, what + ": decode_dsp vs oracle")
    if s16:
        whole = st.one_call(True)
        assert np.array_equal(whole, _s16(want)), what + ": decode_dsp int16 vs oracle"
    for sname, sched in _schedules(rng, st.ns, st.nblk):
        got, _ = st.resumed(sched, s16)
        for s in range(st.ns):
            n = got[s].shape[0 if s16 else 1]
            ref = whole[s][:n] if s16 else whole[s][:, :n]
            assert_bits_equal(got[s], ref, "%s, %s: stream %d" % (what, sname, s))
            rest = whole[s][n:] if s16 else whole[s][:, n:]
            assert not rest.any(), "%s, %s: stream %d is short" % (what, sname, s)


def _random_inputs(ctx, rng, ns, nblk):
    Wseq = rng.integers(0, 2, (ns, nblk)).astype(np.int32)
    Wseq[0] = 1
    Wseq[1] = 0
    coef_len = vlib.synthesis_layout(Wseq, ctx.bs, ctx.channels)[2]
    res = np.rint(rng.standard_normal(coef_len) * 3).astype(np.float32)
    rows = ns * nblk * ctx.channels
    posts = rng.integers(0, 140, (rows, abi.FLOOR1_STRIDE)).astype(np.int32)
    posts[rng.random(posts.shape) < 0.4] |= 0x8000
    posts[:, :2] &= 0x7fff
    present = (rng.random(rows) < 0.9).astype(np.int32)
    return Wseq, res, posts, present


@pytest.mark.parametrize("mode", ["full", "half"])
@pytest.mark.parametrize("s16", [False, True])
def test_golden_stream_resumed(cfg, mode, s16):
    """the real stream of the decode fixture, its blocks cut into resumed calls"""
    name, setup, ctxs, oracles, dec = cfg
    ctx = ctxs[mode]
    Wseq = dec["W"][None, :]
    rows = Wseq.size * ctx.channels
    posts, present = np.full((rows, abi.FLOOR1_STRIDE), 999, np.int32), np.ones(rows, np.int32)
    st = Stream(ctx, Wseq, dec["coef"], posts, present)
    _check(st, oracles[mode], np.random.default_rng(3), s16, "%s %s" % (name, mode))


@pytest.mark.parametrize("mode", ["full", "half"])
@pytest.mark.parametrize("s16", [False, True])
def test_random_streams_resumed(cfg, mode, s16):
    """random long/short sequences (all four overlap cases) and floors, many streams cut differently"""
    name, setup, ctxs, oracles, _ = cfg
    ctx = ctxs[mode]
    rng = np.random.default_rng(77)
    st = Stream(ctx, *_random_inputs(ctx, rng, 7, 17))
    pairs = {(int(a), int(b)) for row in st.Wseq for a, b in zip(row[:-1], row[1:])}
    assert pairs == {(0, 0), (0, 1), (1, 0), (1, 1)}
    _check(st, oracles[mode], rng, s16, "random %s" % mode)


@pytest.mark.parametrize("mode", ["full", "half"])
def test_dev_form_equals_host_form(cfg, mode):
    """vb200_decode_dsp_resume_dev with device buffers (the carry resident on the device between calls) gives
    the host form's PCM and carry"""
    name, setup, ctxs, _, _ = cfg
    ctx = ctxs[mode]
    rng = np.random.default_rng(5)
    st = Stream(ctx, *_random_inputs(ctx, rng, 5, 12))
    sched = [[3, 0, 5, 12, 1], [4, 7, 0, 0, 6], [5, 5, 7, 0, 5]]
    bufs = []

    def put(a):
        a = np.ascontiguousarray(a)
        p = C.c_void_p()
        ctx._chk(ctx.L.vb200_malloc_device(ctx.h, max(a.nbytes, 4), C.byref(p)))
        bufs.append(p)
        ctx._chk(ctx.L.vb200_memcpy_h2d(ctx.h, p, a.ctypes.data, a.nbytes))
        return p.value

    def get(p, like):
        ctx._chk(ctx.L.vb200_synchronize(ctx.h))
        ctx._chk(ctx.L.vb200_memcpy_d2h(ctx.h, like.ctypes.data, p, like.nbytes))
        return like

    try:
        for s16 in (False, True):
            host, host_carry = st.resumed(sched, s16)
            tail0, W0 = ctx.new_decode_carry(st.ns)
            d_tail, d_W = put(tail0), put(W0)

            def dev_call(args, carry, counts):
                Wc, co, res, posts, present, po, plen = args
                shape = (st.ns, plen, ctx.channels) if s16 else (st.ns, ctx.channels, plen)
                pcm = np.zeros(shape, np.int16 if s16 else np.float32)
                d_pcm = put(pcm)
                ctx.decode_dsp_resume_dev(st.ns, Wc.shape[1], put(counts), put(Wc), put(co), put(res), put(posts),
                                          put(present), put(po), d_pcm, 1 if s16 else 0, plen, d_tail, d_W)
                get(d_tail, carry[0])
                get(d_W, carry[1])
                return get(d_pcm, pcm)

            dev, dev_carry = st.resumed(sched, s16, call=dev_call)
            for s in range(st.ns):
                assert_bits_equal(dev[s], host[s], "dev vs host: stream %d" % s)
            assert_bits_equal(dev_carry[0], host_carry[0], "dev vs host: carried tails")
            assert np.array_equal(dev_carry[1], host_carry[1]), "dev vs host: carried W"
    finally:
        for b in bufs:
            ctx.L.vb200_free_device(ctx.h, b)


def test_invalid_arguments(cfg):
    """VB200_EINVAL for a carried W outside {-1, 0, 1}, count[s] outside [0, nblk] and null pointers; a refused
    call leaves the carry as it was"""
    name, setup, ctxs, _, _ = cfg
    ctx = ctxs["full"]
    ns, nblk, ch = 2, 3, ctx.channels
    rng = np.random.default_rng(1)
    Wseq, res, posts, present = _random_inputs(ctx, rng, ns, nblk)
    co, po, clen, plen = vlib.synthesis_layout(Wseq, ctx.bs, ch)
    pcm = np.zeros((ns, ch, plen), np.float32)

    def rc(count=None, W=None, tail_null=False, Wseq_=Wseq, carry_null=False):
        tail, Wc = ctx.new_decode_carry(ns)
        if W is not None:
            Wc[:] = W
        k = abi.DecodeCarry(None if tail_null else tail.ctypes.data, Wc.ctypes.data)
        before = (tail.copy(), Wc.copy())
        cnt = None if count is None else np.asarray(count, np.int32)
        r = ctx.L.vb200_decode_dsp_resume(ctx.h, ns, nblk, vlib._ptr(cnt), Wseq_.ctypes.data, co.ctypes.data,
                                          res.ctypes.data, res.size, posts.ctypes.data, present.ctypes.data,
                                          po.ctypes.data, pcm.ctypes.data, 0, plen, None if carry_null else C.byref(k))
        if r != 0:
            assert np.array_equal(tail, before[0]) and np.array_equal(Wc, before[1])
        return r

    assert rc() == 0
    assert rc(count=[nblk, 0]) == 0
    assert rc(W=0) == 0
    assert rc(W=2) == EINVAL
    assert rc(W=-2) == EINVAL
    assert rc(count=[nblk + 1, 1]) == EINVAL
    assert rc(count=[1, -1]) == EINVAL
    assert rc(tail_null=True) == EINVAL
    assert rc(carry_null=True) == EINVAL
    bad = Wseq.copy()
    bad[1, 2] = 2
    assert rc(Wseq_=bad) == EINVAL
    assert rc(count=[nblk, 2], Wseq_=bad) == 0          # the bad entry lies past count[1]: not read
    k = abi.DecodeCarry(None, None)
    r = ctx.L.vb200_decode_dsp_resume_dev(ctx.h, ns, nblk, None, 1, 1, 1, 1, 1, 1, 1, 0, plen, C.byref(k), None)
    assert r == EINVAL
    r = ctx.L.vb200_decode_dsp_resume_dev(ctx.h, ns, nblk, None, 1, 1, 1, 1, 1, 1, 1, 0, plen, None, None)
    assert r == EINVAL
