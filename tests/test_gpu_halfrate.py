"""Half-rate decode on the device (vb200_synthesis_halfrate): vb200_synthesis[_s16][_dev], vb200_decode_dsp[_dev]
and vb200_mdct_backward with the mode on against the CPU oracle (0 ulp, 0 mismatching int16) and against the
reference's own half-rate decode stored in tests/golden/ref/halfrate/halfrate.npz; switching the mode off restores the
full-rate results; and the function-level drop-in shim decodes real streams in half-rate mode bit-identically
to the stock reference."""
import ctypes as C

import numpy as np
import pytest

from conftest import CONFIG_NAMES, assert_bits_equal, load_npz, load_setup, probe_signal
from oracle import halfrate
from refgold import FIXTURE_OF
from test_halfrate_oracle import decode_only_setup, halfrate_setup
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=CONFIG_NAMES)
def cfg(request, cuda_ok):
    name = request.param
    setup, rec = halfrate_setup(name)
    ctx = vlib.Context(setup)
    ctx.synthesis_halfrate(1, setup.halfrate_windows())
    o = halfrate.Oracle.create(setup, setup.halfrate_windows())
    return name, setup, ctx, o, load_npz("decode", name), rec


def _bs(setup):
    return [setup.blocksize(0), setup.blocksize(1)]


def _s16(x):
    """examples/decoder_example.c:250-262 on [ns][ch][len] float -> interleaved [ns][len][ch] int16"""
    return np.clip(np.floor(x * np.float32(32767.0) + np.float32(0.5)), -32768, 32767).astype(np.int16).transpose(0, 2, 1)


def _unit_floor(rows):
    """floor1_inverse2 inputs whose curve is 1.0 everywhere: every post clamps to 255 (lib/floor1.c:1056-1064) and
    FLOOR1_fromdB_LOOKUP[255] is 1.0, so the floor multiply leaves the spectra bit for bit as they are"""
    return np.full((rows, abi.FLOOR1_STRIDE), 999, np.int32), np.ones(rows, np.int32)


def _dev_calls(ctx, Wseq, coef_off, coef, pcm_off, pcm_len, posts, present):
    """vb200_synthesis_s16_dev and vb200_decode_dsp_dev (float and int16); returns their outputs and the res
    decode_dsp_dev leaves in place"""
    ns, nblk = Wseq.shape
    ch = ctx.channels
    bufs = []

    def put(a):
        a = np.ascontiguousarray(a)
        p = C.c_void_p()
        ctx._chk(ctx.L.vb200_malloc_device(ctx.h, a.nbytes, C.byref(p)))
        bufs.append(p)
        ctx._chk(ctx.L.vb200_memcpy_h2d(ctx.h, p, a.ctypes.data, a.nbytes))
        return p.value

    def get(p, like):
        ctx._chk(ctx.L.vb200_synchronize(ctx.h))
        ctx._chk(ctx.L.vb200_memcpy_d2h(ctx.h, like.ctypes.data, p, like.nbytes))
        return like

    try:
        W, co, po = put(Wseq.astype(np.int32)), put(coef_off.astype(np.int64)), put(pcm_off.astype(np.int64))
        c, p, z = put(coef.astype(np.float32)), put(posts.astype(np.int32)), put(present.astype(np.int32))
        zero16, zero32 = np.zeros((ns, pcm_len, ch), np.int16), np.zeros((ns, ch, pcm_len), np.float32)
        s16 = put(zero16)
        ctx.synthesis_s16_dev(ns, nblk, W, co, c, po, s16, pcm_len)
        out = {"synthesis_s16_dev": get(s16, zero16.copy())}
        for fmt in ("f32", "s16"):
            res = put(coef.astype(np.float32))
            pcm = put(zero16 if fmt == "s16" else zero32)
            ctx._chk(ctx.L.vb200_decode_dsp_dev(ctx.h, ns, nblk, W, co, res, p, z, po, pcm, 1 if fmt == "s16" else 0,
                                                pcm_len, None))
            out["decode_dsp_dev_" + fmt] = get(pcm, (zero16 if fmt == "s16" else zero32).copy())
            out["res_" + fmt] = get(res, np.empty(coef.size, np.float32))
        return out
    finally:
        for b in bufs:
            ctx.L.vb200_free_device(ctx.h, b)


def _check_all(ctx, o, Wseq, coef, posts, present, what, want_ref=None):
    """every decode entry point in half-rate mode == the oracle (and, where given, the reference's PCM)"""
    bs, ch = ctx.bs, ctx.channels
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, bs, ch, halfrate=True)
    assert coef_len == coef.size
    want = o.synthesis(Wseq, coef_off, coef, pcm_off, pcm_len)
    want_dsp = o.decode_dsp(Wseq, coef_off, coef, posts, present, pcm_off, pcm_len)
    assert_bits_equal(ctx.synthesis(Wseq, coef_off, coef, pcm_off, pcm_len), want, what + ": synthesis")
    assert_bits_equal(ctx.decode_dsp(Wseq, coef_off, coef, posts, present, pcm_off, pcm_len), want_dsp,
                      what + ": decode_dsp")
    assert np.array_equal(ctx.decode_dsp(Wseq, coef_off, coef, posts, present, pcm_off, pcm_len, s16=True),
                          _s16(want_dsp)), what + ": decode_dsp int16"
    dev = _dev_calls(ctx, Wseq, coef_off, coef, pcm_off, pcm_len, posts, present)
    assert np.array_equal(dev["synthesis_s16_dev"], _s16(want)), what + ": synthesis_s16_dev"
    assert_bits_equal(dev["decode_dsp_dev_f32"], want_dsp, what + ": decode_dsp_dev")
    assert np.array_equal(dev["decode_dsp_dev_s16"], _s16(want_dsp)), what + ": decode_dsp_dev int16"
    if want_ref is not None:
        assert_bits_equal(want[0], want_ref, what + ": oracle vs reference")
    return want, dev


def test_golden_decode_halfrate(cfg):
    """the real streams of the decode fixtures: device == oracle == the reference's half-rate decode"""
    name, setup, ctx, o, dec, rec = cfg
    ch = setup.channels
    Wseq = dec["W"][None, :]
    posts, present = _unit_floor(Wseq.size * ch)
    want, dev = _check_all(ctx, o, Wseq, dec["coef"], posts, present, name, want_ref=rec["pcm"])
    assert np.array_equal(dev["synthesis_s16_dev"][0], _s16(rec["pcm"][None])[0]), "int16 vs reference"
    if setup.c.coupling_steps[0] == 0 and setup.c.coupling_steps[1] == 0:
        # nothing to de-couple and a unit floor: the whole decode chain reproduces the reference's PCM
        assert_bits_equal(dev["decode_dsp_dev_f32"][0], rec["pcm"], "decode_dsp_dev vs reference")


def test_random_streams_halfrate(cfg):
    """many independent streams with random long/short sequences (all four overlap cases), random floors"""
    name, setup, ctx, o, _, _ = cfg
    ch = setup.channels
    rng = np.random.default_rng(4242)
    ns, nblk = 37, 23
    Wseq = rng.integers(0, 2, (ns, nblk)).astype(np.int32)
    Wseq[0] = 1
    Wseq[1] = 0
    pairs = {(int(a), int(b)) for row in Wseq for a, b in zip(row[:-1], row[1:])}
    assert pairs == {(0, 0), (0, 1), (1, 0), (1, 1)}
    coef_len = vlib.synthesis_layout(Wseq, ctx.bs, ch)[2]
    coef = np.rint(rng.standard_normal(coef_len) * 3).astype(np.float32)
    posts = rng.integers(0, 140, (ns * nblk * ch, abi.FLOOR1_STRIDE)).astype(np.int32)
    posts[rng.random(posts.shape) < 0.4] |= 0x8000
    posts[:, :2] &= 0x7fff
    present = (rng.random(ns * nblk * ch) < 0.9).astype(np.int32)
    _check_all(ctx, o, Wseq, coef, posts, present, "random streams")


def test_long_stream_in_overlapping_segments(cfg):
    """a long stream cut into segments that overlap by one block, all decoded in one call, gives the samples
    of the stream decoded whole"""
    name, setup, ctx, o, _, _ = cfg
    ch, bs = setup.channels, ctx.bs
    rng = np.random.default_rng(99)
    nseg, L = 6, 11
    total = 1 + nseg * (L - 1)
    W1 = rng.integers(0, 2, (1, total)).astype(np.int32)
    co1, po1, clen, plen1 = vlib.synthesis_layout(W1, bs, ch, halfrate=True)
    coef = (rng.uniform(-1, 1, clen) * 0.05).astype(np.float32)
    whole = ctx.synthesis(W1, co1, coef, po1, plen1)
    assert_bits_equal(whole, o.synthesis(W1, co1, coef, po1, plen1), "whole stream")
    idx = np.array([np.arange(s * (L - 1), s * (L - 1) + L) for s in range(nseg)])
    Wseg = W1[0][idx]
    _, poS, _, plenS = vlib.synthesis_layout(Wseg, bs, ch, halfrate=True)
    segs = ctx.synthesis(Wseg, co1[0][idx], coef, poS, plenS)
    dev = _dev_calls(ctx, Wseg, co1[0][idx], coef, poS, plenS, *_unit_floor(Wseg.size * ch))
    got = np.concatenate([segs[s][:, :plen_of(Wseg[s], bs)] for s in range(nseg)], axis=1)
    assert_bits_equal(got, whole[0], "segments")
    assert np.array_equal(np.concatenate([dev["synthesis_s16_dev"][s][:plen_of(Wseg[s], bs)] for s in range(nseg)]),
                          _s16(whole)[0]), "segments int16"


def plen_of(W, bs):
    """half-rate samples a segment with block flags W finishes"""
    return int(sum((bs[a] // 4 + bs[b] // 4) >> 1 for a, b in zip(W[:-1], W[1:])))


def test_mdct_backward_halfrate(cfg):
    """vb200_mdct_backward in half-rate mode is mdct_backward at N/2: [nvec][N/4] -> [nvec][N/2]"""
    name, setup, ctx, o, _, _ = cfg
    rng = np.random.default_rng(5)
    for W in (0, 1):
        N = setup.blocksize(W) // 2
        y = rng.uniform(-1, 1, (200, N // 2)).astype(np.float32)
        y[0] = 0.0
        got = ctx.mdct_backward(W, y)
        assert got.shape == (200, N)
        assert_bits_equal(got, o.mdct_backward(W, y), "mdct_backward N=%d" % N)


def test_switching_off_restores_full_rate(cfg):
    """after vb200_synthesis_halfrate(ctx, 0, ...) every decode entry point returns what a context that never
    enabled half-rate returns; decode_dsp's in-place res is the same in both modes"""
    name, setup, ctx, o, dec, _ = cfg
    ch, bs = setup.channels, ctx.bs
    fresh = vlib.Context(setup)
    rng = np.random.default_rng(17)
    ns, nblk = 9, 13
    Wseq = rng.integers(0, 2, (ns, nblk)).astype(np.int32)
    coef_len = vlib.synthesis_layout(Wseq, bs, ch)[2]
    coef = np.rint(rng.standard_normal(coef_len) * 3).astype(np.float32)
    posts = rng.integers(0, 140, (ns * nblk * ch, abi.FLOOR1_STRIDE)).astype(np.int32)
    present = (rng.random(ns * nblk * ch) < 0.9).astype(np.int32)
    y = [rng.uniform(-1, 1, (40, bs[W] // 2)).astype(np.float32) for W in (0, 1)]
    hs_layout = vlib.synthesis_layout(Wseq, bs, ch, halfrate=True)
    res_hs = _dev_calls(ctx, Wseq, hs_layout[0], coef, hs_layout[1], hs_layout[3], posts, present)["res_f32"]
    try:
        ctx.synthesis_halfrate(0)
        co, po, _, plen = vlib.synthesis_layout(Wseq, bs, ch)
        a = _dev_calls(ctx, Wseq, co, coef, po, plen, posts, present)
        b = _dev_calls(fresh, Wseq, co, coef, po, plen, posts, present)
        for k in a:
            assert_bits_equal(a[k], b[k], "after switching off: " + k)
        assert_bits_equal(res_hs, b["res_f32"], "decode_dsp res in half-rate vs full-rate mode")
        assert_bits_equal(ctx.synthesis(Wseq, co, coef, po, plen), fresh.synthesis(Wseq, co, coef, po, plen), "synthesis")
        assert_bits_equal(ctx.decode_dsp(Wseq, co, coef, posts, present, po, plen),
                          fresh.decode_dsp(Wseq, co, coef, posts, present, po, plen), "decode_dsp")
        for W in (0, 1):
            assert_bits_equal(ctx.mdct_backward(W, y[W]), fresh.mdct_backward(W, y[W]), "mdct_backward W%d" % W)
        Wg = dec["W"][None, :]
        co, po, _, plen = vlib.synthesis_layout(Wg, bs, ch)
        assert_bits_equal(ctx.synthesis(Wg, co, dec["coef"], po, plen)[0], dec["pcm"], "golden full-rate decode")
    finally:
        ctx.synthesis_halfrate(1, setup.halfrate_windows())
    fresh.close()


def test_halfrate_refused_for_64_sample_blocks(cuda_ok):
    """a decode-only context with blocksizes[0] = 64 gets VB200_EINVAL (the reference returns -1 there)"""
    ctx = vlib.Context(decode_only_setup(64))
    rc = ctx.L.vb200_synthesis_halfrate(ctx.h, 1, None)
    assert rc == -131, rc                                         # VB200_EINVAL
    ctx.synthesis_halfrate(0)
    ctx.close()
    # blocksizes[0] = 128: the 64- and 128-point transforms through the generic k_mdct_backward instance
    setup = decode_only_setup(128)
    ctx = vlib.Context(setup)
    ctx.synthesis_halfrate(1)
    o = halfrate.Oracle.create(setup)
    y = np.random.default_rng(3).uniform(-1, 1, (50, 32)).astype(np.float32)
    assert_bits_equal(ctx.mdct_backward(0, y), o.mdct_backward(0, y), "mdct_backward N=64")
    ctx.close()


@pytest.mark.parametrize("ch,rate,q", [(2, 44100, 0.5), (1, 44100, 0.4), (2, 44100, 0.1), (6, 48000, 0.2)])
def test_dropin_halfrate_decode_identical(cuda_ok, ch, rate, q):
    """Drop-in: the reference decoder with mdct_backward bound to the CUDA shim (vb200_ref_shim.c) decodes real
    encoded streams after vorbis_synthesis_halfrate(vi, 1); its PCM is bit-identical to the stock reference's
    half-rate PCM."""
    if not (halfrate.ref_available() and halfrate.ref_available(dropin=True)):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    pcm = probe_signal(ch, rate, 0.6, seed=5)
    packets = halfrate.ref_encode(ch, rate, q, pcm)
    setup = load_setup(FIXTURE_OF[(ch, rate, q)])
    bs = [setup.blocksize(0), setup.blocksize(1)]
    want = halfrate.ref_decode(packets, bs, ch, pcm.shape[1] + 8192)
    got = halfrate.ref_decode(packets, bs, ch, pcm.shape[1] + 8192, dropin=True)
    assert set(want["W"].tolist()) == {0, 1}
    assert want["pcm"].shape[1] > pcm.shape[1] // 2 - 4096
    assert np.array_equal(got["W"], want["W"])
    assert got["pcm"].shape == want["pcm"].shape
    assert np.array_equal(got["pcm"].view(np.uint32), want["pcm"].view(np.uint32))
    # the full-rate decode through the same shim is unchanged
    full = halfrate.ref_decode(packets, bs, ch, pcm.shape[1] + 8192, halfrate=False)
    got = halfrate.ref_decode(packets, bs, ch, pcm.shape[1] + 8192, halfrate=False, dropin=True)
    assert np.array_equal(got["pcm"].view(np.uint32), full["pcm"].view(np.uint32))
