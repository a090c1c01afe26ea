"""CPU oracle (our restatement) against the compiled reference itself on fresh signals, for a grid
of (channels, rate, quality): every stage, the fused Phase-A chain recorded from the real
mapping0_forward, Phase B, the ampmax chain and the decoded PCM.  Bit-exact.
What the reference computed for these signals is stored under tests/golden/ref (tests/refgold.py;
regenerate with tests/golden/make_golden_ref.py where the reference can be compiled)."""
import numpy as np
import pytest

import refgold as G
from conftest import assert_bits_equal, probe_signal
from vorbis_b200 import abi, lib as vlib

# the setups vorbisenc picks above q = 0.5: full-band residue with the _residue_44_high / _hi_un / _44p_hi books,
# uncoupled 5.1 (no coupling steps, two submaps), 96 kHz and coupled 22.05 kHz stereo (tests/test_gpu_high_quality.py)
HIGH = [(2, 44100, 0.6), (2, 44100, 1.0), (1, 44100, 0.9), (6, 48000, 0.5), (6, 48000, 0.9), (2, 96000, 0.7),
        (2, 22050, 0.9)]
HIGH_NEW = [a for a in HIGH if a != (2, 96000, 0.7)]          # the lists that already hold (2, 96000, 0.7)
GRID = [(2, 44100, 0.5), (1, 44100, 0.4), (2, 44100, 0.1), (2, 44100, 0.3), (1, 44100, 0.2),
        (2, 48000, 0.9), (2, 32000, 0.0), (1, 22050, 0.3), (2, 44100, -0.1), (6, 48000, -0.1)] + HIGH
FLOOR1_ARGS = [(2, 44100, 0.5), (6, 48000, 0.2), (2, 32000, -0.1), (1, 16000, 0.5), (2, 96000, 0.7)] + HIGH_NEW
CHAIN_ARGS = [(2, 44100, 0.5), (2, 44100, 0.1), (1, 44100, 0.4), (6, 48000, 0.2),
              (2, 44100, -0.1), (6, 48000, -0.1), (2, 96000, -0.1)] + HIGH
MANAGED_ARGS = [(2, 44100, 0.5), (1, 44100, 0.4), (6, 48000, 0.2),
                (2, 44100, -0.1), (6, 48000, -0.1), (2, 96000, -0.1)] + HIGH
ENVELOPE_ARGS = [(2, 44100, 0.5), (1, 44100, 0.4), (6, 48000, 0.2), (1, 22050, 0.3), (2, 32000, 0.0), (2, 96000, 0.7),
                 (2, 44100, -0.1), (6, 48000, -0.1), (2, 96000, -0.1)] + HIGH_NEW
INVERSE2_ARGS = [(2, 44100, 0.5), (6, 48000, 0.2), (1, 22050, 0.3),
                 (2, 44100, -0.1), (6, 48000, -0.1), (2, 96000, -0.1)] + HIGH
RESIDUE_ARGS = [(2, 44100, 0.5), (1, 44100, 0.4), (6, 48000, 0.2), (1, 22050, 0.3), (2, 44100, 0.1),
                (2, 44100, -0.1), (6, 48000, -0.1), (2, 96000, -0.1)] + HIGH
IDS = lambda g: G.case_id(*g)  # noqa: E731


# ---- the signals and random inputs (tests/golden/make_golden_ref.py runs the reference on the same ones)
def pair_signal(ch, rate):
    pcm = probe_signal(ch, rate, 1.2, seed=11)
    if ch == 2:
        pcm[1] = (0.7 * pcm[0] + 0.3 * pcm[1]).astype(np.float32)
    return pcm


def floor1_signal(ch, rate, q):
    pcm = probe_signal(ch, rate, 1.0, seed=5)
    pcm[:, :3000] = 0
    return pcm


def chain_signal(ch, rate, q):
    pcm = probe_signal(ch, rate, 1.0, seed=9)
    pcm[:, 5000:9000] = 0
    return pcm


def managed_signal(ch, rate, q):
    pcm = probe_signal(ch, rate, 0.6, seed=21)
    pcm[:, 5000:9000] = 0
    return pcm


def envelope_signal(ch, rate, q):
    rng = np.random.default_rng(3)
    pcm = probe_signal(ch, rate, 44100 / rate, seed=5)[:, :44100].copy()
    pcm[:, 8000:12000] *= 0.001
    pcm[:, 20000:20300] = rng.uniform(-.9, .9, (ch, 300))
    pcm[:, 30000:33000] = 0
    return pcm


def transform_inputs(N, rng=None):
    rng = rng or np.random.default_rng(7)
    x = rng.uniform(-1, 1, (16, N)).astype(np.float32)
    y = rng.uniform(-1, 1, (16, N // 2)).astype(np.float32)
    lW = rng.integers(0, 2, 16).astype(np.int32)
    nW = rng.integers(0, 2, 16).astype(np.int32)
    return x, y, lW, nW


def inverse2_inputs(ch, bs):
    rng = np.random.default_rng(4)
    for W in (0, 1):
        n, rows = bs[W] // 2, ch * 7
        posts = rng.integers(0, 140, (rows, abi.FLOOR1_STRIDE)).astype(np.int32)
        flag = rng.random(posts.shape) < 0.4
        flag[:, :2] = False
        posts[flag] |= 0x8000
        posts[3, 5] = 400
        posts[4, 0] = 999
        present = (rng.random(rows) < 0.85).astype(np.int32)
        data = (rng.standard_normal((rows, n)) * 5).astype(np.float32)
        yield W, (posts, present, data)


def residue_inputs(ch, bs):
    rng = np.random.default_rng(13)
    for W in (0, 1):
        n, nb = bs[W] // 2, 6
        mag = np.exp(rng.uniform(-2, 3, (nb, ch, 1))) * np.exp(-np.arange(n) / (n / 4.0))[None, None, :]
        iwork = np.rint(rng.standard_normal((nb, ch, n)) * mag).astype(np.int32)
        nonzero = (rng.random((nb, ch)) < 0.8).astype(np.int32)
        nonzero[1] = 0
        yield W, (iwork, nonzero)


def _bs(setup):
    return [setup.blocksize(0), setup.blocksize(1)]


def _ref_batch(args, name, W, blocks, desc):
    """bench.py's CPU arm runs the reference driver's batched helpers (oracle/ref_driver.c): where oracle/_ref is
    built they are run too and must give the stored results"""
    from oracle import pyref
    return getattr(pyref.Ref(*args), name)(W, blocks, desc) if pyref.available() else None


def _phaseA(o, rec, tl, bs, W, idx, taps=False):
    """the oracle's Phase A on the blocks idx (one size) the reference's API loop cut from its stream"""
    return o.phaseA(W, G.blocks(rec, tl, bs, idx), G.desc(rec, idx), taps=taps)


@pytest.fixture(scope="module", params=GRID, ids=IDS)
def pair(request, oracle_lib):
    ch, rate, q = request.param
    setup = G.load_setup(ch, rate, q)
    o = oracle_lib.Oracle(setup)
    pcm = pair_signal(ch, rate)
    rec = G.load("pair_" + G.case_id(ch, rate, q))
    rec["args"] = request.param
    return rec, setup, o, G.timeline(rec, pcm), pcm


def test_tables(pair):
    rec, setup, o, tl, _ = pair
    for W in (0, 1):
        for which in (0, 1, 2, 3):
            G.assert_digest(o.table(W, which), rec["d_table_W%d_%d" % (W, which)], "table W%d #%d" % (W, which))


def test_transforms_random(pair):
    rec, setup, o, tl, _ = pair
    rng = np.random.default_rng(7)
    for W in (0, 1):
        x, y, lW, nW = transform_inputs(setup.blocksize(W), rng)
        G.assert_digest(o.mdct_forward(W, x), rec["d_mdct_forward_W%d" % W], "mdct_forward")
        G.assert_digest(o.mdct_backward(W, y), rec["d_mdct_backward_W%d" % W], "mdct_backward")
        G.assert_digest(o.drft_forward(W, x), rec["d_drft_forward_W%d" % W], "drft_forward")
        G.assert_digest(o.apply_window(W, x, lW, nW), rec["d_window_W%d" % W], "window")


def test_phaseA_chain_of_the_real_encoder(pair):
    rec, setup, o, tl, _ = pair
    bs = _bs(setup)
    for W in (0, 1):
        idx = np.where(rec["W"] == W)[0]
        if not len(idx):
            continue
        out = _phaseA(o, rec, tl, bs, W, idx, taps=True)
        for k, g in (("mdct_raw", "mdct_raw"), ("logfft", "logfft"), ("noise", "noise"), ("tone", "tone"),
                     ("logmdct", "logmdct"), ("logmask", "logmask"), ("mdct", "mdct_m1")):
            G.assert_digest(out[k], rec["d_%s_W%d" % (g, W)], "W%d %s" % (W, k))
        assert_bits_equal(out["ampmax_out"], rec["ampmax_out"][idx], "ampmax_out")
        # the driver's batched reference helper (used by bench.py's CPU legs) agrees too
        G.assert_digest(out["logmask"], rec["d_batch_logmask_W%d" % W], "ref_phaseA_batch logmask")
        G.assert_digest(out["mdct"], rec["d_batch_mdct_W%d" % W], "ref_phaseA_batch mdct")
        b = _ref_batch(rec["args"], "phaseA_batch", W, G.blocks(rec, tl, bs, idx), G.desc(rec, idx))
        if b is not None:
            G.assert_digest(b[2], rec["d_batch_logmask_W%d" % W], "ref_phaseA_batch logmask (run)")
            G.assert_digest(b[0], rec["d_batch_mdct_W%d" % W], "ref_phaseA_batch mdct (run)")


def test_phaseB_of_the_real_encoder(pair):
    rec, setup, o, tl, _ = pair
    bs = _bs(setup)
    for W in (0, 1):
        idx = np.where(rec["W"] == W)[0]
        if not len(idx):
            continue
        n = bs[W] // 2
        # the reference's Phase-B inputs of these blocks, recomputed and pinned to its own by digest
        a = _phaseA(o, rec, tl, bs, W, idx)
        G.assert_digest(a["mdct"], rec["d_mdct_m1_W%d" % W], "mdct_m1 input")
        posts, nz = o.floor1_fit(W, a["logmdct"], a["logmask"])
        _, ilog, _ = o.floor1_render(W, posts, nz)
        ilog = ilog.reshape(len(idx), -1, n)
        G.assert_digest(ilog, rec["d_ilogmask_W%d" % W], "ilogmask input")
        for bt in (0, 1):
            sel = np.where(rec["blocktype"][idx] == bt)[0]
            if not len(sel):
                continue
            iw, nzo = o.couple_quantize_normalize(W, bt, 7, a["mdct"][sel], ilog[sel], rec["nonzero_in"][idx[sel]])
            G.assert_digest(iw, rec["d_iwork_out_W%d_bt%d" % (W, bt)], "iwork")
            assert np.array_equal(nzo, rec["nonzero_out"][idx[sel]])


def test_decode_of_the_real_stream(pair):
    rec, setup, o, tl, pcm = pair
    Wseq = rec["dec_W"][None, :]
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, _bs(setup), setup.channels)
    out = o.synthesis(Wseq, coef_off, rec["dec_coef"], pcm_off, pcm_len)
    m = int(rec["dec_m"])
    assert m > 0
    G.assert_digest(out[0][:, :m], rec["d_dec_pcm"], "decoded pcm")


def _capture(kind, args, pcm, oracle_lib):
    setup = G.load_setup(*args)
    rec = G.load("%s_%s" % (kind, G.case_id(*args)))
    return rec, setup, oracle_lib.Oracle(setup), G.timeline(rec, pcm)


@pytest.mark.parametrize("args", FLOOR1_ARGS, ids=IDS)
def test_floor1_vs_reference(args, oracle_lib):
    """floor1_fit / floor1_encode recorded inside the reference's own mapping0_forward, incl. silent
    blocks (NULL fit) and the 5.1 LFE submap with its own 2-post floor."""
    rec, setup, o, tl = _capture("floor1", args, floor1_signal(*args), oracle_lib)
    bs = _bs(setup)
    nulls = 0
    for W in (0, 1):
        idx = np.where(rec["W"] == W)[0]
        if not len(idx):
            continue
        n = bs[W] // 2
        a = _phaseA(o, rec, tl, bs, W, idx)
        G.assert_digest(a["logmdct"], rec["d_logmdct_W%d" % W], "logmdct input")
        G.assert_digest(a["logmask"], rec["d_logmask_W%d" % W], "logmask input")
        posts, nz = o.floor1_fit(W, a["logmdct"], a["logmask"])
        want = rec["fit_posts"][idx].reshape(-1, abi.FLOOR1_STRIDE).copy()
        wnz = (want[:, 0] != -1).astype(np.int32)
        want[wnz == 0] = 0
        nulls += int((wnz == 0).sum())
        assert np.array_equal(nz, wnz)
        assert np.array_equal(posts, want)
        p2, ilog, nz2 = o.floor1_render(W, posts, nz)
        wenc = rec["enc_posts"][idx].reshape(-1, abi.FLOOR1_STRIDE)
        assert np.array_equal(p2[wnz == 1], wenc[wnz == 1])
        G.assert_digest(ilog.reshape(len(idx), -1, n), rec["d_ilogmask_W%d" % W], "ilogmask")
        assert np.array_equal(nz2, rec["nonzero_in"][idx].reshape(-1))
    assert nulls > 0


@pytest.mark.parametrize("args", CHAIN_ARGS, ids=IDS)
def test_encode_chain_vs_reference(args, oracle_lib):
    """the composed oracle chain (what vb200_encode_dsp is checked against) equals the reference's own
    functions called in mapping0_forward's order (ref_encode_dsp_batch, also bench.py's CPU arm), on the
    PCM blocks, block flags and ampmax the reference's own API loop handed to mapping0_forward"""
    rec, setup, o, tl = _capture("chain", args, chain_signal(*args), oracle_lib)
    bs = _bs(setup)
    for W in (0, 1):
        idx = np.where(rec["W"] == W)[0]
        if not len(idx):
            continue
        blocks, desc = G.blocks(rec, tl, bs, idx), G.desc(rec, idx)
        a = o.encode_dsp(W, blocks, desc)
        for x in filter(None, (a, _ref_batch(args, "encode_dsp_batch", W, blocks, desc))):
            for k in ("posts", "nonzero", "iwork"):
                G.assert_digest(x[k], rec["d_batch_%s_W%d" % (k, W)], k)
            assert_bits_equal(x["ampmax_out"], rec["batch_ampmax_out_W%d" % W], "ampmax_out")
        G.assert_digest(a["iwork"], rec["d_iwork_out_W%d" % W], "iwork vs the API loop's capture")


@pytest.mark.parametrize("args", MANAGED_ARGS, ids=IDS)
def test_managed_chain_vs_reference(args, oracle_lib):
    """bitrate-managed mode: the composed oracle (three masks, three fits, twelve interpolated curves, render +
    couple/quantise per curve; what vb200_encode_dsp_managed is checked against) equals the reference's own
    functions called in mapping0_forward's managed order (lib/mapping0.c:500-573, 596-646), incl. silent blocks
    (NULL curves) and both block sizes"""
    rec, setup, o, tl = _capture("managed", args, managed_signal(*args), oracle_lib)
    bs = _bs(setup)
    nulls = 0
    for W in (0, 1):
        idx = np.where(rec["W"] == W)[0][:10]
        if not len(idx):
            continue
        blocks, desc = G.blocks(rec, tl, bs, idx), G.desc(rec, idx)
        a = o.encode_dsp_managed(W, blocks, desc)
        for x in filter(None, (a, _ref_batch(args, "encode_dsp_managed_batch", W, blocks, desc))):
            for k in ("posts", "nonzero", "iwork"):
                G.assert_digest(x[k], rec["d_managed_%s_W%d" % (k, W)], "%s W%d" % (k, W))
            assert_bits_equal(x["ampmax_out"], rec["managed_ampmax_out_W%d" % W], "ampmax_out")
        mid = abi.PACKETBLOBS // 2
        assert np.array_equal(a["iwork"][mid], o.encode_dsp(W, blocks, desc)["iwork"]), "curve 7 is the un-managed chain"
        assert not np.array_equal(a["iwork"][0], a["iwork"][abi.PACKETBLOBS - 1]), "low and high rate curves differ"
        nulls += int((a["posts"].reshape(abi.PACKETBLOBS, -1, abi.FLOOR1_STRIDE)[:, :, :2] == 0).all(axis=2).sum())
    assert nulls > 0, "the probe holds silent blocks"


@pytest.mark.parametrize("args", ENVELOPE_ARGS, ids=IDS)
def test_envelope_vs_reference(args, oracle_lib):
    """the reference's own _ve_envelope_search on a fresh dsp state vs the restatement: marks, filter
    states and stretch bit-identical (the stream buffer, incl. the pre-extrapolated preamble, is taken
    from the reference)"""
    o = oracle_lib.Oracle(G.load_setup(*args))
    rec = G.load("envelope_" + G.case_id(*args))
    stream = np.concatenate([rec["stream_pre"], envelope_signal(*args)], axis=1)
    steps = int(rec["steps"])
    ret, state = o.envelope_search(stream[None], 0, steps)
    assert np.array_equal(o.envelope_marks(ret[0])[:steps + 2], rec["marks"])
    assert np.array_equal(state[0], rec["state"])
    assert rec["marks"].sum() > 0


@pytest.mark.parametrize("args", INVERSE2_ARGS, ids=IDS)
def test_floor1_inverse2_vs_reference(args, oracle_lib):
    """decode-side floor: the reference's own floor1_inverse2 (through floor1_exportbundle) vs the
    restatement, on random fit_value[] incl. unused posts (bit 15), out-of-range values (clamped,
    lib/floor1.c:1056-1064) and absent floors (row zeroed)"""
    setup = G.load_setup(*args)
    o = oracle_lib.Oracle(setup)
    rec = G.load("inverse2_" + G.case_id(*args))
    for W, (posts, present, data) in inverse2_inputs(args[0], _bs(setup)):
        G.assert_digest(o.floor1_inverse2(W, posts, present, data), rec["d_inverse2_W%d" % W],
                        "floor1_inverse2 W=%d" % W)


@pytest.mark.parametrize("args", RESIDUE_ARGS, ids=IDS)
def test_residue_classify_vs_reference(args, oracle_lib):
    """res1_class / res2_class through the reference's own _residue_P[] (per submap, as mapping0_forward
    calls them) vs the restatement; residue types 1 and 2, the 5.1 setup's two submaps and 30-sample
    partitions, silent channels and silent bundles"""
    setup = G.load_setup(*args)
    o = oracle_lib.Oracle(setup)
    rec = G.load("residue_" + G.case_id(*args))
    for W, (iwork, nonzero) in residue_inputs(args[0], _bs(setup)):
        assert o.residue_partvals(W) > 0
        a = o.residue_classify(W, iwork, nonzero)
        G.assert_digest(a, rec["d_classes_W%d" % W], "classes W=%d" % W)
        assert a.max() > 0 and not a[1].any()
