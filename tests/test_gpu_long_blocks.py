"""Every device path on the 512/4096 block sizes that vorbisenc picks below q = 0 at 32-96 kHz and for low-rate
bitrate-managed encodes, and the generic-size transform instances (64, 128, 4096, 8192).  Bit-exact.

At these sizes the device runs code that the 256/2048 setups never launch: the generic `<0>` instances of
k_mdct_forward, k_mdct_backward and k_phaseA_transform (4096 and 8192 points, each thread striding over more
elements), the K = 16 instance of k_phaseA_psy3 (n = 2048), the generic k_phaseA_psy at n = 2048, and every buffer
that grows with n: the floor-1 fit's shared memory, twice the residue partitions, the half-rate decoder's <2048>
instances and a 106-step planner mark window.

- The stages against the oracle, which tests/test_oracle_vs_ref.py pins to the reference at (2, 44100, -0.1) and
  (6, 48000, -0.1) and tests/test_oracle_vs_ref.py::test_floor1_vs_reference at (2, 32000, -0.1).  Many checks run
  the bodies of the tests of tests/test_gpu_parity.py on these setups.  The blocks the reference encoder cut are
  stored with its results under tests/golden/ref.
- Packets and PCM against the stock encoder and decoder (needs oracle/_ref).
- The generic sizes against the oracle bit for bit and against float64 direct formulas
  (tests/test_transform_fp64.py)."""
import numpy as np
import pytest

import refgold as G
import test_gpu_dropin as DI
import test_gpu_encode_packets as EP
import test_gpu_halfrate as HR
import test_gpu_parity as P
import test_gpu_stream_packets as SP
import test_gpu_stream_resume as SR
import test_oracle_vs_ref as T
import test_transform_fp64 as F
from conftest import assert_bits_equal, make_desc, probe_signal
from oracle import bitrate as B
from oracle import decode, halfrate, pyref
from oracle import decode_packets as dp
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu

LONG = [(2, 32000, -0.1), (2, 44100, -0.1), (6, 48000, -0.1)]
CAPTURE = {(2, 32000, -0.1): ("floor1", T.floor1_signal), (2, 44100, -0.1): ("chain", T.chain_signal),
           (6, 48000, -0.1): ("chain", T.chain_signal)}
GENERIC = [(64, 8192), (128, 4096)]


def _encoder_blocks(args, o, capture=CAPTURE):
    """the blocks the reference encoder cut from its stream (tests/golden/ref), in the layout of the golden encode
    fixtures that the tests of test_gpu_parity.py read: <tag>_pcm, _W, _lW, _nW, _blocktype, _ampmax_in, and the
    reference's quantised residue and nonzero flags (the oracle's, checked against the reference's digest)"""
    group, signal = capture[args]
    rec = G.load("%s_%s" % (group, G.case_id(*args)))
    tl = G.timeline(rec, signal(*args))
    bs = o.bs
    enc = {}
    for W, tag in ((0, "S"), (1, "L")):
        idx = np.where(rec["W"] == W)[0]
        assert len(idx) >= 4, "the reference's stream has blocks of both sizes"
        enc[tag + "_pcm"] = G.blocks(rec, tl, bs, idx)
        for k in ("W", "lW", "nW", "blocktype", "ampmax_in", "nonzero_out"):
            enc["%s_%s" % (tag, k)] = rec[k][idx]
        want = o.encode_dsp(W, enc[tag + "_pcm"], G.desc(rec, idx))
        G.assert_digest(want["iwork"], rec["d_iwork_out_W%d" % W], "oracle residue W%d" % W)
        enc[tag + "_iwork_out"] = want["iwork"]
        enc[tag + "_enc_posts"] = rec["enc_posts"][idx]
        enc[tag + "_fit_posts"] = rec["fit_posts"][idx]
    enc["d_iwork_out"] = [rec["d_iwork_out_W0"], rec["d_iwork_out_W1"]]
    return enc


@pytest.fixture(scope="module", params=LONG, ids=lambda a: G.case_id(*a))
def cfg(request, oracle_lib, cuda_ok):
    """(name, setup, context, oracle, encoder blocks, None): the shape of test_gpu_parity.py's fixture"""
    args = request.param
    setup = G.load_setup(*args)
    assert [setup.blocksize(0), setup.blocksize(1)] == [512, 4096]
    assert [setup.psy_n(k) for k in range(4)] == [256, 256, 2048, 2048]
    o = oracle_lib.Oracle(setup)
    ctx = vlib.Context(setup)
    yield G.case_id(*args), setup, ctx, o, _encoder_blocks(args, o), None
    ctx.close()


# ---- stages against the oracle --------------------------------------------------------------------------------------
def test_tables(cfg):
    P.test_tables_match_oracle(cfg)


def _transform_inputs(rng, nvec, N):
    x = rng.uniform(-1, 1, (nvec, N)).astype(np.float32)
    y = rng.uniform(-1, 1, (nvec, N // 2)).astype(np.float32)
    if nvec > 4:
        for a in (x, y):
            a[0] = 0.0                                    # silence
            a[1] = 1.0                                    # full-scale DC
            a[2, ::2], a[2, 1::2] = 1.0, -1.0             # alternating +-1
            a[3] *= 1e-30                                 # products in the denormal range
            a[4] = 1e-40                                  # denormal input
    return x, y


def _check_transforms(ctx, o, W, nvec, seed):
    N = o.bs[W]
    rng = np.random.default_rng(seed)
    x, y = _transform_inputs(rng, nvec, N)
    what = "N=%d, %d vectors: " % (N, nvec)
    assert_bits_equal(ctx.mdct_forward(W, x), o.mdct_forward(W, x), what + "mdct_forward")
    assert_bits_equal(ctx.mdct_backward(W, y), o.mdct_backward(W, y), what + "mdct_backward")
    assert_bits_equal(ctx.drft_forward(W, x), o.drft_forward(W, x), what + "drft_forward")
    lW = rng.integers(0, 2, nvec).astype(np.int32)
    nW = rng.integers(0, 2, nvec).astype(np.int32)
    assert_bits_equal(ctx.apply_window(W, x, lW, nW), o.apply_window(W, x, lW, nW), what + "window")


@pytest.mark.parametrize("nvec", [1, 133, 4000])
@pytest.mark.parametrize("W", [0, 1])
def test_transforms_vs_oracle(cfg, W, nvec):
    """1 vector, fewer vectors than CTAs, and more vectors than resident CTAs (132 SMs x 8), so that every CTA walks
    several rows and stages the next one with cp.async"""
    name, setup, ctx, o, _, _ = cfg
    _check_transforms(ctx, o, W, nvec, 100 * W + nvec)


@pytest.mark.parametrize("look", [0, 1, 2, 3])
def test_psy_stages(cfg, look):
    P.test_psy_stages_vs_oracle_random(cfg, look)


@pytest.mark.parametrize("kernel", ["fast", "generic"])
@pytest.mark.parametrize("W", [0, 1])
def test_phaseA(cfg, W, kernel, monkeypatch):
    """the fused Phase A on the reference encoder's blocks, with taps and without (the debug and the plain instance of
    k_phaseA_psy3), random blocks and adversarial ones, through the fast psy kernel and the generic one"""
    name, setup, ctx, o, enc, _ = cfg
    if kernel == "generic":
        monkeypatch.setenv("VB200_PSY_V1", "1")
    tag = "L" if W else "S"
    desc = make_desc(enc, tag)
    a = ctx.phaseA(W, enc[tag + "_pcm"], desc, taps=True)
    b = o.phaseA(W, enc[tag + "_pcm"], desc, taps=True)
    for k in ("mdct_raw", "logfft", "noise", "tone", "logmdct", "logmask", "mdct", "ampmax_out"):
        assert_bits_equal(a[k], b[k], "phaseA " + k)
    a = ctx.phaseA(W, enc[tag + "_pcm"], desc)
    for k in ("mdct", "logmdct", "logmask", "ampmax_out"):
        assert_bits_equal(a[k], b[k], "phaseA without taps " + k)
    P.test_phaseA_vs_oracle_random(cfg, W)
    P.test_phaseA_adversarial_inputs(cfg, W)


def test_phaseA_host_multichunk_and_streams(cfg, monkeypatch):
    P.test_phaseA_stream_mode_device(cfg)
    for fmt in ("f32", "s16"):
        P.test_phaseA_pcm_ingest_from_stream_buffers(cfg, fmt)
    P.test_phaseA_host_path_multichunk(cfg, monkeypatch)


@pytest.mark.parametrize("W", [0, 1])
def test_floor1(cfg, W):
    """floor1_fit / floor1_render on the oracle's masks of random PCM and on synthetic corner-case curves, and on the
    reference encoder's own blocks through the one-call chain (posts against the reference's floor1_encode)"""
    P.test_floor1_vs_oracle_random(cfg, W)
    name, setup, ctx, o, enc, _ = cfg
    tag = "L" if W else "S"
    got = ctx.encode_dsp(W, enc[tag + "_pcm"], make_desc(enc, tag))
    G.assert_digest(got["iwork"], enc["d_iwork_out"][W], "residue vs reference")
    assert np.array_equal(got["nonzero"], enc[tag + "_nonzero_out"]), "nonzero vs reference"
    ep = enc[tag + "_enc_posts"].astype(np.int32).copy()
    ep[enc[tag + "_fit_posts"][..., 0] == -1] = 0
    assert np.array_equal(got["posts"], ep), "posts vs reference (floor1_encode)"


@pytest.mark.parametrize("W", [0, 1])
def test_couple_quantize_normalize(cfg, W):
    """k_cqn_fast for one and two channels, k_cqn for six"""
    P.test_couple_quantize_normalize_vs_oracle_random(cfg, W)


@pytest.mark.parametrize("W", [0, 1])
def test_residue_and_inverse_floor(cfg, W):
    P.test_residue_classify_vs_oracle(cfg, W)
    P.test_floor1_inverse2_vs_oracle(cfg, W)


def test_synthesis_and_decode(cfg):
    """decouple, synthesis in float and int16, the one-call decode in float and int16, and an encode-decode trip"""
    P.test_decouple_vs_oracle(cfg)
    P.test_decode_vs_oracle_random_streams(cfg)
    P.test_decode_int16_egress(cfg)
    for s16 in (False, True):
        P.test_decode_dsp_one_call_vs_oracle(cfg, s16)
    P.test_encode_then_decode_round_trip(cfg)


@pytest.mark.parametrize("fmt", ["blocks", "f32", "s16"])
@pytest.mark.parametrize("W", [0, 1])
def test_encode_dsp_streams(cfg, W, fmt, monkeypatch):
    P.test_encode_dsp_streams_vs_oracle(cfg, W, fmt, monkeypatch)


def test_encode_dsp_pipeline_forms(cfg, monkeypatch):
    """the many-chunk host pipeline, device pointers and their errors, two concurrent half batches, int16 residue and
    partition classes"""
    for ramp in ("1", "0"):
        P.test_encode_dsp_many_chunks(cfg, ramp, monkeypatch)
    P.test_encode_dsp_device_pointers_and_errors(cfg)
    P.test_encode_dsp_dev_split_half_batches(cfg, monkeypatch)
    for W in (0, 1):
        P.test_encode_dsp_int16_residue(cfg, W, monkeypatch)
    P.test_encode_dsp_with_classes(cfg, monkeypatch)


@pytest.mark.parametrize("fmt", ["s16", "blocks"])
@pytest.mark.parametrize("W", [0, 1])
def test_encode_dsp_managed(cfg, W, fmt):
    P.test_encode_dsp_managed_vs_oracle(cfg, W, fmt)


def test_envelope_and_plan(cfg):
    for fmt in ("f32", "s16"):
        P.test_envelope_search_streams_vs_oracle(cfg, fmt)
    P.test_plan_blocks_device_vs_oracle(cfg)


@pytest.mark.parametrize("args", [(2, 44100, -0.1), (6, 48000, -0.1)], ids=lambda a: G.case_id(*a))
def test_envelope_search_vs_reference(cuda_ok, args):
    """the device's envelope search on the reference's own stream buffer gives the reference's marks and filter state
    (stored by tests/golden/make_golden_ref.py)"""
    ctx = vlib.Context(G.load_setup(*args))
    rec = G.load("envelope_" + G.case_id(*args))
    stream = np.concatenate([rec["stream_pre"], T.envelope_signal(*args)], axis=1)
    steps = int(rec["steps"])
    ret, state = ctx.envelope_search(stream[None], 0, steps)
    assert np.array_equal(ctx.envelope_marks(ret[0])[:steps + 2], rec["marks"])
    assert np.array_equal(state[0], rec["state"])
    ctx.close()


@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_encode_streams_mixed_block_sizes(cfg, fmt):
    """vb200_encode_streams on streams that switch block sizes: plan, posts, nonzero and residue of every block equal
    the oracle's composition (envelope search, planner with its 4096-sample mark window, ampmax chain)"""
    name, setup, ctx, o, _, _ = cfg
    ch, half = setup.channels, setup.blocksize(1) // 2
    sig = P.streams_signals(ch, setup.rate, None)
    stride = (max(s.shape[1] for s in sig) + 4 * half + 3) & ~3
    tl = np.zeros((len(sig), ch, stride), np.float32)
    for i, s in enumerate(sig):
        tl[i, :, half:half + s.shape[1]] = s
    pcm_len = np.array([half + s.shape[1] + 2 * half for s in sig], np.int64)
    eof = np.array([half + s.shape[1] for s in sig], np.int64)
    if fmt == "f32":
        got = ctx.encode_streams(tl, pcm_len, eof)
    else:
        s16 = np.clip(np.rint(tl * 32767.0), -32768, 32767).astype(np.int16)
        tl = s16.astype(np.float32) / np.float32(32768.0)
        got = ctx.encode_streams(np.ascontiguousarray(s16.transpose(0, 2, 1)), pcm_len, eof, fmt=vlib.PCM_S16_INTERLEAVED)
    nshort = 0
    for i in range(len(sig)):
        wplan, wouts = o.encode_stream(tl[i], int(pcm_len[i]), int(eof[i]))
        k = len(wplan)
        assert got["nblocks"][i] == k, "stream %d: %d blocks, want %d" % (i, got["nblocks"][i], k)
        plan = got["plan"][i, :k]
        for nm in ("pos", "W", "lW", "nW", "blocktype"):
            assert np.array_equal(plan[nm], wplan[nm]), "stream %d %s" % (i, nm)
        for b in range(k):
            W, slot = int(plan[b]["W"]), int(plan[b]["slot"])
            nshort += W == 0
            g, w = got[W], wouts[b]
            assert np.array_equal(g["posts"][slot], w["posts"][0]), "stream %d block %d posts" % (i, b)
            assert np.array_equal(g["nonzero"][slot], w["nonzero"][0]), "stream %d block %d nonzero" % (i, b)
            assert np.array_equal(g["iwork"][slot], w["iwork"][0]), "stream %d block %d residue" % (i, b)
    assert nshort >= 10 and got["count"][0] == nshort          # the streams really mix the two sizes


@pytest.fixture(scope="module")
def halfrate_cfg(cfg):
    """the same setups decoding at half rate (closed-form windows of 256 and 2048 samples)"""
    name, setup, _, _, enc, _ = cfg
    ctx = vlib.Context(setup)
    ctx.synthesis_halfrate(1)
    yield name, setup, ctx, halfrate.Oracle.create(setup), enc, None
    ctx.close()


def test_halfrate(halfrate_cfg):
    """half-rate synthesis and decode (the long block's half takes the <2048> instances) and mdct_backward"""
    HR.test_random_streams_halfrate(halfrate_cfg)
    HR.test_long_stream_in_overlapping_segments(halfrate_cfg)
    HR.test_mdct_backward_halfrate(halfrate_cfg)


# ---- against the stock encoder and decoder (oracle/_ref) ------------------------------------------------------------
STOCK = [(2, 44100, -0.1), (1, 44100, -0.1), (6, 48000, -0.1)]


def _stock_bs(ch, rate, q):
    """the block sizes of the stock encoder's setup; the device coder must be taken at them"""
    d = EP._driver(ch, rate, q)                        # skips without oracle/_ref; asserts Driver.on_device
    bs = list(d.ctx.bs)
    d.close()
    assert bs == [512, 4096], "vorbisenc chose %s at (%d, %d, %g)" % (bs, ch, rate, q)


@pytest.mark.parametrize("ch,rate,q", STOCK)
def test_stock_encoder_packets(cuda_ok, ch, rate, q):
    """the stock encoder's captured blocks give its audio packets through encode_dsp + encode_entropy and through
    encode_packets; whole streams give its packets, granulepos, e_o_s and packetno, in one call and cut into pieces"""
    _stock_bs(ch, rate, q)
    EP.test_stage_parity_captured_blocks(cuda_ok, ch, rate, q)
    SP.test_unmanaged_whole_streams(cuda_ok, ch, rate, q)
    SR.test_fresh_carry_one_call_equals_packets_call(cuda_ok, ch, rate, q)


def test_stock_encoder_streams_in_pieces(cuda_ok):
    _stock_bs(2, 44100, -0.1)
    SR.test_cuts_equal_one_call_unmanaged(cuda_ok, 2, 44100, -0.1)


def test_entropy_coder_fuzz(cuda_ok):
    EP.test_fuzz_against_reference_functions(cuda_ok, 2, 44100, -0.1)


MANAGED = [("abr48", 2, 44100, -1, 48000, -1, None), ("mono32", 1, 44100, -1, 32000, -1, None)]


@pytest.mark.parametrize("name,ch,rate,max_br,nominal,min_br,rm2", MANAGED)
def test_stock_managed_encoder(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2):
    """low-rate ABR, where vorbis_encode_setup_managed picks 512/4096: whole streams, in one call and in pieces"""
    SP._need_ref()
    if not B.ref_available(True):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    d = B.ManagedDriver(ch, rate, max_br, nominal, min_br)
    bs = list(d.ctx.bs)
    d.close()
    assert bs == [512, 4096], "vorbisenc chose %s for %s" % (bs, name)
    SP.test_managed_whole_streams(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2)
    SR.test_cuts_equal_one_call_managed(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2)


@pytest.fixture
def driver():
    made = []

    def make(p):
        d = dp.Driver(p)
        made.append(d)
        return d
    yield make
    for d in made:
        d.close()


@pytest.mark.parametrize("ch,rate,q", STOCK)
def test_stock_decoder(cuda_ok, driver, ch, rate, q):
    """device decode of the stock encoder's packets: the entropy decode's staging equals the reference's, the fused
    resume decode equals entropy decode + DSP (full and half rate, float and int16), and the vb200md driver gives the
    stock decoder's PCM on its device and host paths"""
    import test_gpu_decode_packets as DP
    if not (decode.available() and dp.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    DP.test_stage_parity(cuda_ok, driver, ch, rate, q)
    DP.test_fused_equals_entropy_then_dsp(cuda_ok, driver, ch, rate, q, "two")
    for s16 in (False, True):
        DP.test_driver_device_and_host_paths_equal_stock(cuda_ok, ch, rate, q, s16)


@pytest.mark.parametrize("ch,rate,q", STOCK)
def test_stock_halfrate_decoder(cuda_ok, ch, rate, q):
    """the reference decoder with mdct_backward on the device, at half rate and at full rate, gives the stock PCM"""
    if not (halfrate.ref_available() and halfrate.ref_available(dropin=True)):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    pcm = probe_signal(ch, rate, 0.6, seed=5)
    packets = halfrate.ref_encode(ch, rate, q, pcm)
    for half in (True, False):
        want = halfrate.ref_decode(packets, [512, 4096], ch, pcm.shape[1] + 8192, halfrate=half)
        got = halfrate.ref_decode(packets, [512, 4096], ch, pcm.shape[1] + 8192, halfrate=half, dropin=True)
        assert set(want["W"].tolist()) == {0, 1}
        assert np.array_equal(got["W"], want["W"]) and got["pcm"].shape == want["pcm"].shape
        assert np.array_equal(got["pcm"].view(np.uint32), want["pcm"].view(np.uint32)), "half rate %s" % half


@pytest.mark.parametrize("ch,rate,q", [(2, 44100, -0.1), (6, 48000, -0.1)])
def test_function_level_dropin(cuda_ok, ch, rate, q):
    """the reference's encoder and decoder with their hot callees bound to the device: byte-identical packets and
    bit-identical PCM"""
    if pyref.available():
        r = pyref.Ref(ch, rate, q)
        assert list(r.bs) == [512, 4096]
        r.close()
    DI.test_encoder_packets_identical(cuda_ok, ch, rate, q)


# ---- the generic sizes ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=GENERIC, ids=lambda b: "%d_%d" % b)
def gen_cfg(request, oracle_lib, cuda_ok):
    setup = F._decode_only_setup(*request.param)
    ctx = vlib.Context(setup)
    yield "%d_%d" % request.param, setup, ctx, oracle_lib.Oracle(setup), None, None
    ctx.close()


@pytest.mark.parametrize("nvec", [1, 133, 2500])
@pytest.mark.parametrize("W", [0, 1])
def test_generic_size_transforms(gen_cfg, W, nvec):
    name, setup, ctx, o, _, _ = gen_cfg
    _check_transforms(ctx, o, W, nvec, 7 * W + nvec)


def test_generic_size_transforms_vs_fp64(gen_cfg, oracle_lib):
    """the device's MDCT (both directions) and real FFT against the float64 direct formulas, with the bound that
    tests/test_transform_fp64.py calibrates at N = 2048"""
    name, setup, ctx, o, _, _ = gen_cfg
    bound = F._bounds(oracle_lib)
    for W in (0, 1):
        N = setup.blocksize(W)
        errs = F._errors(ctx, N, *F._inputs(N), W)
        for what, e, b in zip(("mdct_forward", "mdct_backward", "drft_forward"), errs, bound(N)):
            assert e <= b, "%s N=%d: relative error %.3g over the bound %.3g" % (what, N, e, b)


def test_generic_size_synthesis(gen_cfg):
    P.test_decode_vs_oracle_random_streams(gen_cfg)
    P.test_decode_int16_egress(gen_cfg)


def test_generic_size_halfrate(cuda_ok):
    """(128, 4096) at half rate: the 64- and 2048-point inverse transforms and the overlap-add"""
    setup = F._decode_only_setup(128, 4096)
    ctx = vlib.Context(setup)
    ctx.synthesis_halfrate(1)
    o = halfrate.Oracle.create(setup)
    rng = np.random.default_rng(12)
    for W in (0, 1):
        y = rng.uniform(-1, 1, (300, setup.blocksize(W) // 4)).astype(np.float32)
        assert_bits_equal(ctx.mdct_backward(W, y), o.mdct_backward(W, y), "half-rate mdct_backward W%d" % W)
    Wseq = rng.integers(0, 2, (9, 17)).astype(np.int32)
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, ctx.bs, setup.channels, halfrate=True)
    coef = (rng.uniform(-1, 1, coef_len) * 0.05).astype(np.float32)
    assert_bits_equal(ctx.synthesis(Wseq, coef_off, coef, pcm_off, pcm_len),
                      o.synthesis(Wseq, coef_off, coef, pcm_off, pcm_len), "half-rate synthesis")
    ctx.close()
