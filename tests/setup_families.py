"""The device-path suite for families of vorbisenc setups whose structure the default setups never show the device.
Bit-exact.

Every test here is written once and collected by one module per family, which defines FAMILY, a Family row, and
takes the suite with `from setup_families import *` (pytest does not collect this module itself, since its name does
not start with test_):
- tests/test_gpu_long_blocks.py: the 512/4096 block sizes vorbisenc picks below q = 0, and the generic sizes;
- tests/test_gpu_multichannel.py: the uncoupled setups for 3, 4, 5, 8 and more channels;
- tests/test_gpu_high_quality.py: the setups above q = 0.5.
A family module adds its structural check, its content and its limits.  pytest_generate_tests parametrizes each
test from the module's FAMILY.

- The stages against the oracle, which tests/test_oracle_vs_ref.py pins to the reference at these setups, fed the
  blocks the reference encoder cut from its stream (tests/golden/ref).  The checks run the bodies of the tests of
  tests/test_gpu_parity.py on these setups.
- Packets and PCM against the stock encoder and decoder (needs oracle/_ref), on the rows each family gives.
- The generic transform sizes against the oracle bit for bit and against float64 direct formulas
  (tests/test_transform_fp64.py)."""
import collections

import numpy as np
import pytest

import refgold as G
import test_gpu_decode_packets as DP
import test_gpu_decode_ranges as DR
import test_gpu_decode_streams as DS
import test_gpu_dropin as DI
import test_gpu_encode_packets as EP
import test_gpu_halfrate as HR
import test_gpu_parity as P
import test_gpu_pcm_packets as PC
import test_gpu_stream_packets as SP
import test_gpu_stream_resume as SR
import test_oracle_vs_ref as T
import test_transform_fp64 as F
from conftest import assert_bits_equal, make_desc, probe_signal
from oracle import bitrate as B
from oracle import decode, halfrate, pyref
from oracle import decode_packets as dp
from test_gpu_decode_streams import drivers
from vorbis_b200 import lib as vlib

# what every family module collects; the family-specific tests further down are imported by name
__all__ = ["pytest_generate_tests", "cfg", "halfrate_cfg", "driver", "drivers", "family", "vector_counts", "formats",
           "envelope_setups", "test_tables", "test_transforms_vs_oracle", "test_psy_stages", "test_phaseA",
           "test_phaseA_host_multichunk_and_streams", "test_floor1", "test_couple_quantize_normalize",
           "test_residue_and_inverse_floor", "test_synthesis_and_decode", "test_encode_dsp_streams",
           "test_encode_dsp_pipeline_forms", "test_encode_dsp_managed", "test_envelope_and_plan",
           "test_envelope_search_vs_reference", "test_encode_streams_mixed_block_sizes", "test_halfrate",
           "test_stock_encoder_packets", "test_stock_managed_encoder", "test_stock_decoder",
           "test_stock_halfrate_decoder", "test_function_level_dropin"]

# name: "long", "multi" or "high"
# setups: what the stage tests run on
# capture: the group and signal of the stored reference capture a setup's encoder blocks come from, where that is not
#   the chain stream
# check(setup, args): the structure the family is about, so that a vorbisenc change cannot turn its tests into a
#   repeat of the default ones
# blocksizes(args): the block sizes of a stock row
# nvec, fmts, envelope: groups of transform vector counts, of sample formats for the mixed-block-size streams, and of
#   setups for the envelope search against the reference; one test each group, and one unparametrized test where a
#   family has one group
# rows: the parameter sets of each stock-codec test; (ch, rate, q), or the managed settings for
#   test_stock_managed_encoder
# fuzz: the setups of test_entropy_coder_fuzz, for the families that collect it
# uncoupled_q: the VBR quality whose template vorbisenc picks for a managed multi row's nominal rate per channel
Family = collections.namedtuple("Family", "name setups capture check blocksizes nvec fmts envelope rows fuzz "
                                           "uncoupled_q", defaults=((), {}))
MANAGED_ARGS = "name,ch,rate,max_br,nominal,min_br,rm2"
LOOPS = {"vector_counts": "nvec", "formats": "fmts", "envelope_setups": "envelope"}


def _group_id(group):
    return "-".join(G.case_id(*v) if isinstance(v, tuple) else str(v) for v in group)


def pytest_generate_tests(metafunc):
    fam = metafunc.module.FAMILY
    names = metafunc.fixturenames
    if "cfg" in names:
        metafunc.parametrize("cfg", fam.setups, indirect=True, ids=lambda a: G.case_id(*a))
        if "vector_counts" in names:
            metafunc.parametrize("W", [0, 1])                # ahead of the vector counts in the ids
    for argname, field in LOOPS.items():
        groups = getattr(fam, field)
        if argname in names and len(groups) > 1:
            metafunc.parametrize(argname, groups, indirect=True, ids=_group_id)
    rows = fam.rows.get(metafunc.definition.name)
    if rows is not None:
        metafunc.parametrize(MANAGED_ARGS if "max_br" in names else "ch,rate,q", rows)


@pytest.fixture
def family(request):
    return request.module.FAMILY


def _group(request, field):
    return request.param if hasattr(request, "param") else getattr(request.module.FAMILY, field)[0]


@pytest.fixture
def vector_counts(request):
    return _group(request, "nvec")


@pytest.fixture
def formats(request):
    return _group(request, "fmts")


@pytest.fixture
def envelope_setups(request):
    return _group(request, "envelope")


def _encoder_blocks(args, o, group, signal):
    """the blocks the reference encoder cut from its stream (tests/golden/ref), in the layout of the golden encode
    fixtures that the tests of test_gpu_parity.py read: <tag>_pcm, _W, _lW, _nW, _blocktype, _ampmax_in, and the
    reference's quantised residue and nonzero flags (the oracle's, checked against the reference's digest)"""
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


@pytest.fixture(scope="module")
def cfg(request, oracle_lib, cuda_ok):
    """(name, setup, context, oracle, encoder blocks, None): the shape of test_gpu_parity.py's fixture"""
    fam, args = request.module.FAMILY, request.param
    setup = G.load_setup(*args)
    fam.check(setup, args)
    o = oracle_lib.Oracle(setup)
    ctx = vlib.Context(setup)
    enc = _encoder_blocks(args, o, *fam.capture.get(args, ("chain", T.chain_signal)))
    yield G.case_id(*args), setup, ctx, o, enc, None
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


def test_transforms_vs_oracle(cfg, W, vector_counts):
    """1 vector, fewer vectors than CTAs, and more vectors than resident CTAs (132 SMs x 8), so that every CTA walks
    several rows and stages the next one with cp.async"""
    name, setup, ctx, o, _, _ = cfg
    for nvec in vector_counts:
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
    """stream mode, float planar and int16 interleaved ingest (the s16 staging takes its stereo path only at two
    channels), and the host path in many chunks"""
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
    """k_cqn_fast for one and two channels, k_cqn for six and for every count above two"""
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
    """the many-chunk host pipeline (ramped and flat chunk schedules), device pointers and their errors, two concurrent
    half batches, int16 residue and partition classes"""
    for ns in (30, 20):
        P.test_encode_dsp_many_chunks(cfg, ns, monkeypatch)
    P.test_encode_dsp_device_pointers_and_errors(cfg)
    P.test_encode_dsp_dev_split_half_batches(cfg)
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


def test_envelope_search_vs_reference(cuda_ok, envelope_setups):
    """the device's envelope search on the reference's own stream buffer gives the reference's marks and filter state
    (stored by tests/golden/make_golden_ref.py)"""
    for args in envelope_setups:
        ctx = vlib.Context(G.load_setup(*args))
        rec = G.load("envelope_" + G.case_id(*args))
        stream = np.concatenate([rec["stream_pre"], T.envelope_signal(*args)], axis=1)
        steps = int(rec["steps"])
        ret, state = ctx.envelope_search(stream[None], 0, steps)
        assert np.array_equal(ctx.envelope_marks(ret[0])[:steps + 2], rec["marks"])
        assert np.array_equal(state[0], rec["state"])
        ctx.close()


def test_encode_streams_mixed_block_sizes(cfg, formats):
    """vb200_encode_streams on streams that switch block sizes: plan, posts, nonzero and residue of every block equal
    the oracle's composition (envelope search, planner with its mark window, ampmax chain)"""
    name, setup, ctx, o, _, _ = cfg
    ch, half = setup.channels, setup.blocksize(1) // 2
    sig = P.streams_signals(ch, setup.rate, None)
    stride = (max(s.shape[1] for s in sig) + 4 * half + 3) & ~3
    for fmt in formats:
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
            got = ctx.encode_streams(np.ascontiguousarray(s16.transpose(0, 2, 1)), pcm_len, eof,
                                     fmt=vlib.PCM_S16_INTERLEAVED)
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
    """the same setups decoding at half rate"""
    name, setup, _, _, enc, _ = cfg
    ctx = vlib.Context(setup)
    ctx.synthesis_halfrate(1)
    yield name, setup, ctx, halfrate.Oracle.create(setup), enc, None
    ctx.close()


def test_halfrate(halfrate_cfg):
    """half-rate synthesis and decode (at 512/4096 the long block's half takes the <2048> instances) and
    mdct_backward"""
    HR.test_random_streams_halfrate(halfrate_cfg)
    HR.test_long_stream_in_overlapping_segments(halfrate_cfg)
    HR.test_mdct_backward_halfrate(halfrate_cfg)


# ---- against the stock encoder and decoder (oracle/_ref) ------------------------------------------------------------
def _stock_bs(ch, rate, q):
    """the block sizes of the stock encoder's setup; the device coder must be taken at them"""
    d = EP._driver(ch, rate, q)                        # skips without oracle/_ref; asserts Driver.on_device
    bs = list(d.ctx.bs)
    d.close()
    assert bs == [512, 4096], "vorbisenc chose %s at (%d, %d, %g)" % (bs, ch, rate, q)


def test_stock_encoder_packets(cuda_ok, family, ch, rate, q):
    """the stock encoder's captured blocks give its audio packets through encode_dsp + encode_entropy and through
    encode_packets; whole streams give its packets, granulepos, e_o_s and packetno, in one call and through a fresh
    carry (multi: also cut into pieces, and raw float and int16 PCM one call per stock write)"""
    if family.name == "long":
        _stock_bs(ch, rate, q)
    EP.test_stage_parity_captured_blocks(cuda_ok, ch, rate, q)
    SP.test_unmanaged_whole_streams(cuda_ok, ch, rate, q)
    SR.test_fresh_carry_one_call_equals_packets_call(cuda_ok, ch, rate, q)
    if family.name == "multi":
        SR.test_cuts_equal_one_call_unmanaged(cuda_ok, ch, rate, q)
        PC.test_one_call_per_stock_write(cuda_ok, ch, rate, q)


def test_stock_encoder_streams_in_pieces(cuda_ok):
    """long: whole streams cut into pieces, at the setup where the stock encoder picks 512/4096"""
    _stock_bs(2, 44100, -0.1)
    SR.test_cuts_equal_one_call_unmanaged(cuda_ok, 2, 44100, -0.1)


def test_stock_encoder_streams_in_pieces_and_raw_pcm(cuda_ok, family, ch, rate, q):
    """high: whole streams cut into pieces, and raw float and int16 PCM one call per stock write"""
    SR.test_cuts_equal_one_call_unmanaged(cuda_ok, ch, rate, q)
    PC.test_one_call_per_stock_write(cuda_ok, ch, rate, q)


def test_entropy_coder_fuzz(cuda_ok, family):
    for args in family.fuzz:
        EP.test_fuzz_against_reference_functions(cuda_ok, *args)


def test_stock_managed_encoder(cuda_ok, family, name, ch, rate, max_br, nominal, min_br, rm2):
    """the block sizes and residue partitions the managed encoder picks; whole streams in one call, in pieces and (multi
    and high) from raw PCM; at cbr320_small packets are both cut and padded"""
    SP._need_ref()
    if not B.ref_available(True):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    d = B.ManagedDriver(ch, rate, max_br, nominal, min_br)       # refuses a host entropy path
    bs, partvals = list(d.ctx.bs), [d.ctx.residue_partvals(W) for W in (0, 1)]
    d.close()
    if family.name == "long":
        assert bs == [512, 4096], "vorbisenc chose %s for %s" % (bs, name)
    elif family.name == "multi":
        r = pyref.Ref(ch, rate, family.uncoupled_q[name])
        s = r.setup()
        r.close()
        assert list(s.c.coupling_steps) == [0, 0] and list(s.c.submaps) == [1, 1]
        assert bs == [s.blocksize(0), s.blocksize(1)] == [256, 2048], name
        assert partvals == [(s.c.residue[W][0].end - s.c.residue[W][0].begin) // s.c.residue[W][0].grouping
                            for W in (0, 1)], "%s: %s partitions" % (name, partvals)
    else:
        assert bs == [256, 2048], name
        # the long block's residue partitions: 2048 / 32 over the whole stereo vector (1888 / 32 below q 0.6), and at
        # least 4290 / 30 in the uncoupled 5.1 setups (4 coupling steps and 135 below q 0.5)
        assert partvals[1] == 64 if ch == 2 else partvals[1] >= 143, "%s: %d partitions" % (name, partvals[1])
    SP.test_managed_whole_streams(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2)
    SR.test_cuts_equal_one_call_managed(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2)
    if family.name != "long":
        PC.test_managed_one_call_per_stock_write(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2)


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


def _streams_and_ranges(cuda_ok, drivers, ch, rate, q):
    for page_final in (False, True):
        DS.test_streams_equal_stock_decoder(cuda_ok, drivers, ch, rate, q, page_final)
        DR.test_index_and_ranges_equal_stock_decoder(cuda_ok, drivers, ch, rate, q, page_final)


def test_stock_decoder(cuda_ok, driver, drivers, family, ch, rate, q):
    """device decode of the stock encoder's packets: the entropy decode's staging equals the reference's, the fused
    resume decode equals entropy decode + DSP (full and half rate, float and int16), and the vb200md driver gives the
    stock decoder's PCM on its device and host paths (multi: also decode_streams_packets and decode_ranges on the
    seven kinds of stream of tests/test_decode_streams_oracle.py)"""
    if not (decode.available() and dp.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    DP.test_stage_parity(cuda_ok, driver, ch, rate, q)
    DP.test_fused_equals_entropy_then_dsp(cuda_ok, driver, ch, rate, q, "two")
    for s16 in (False, True):
        DP.test_driver_device_and_host_paths_equal_stock(cuda_ok, ch, rate, q, s16)
    if family.name == "multi":
        _streams_and_ranges(cuda_ok, drivers, ch, rate, q)


def test_stock_decoder_streams_and_ranges(cuda_ok, drivers, family, ch, rate, q):
    """high: decode_streams_packets and decode_ranges on the seven kinds of stream of
    tests/test_decode_streams_oracle.py"""
    _streams_and_ranges(cuda_ok, drivers, ch, rate, q)


def test_stock_halfrate_decoder(cuda_ok, drivers, family, ch, rate, q):
    """half rate: decode_streams_packets and decode_ranges against the stock half-rate decoder (multi and high), and
    the reference decoder with mdct_backward on the device at half and full rate, which gives the stock PCM"""
    if family.name != "long":
        DS.test_halfrate_equals_stock_halfrate_decoder(cuda_ok, drivers, ch, rate, q)
        DR.test_halfrate_equals_stock_halfrate_decoder(cuda_ok, drivers, ch, rate, q)
    if not (halfrate.ref_available() and halfrate.ref_available(dropin=True)):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    pcm = probe_signal(ch, rate, 0.6, seed=5)
    packets = halfrate.ref_encode(ch, rate, q, pcm)
    bs = family.blocksizes((ch, rate, q))
    for half in (True, False):
        want = halfrate.ref_decode(packets, bs, ch, pcm.shape[1] + 8192, halfrate=half)
        got = halfrate.ref_decode(packets, bs, ch, pcm.shape[1] + 8192, halfrate=half, dropin=True)
        assert set(want["W"].tolist()) == {0, 1}
        assert np.array_equal(got["W"], want["W"]) and got["pcm"].shape == want["pcm"].shape
        assert np.array_equal(got["pcm"].view(np.uint32), want["pcm"].view(np.uint32)), "half rate %s" % half


def test_function_level_dropin(cuda_ok, family, ch, rate, q):
    """the reference's encoder and decoder with their hot callees bound to the device: byte-identical packets and
    bit-identical PCM"""
    if family.name == "long" and pyref.available():
        r = pyref.Ref(ch, rate, q)
        assert list(r.bs) == [512, 4096]
        r.close()
    DI.test_encoder_packets_identical(cuda_ok, ch, rate, q)


# ---- the generic sizes (collected by tests/test_gpu_long_blocks.py) -------------------------------------------------
@pytest.fixture(scope="module", params=[(64, 8192), (128, 4096)], ids=lambda b: "%d_%d" % b)
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
