"""CUDA path (through the C ABI of libvorbis_b200.so) against
  (a) the golden vectors recorded from the reference, and
  (b) the CPU oracle on seeded inputs.
Bit-exact for every stage: the kernels execute the reference's arithmetic DAG with
FMA contraction off (tolerance stated by north_star is 1e-4 relative; we hold 0)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CONFIG_NAMES, REF_ARGS, assert_bits_equal, load_npz, load_setup, make_desc, probe_signal
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=CONFIG_NAMES)
def cfg(request, oracle_lib, cuda_ok):
    name = request.param
    setup = load_setup(name)
    return name, setup, vlib.Context(setup), oracle_lib.Oracle(setup), load_npz("encode", name), load_npz("decode", name)


def test_tables_match_oracle(cfg):
    name, setup, ctx, o, enc, _ = cfg
    for W in (0, 1):
        for which in (0, 1, 2, 3):
            assert_bits_equal(ctx.table(W, which), o.table(W, which), "table W%d #%d" % (W, which))


@pytest.mark.parametrize("tag", ["L", "S"])
def test_transforms_golden(cfg, tag):
    name, setup, ctx, o, enc, _ = cfg
    W = 1 if tag == "L" else 0
    N = setup.blocksize(W)
    pcm = enc[tag + "_pcm"].reshape(-1, N)
    lW = np.repeat(enc[tag + "_lW"], setup.channels)
    nW = np.repeat(enc[tag + "_nW"], setup.channels)
    win = ctx.apply_window(W, pcm, lW, nW)
    assert_bits_equal(win, enc[tag + "_windowed"].reshape(-1, N), "window")
    assert_bits_equal(ctx.mdct_forward(W, win), enc[tag + "_mdct_raw"].reshape(-1, N // 2), "mdct_forward")
    assert_bits_equal(ctx.drft_forward(W, win), enc[tag + "_fft"].reshape(-1, N), "drft_forward")


@pytest.mark.parametrize("W", [0, 1])
def test_transforms_vs_oracle_random(cfg, W):
    name, setup, ctx, o, enc, _ = cfg
    N = setup.blocksize(W)
    rng = np.random.default_rng(12345 + W)
    x = rng.uniform(-1, 1, (300, N)).astype(np.float32)
    x[0] = 0.0                      # silence
    x[1, :] = 1.0                   # DC at full scale
    x[2, ::2] = 1.0; x[2, 1::2] = -1.0
    x[3] *= 1e-30                   # denormal-range products
    assert_bits_equal(ctx.mdct_forward(W, x), o.mdct_forward(W, x), "mdct_forward")
    y = rng.uniform(-1, 1, (300, N // 2)).astype(np.float32)
    y[0] = 0.0
    assert_bits_equal(ctx.mdct_backward(W, y), o.mdct_backward(W, y), "mdct_backward")
    assert_bits_equal(ctx.drft_forward(W, x), o.drft_forward(W, x), "drft_forward")
    lW = rng.integers(0, 2, 300).astype(np.int32)
    nW = rng.integers(0, 2, 300).astype(np.int32)
    assert_bits_equal(ctx.apply_window(W, x, lW, nW), o.apply_window(W, x, lW, nW), "window")
    # empty batch is a no-op
    assert ctx.mdct_forward(W, np.zeros((0, N), np.float32)).shape == (0, N // 2)
    # more vectors than resident CTAs (132 SMs x 8): every CTA walks several vectors, the next one staged by
    # cp.async while the current one is transformed
    big = rng.uniform(-1, 1, (4000, N)).astype(np.float32)
    assert_bits_equal(ctx.mdct_forward(W, big), o.mdct_forward(W, big), "mdct_forward, 4000 vectors")


@pytest.mark.parametrize("tag", ["L", "S"])
def test_psy_stages_isolated_golden(cfg, tag):
    """each stage fed the REFERENCE's upstream vectors (SURVEY §8d parity metric)"""
    name, setup, ctx, o, enc, _ = cfg
    W = 1 if tag == "L" else 0
    n = setup.blocksize(W) // 2
    ch = setup.channels
    for bt in (0, 1):
        sel = np.where(enc[tag + "_blocktype"] == bt)[0]
        if not len(sel):
            continue
        look = bt + 2 * W
        assert_bits_equal(ctx.noisemask(look, enc[tag + "_logmdct"][sel].reshape(-1, n)),
                          enc[tag + "_noise"][sel].reshape(-1, n), "noise look %d" % look)
        g = np.repeat(enc[tag + "_global_ampmax"][sel], ch)
        l = enc[tag + "_local_ampmax"][sel].reshape(-1)
        assert_bits_equal(ctx.tonemask(look, enc[tag + "_logfft"][sel].reshape(-1, n), g, l),
                          enc[tag + "_tone"][sel].reshape(-1, n), "tone look %d" % look)
        lm, m1 = ctx.offset_and_mix(look, 1, enc[tag + "_noise"][sel].reshape(-1, n),
                                    enc[tag + "_tone"][sel].reshape(-1, n),
                                    enc[tag + "_mdct_raw"][sel].reshape(-1, n),
                                    enc[tag + "_logmdct"][sel].reshape(-1, n))
        assert_bits_equal(lm, enc[tag + "_logmask"][sel].reshape(-1, n), "logmask")
        assert_bits_equal(m1, enc[tag + "_mdct_m1"][sel].reshape(-1, n), "mdct after M1")


@pytest.mark.parametrize("look", [0, 1, 2, 3])
def test_psy_stages_vs_oracle_random(cfg, look):
    name, setup, ctx, o, enc, _ = cfg
    n = setup.psy_n(look)
    rng = np.random.default_rng(99 + look)
    nv = 200
    logmdct = (rng.uniform(-140, 0, (nv, n)) + 20 * np.sin(np.arange(n) / 37.0)).astype(np.float32)
    logmdct[0] = -764.6          # todB(0): digital silence
    logmdct[1] = -3.0            # flat loud
    assert_bits_equal(ctx.noisemask(look, logmdct), o.noisemask(look, logmdct), "noise")
    logfft = (rng.uniform(-120, -10, (nv, n))).astype(np.float32)
    logfft[2, n // 3] = 0.0      # one strong tone
    logfft[3] = -200.0
    lmax = np.minimum(logfft.max(axis=1), 0).astype(np.float32)
    gmax = np.maximum(lmax, rng.uniform(-60, 0, nv)).astype(np.float32)
    assert_bits_equal(ctx.tonemask(look, logfft, gmax, lmax), o.tonemask(look, logfft, gmax, lmax), "tone")
    noise = rng.uniform(-120, -10, (nv, n)).astype(np.float32)
    tone = rng.uniform(-120, -10, (nv, n)).astype(np.float32)
    mdct = rng.uniform(-1, 1, (nv, n)).astype(np.float32)
    for sel in (0, 1, 2):
        a = ctx.offset_and_mix(look, sel, noise, tone, mdct, logmdct)
        b = o.offset_and_mix(look, sel, noise, tone, mdct, logmdct)
        assert_bits_equal(a[0], b[0], "logmask sel %d" % sel)
        assert_bits_equal(a[1], b[1], "mdct sel %d" % sel)


@pytest.mark.parametrize("tag", ["L", "S"])
def test_phaseA_golden(cfg, tag):
    """the fused chain against the real mapping0_forward; bit-exact, so no statistical caveat"""
    name, setup, ctx, o, enc, _ = cfg
    W = 1 if tag == "L" else 0
    out = ctx.phaseA(W, enc[tag + "_pcm"], make_desc(enc, tag), taps=True)
    for k, g in (("mdct_raw", "mdct_raw"), ("logfft", "logfft"), ("noise", "noise"), ("tone", "tone"),
                 ("logmdct", "logmdct"), ("logmask", "logmask"), ("mdct", "mdct_m1")):
        assert_bits_equal(out[k], enc[tag + "_" + g], "phaseA " + k)
    assert_bits_equal(out["ampmax_out"], enc[tag + "_ampmax_out"], "ampmax_out")
    # and without taps (the in-place mdct path)
    out2 = ctx.phaseA(W, enc[tag + "_pcm"], make_desc(enc, tag), taps=False)
    for k in ("mdct", "logmdct", "logmask", "ampmax_out"):
        assert_bits_equal(out2[k], out[k], "phaseA(no taps) " + k)


@pytest.mark.parametrize("W", [0, 1])
def test_phaseA_vs_oracle_random(cfg, W):
    name, setup, ctx, o, enc, _ = cfg
    N, ch = setup.blocksize(W), setup.channels
    rng = np.random.default_rng(4242 + W)
    nb = 64
    t = np.arange(N)
    pcm = (0.25 * rng.uniform(-1, 1, (nb, ch, N)) +
           0.5 * np.sin(2 * np.pi * rng.uniform(50, 8000, (nb, ch, 1)) * t / setup.rate)).astype(np.float32)
    pcm[0] = 0.0
    pcm[1] *= 1e-4
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["lW"] = rng.integers(0, 2, nb) if W else 0
    desc["nW"] = rng.integers(0, 2, nb) if W else 0
    desc["blocktype"] = rng.integers(0, 2, nb)
    desc["ampmax"] = rng.choice([-9999.0, -30.0, -3.0, 0.0], nb).astype(np.float32)
    a = ctx.phaseA(W, pcm, desc, taps=True)
    b = o.phaseA(W, pcm, desc, taps=True)
    for k in ("mdct_raw", "logfft", "noise", "tone", "logmdct", "logmask", "mdct", "ampmax_out"):
        assert_bits_equal(a[k], b[k], "phaseA " + k)


# ---------------------------------------------------------------------------------------------
# Phase B: _vp_couple_quantize_normalize (integer outputs: exact match required)
@pytest.mark.parametrize("tag", ["L", "S"])
def test_couple_quantize_normalize_golden(cfg, tag):
    name, setup, ctx, o, enc, _ = cfg
    W = 1 if tag == "L" else 0
    for bt in (0, 1):
        sel = np.where(enc[tag + "_blocktype"] == bt)[0]
        if not len(sel):
            continue
        iw, nz = ctx.couple_quantize_normalize(W, bt, 7, enc[tag + "_mdct_m1"][sel], enc[tag + "_ilogmask"][sel],
                                               enc[tag + "_nonzero_in"][sel])
        assert np.array_equal(iw, enc[tag + "_iwork_out"][sel]), "iwork"
        assert np.array_equal(nz, enc[tag + "_nonzero_out"][sel]), "nonzero"


@pytest.mark.parametrize("W", [0, 1])
def test_couple_quantize_normalize_vs_oracle_random(cfg, W):
    name, setup, ctx, o, enc, _ = cfg
    n, ch = setup.blocksize(W) // 2, setup.channels
    rng = np.random.default_rng(777 + W)
    nb = 48
    # spectra with a wide dynamic range around the floor so that all branches fire:
    # quantise-to-zero pools (noise normalisation), lossless and point stereo, ties
    ilog = rng.integers(40, 220, (nb, ch, n)).astype(np.int32)
    amp = 10.0 ** ((ilog.astype(np.float64) * (140.0 / 255.0) - 140.0 + rng.normal(0, 9, ilog.shape)) / 20.0)
    mdct = (amp * rng.choice([-1.0, 1.0], ilog.shape)).astype(np.float32)
    mdct[0] = 0.0                                   # silence: every line ties
    mdct[1] = np.float32(0.01)                      # constant: ties inside the sort
    if ch == 2:
        mdct[2, 1] = mdct[2, 0]                     # identical channels
        mdct[3, 1] = -mdct[3, 0]
    nz = rng.integers(0, 2, (nb, ch)).astype(np.int32)
    nz[:8] = 1
    for bt in (0, 1):
        for blob in (0, 7, 14):
            a = ctx.couple_quantize_normalize(W, bt, blob, mdct, ilog, nz)
            b = o.couple_quantize_normalize(W, bt, blob, mdct, ilog, nz)
            assert np.array_equal(a[0], b[0]), "iwork bt%d blob%d: %d diffs" % (bt, blob, (a[0] != b[0]).sum())
            assert np.array_equal(a[1], b[1]), "nonzero"


# ---------------------------------------------------------------------------------------------
# decode: mdct_backward + overlap-add
def test_decode_golden(cfg):
    name, setup, ctx, o, _, dec = cfg
    bs = [setup.blocksize(0), setup.blocksize(1)]
    Wseq = dec["W"][None, :]
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, bs, setup.channels)
    pcm = ctx.synthesis(Wseq, coef_off, dec["coef"], pcm_off, pcm_len)
    assert_bits_equal(pcm[0], dec["pcm"], "decoded pcm")


def test_decode_vs_oracle_random_streams(cfg):
    """many independent streams, random long/short sequences (all four overlap cases)"""
    name, setup, ctx, o, _, _ = cfg
    bs = [setup.blocksize(0), setup.blocksize(1)]
    ch = setup.channels
    rng = np.random.default_rng(31337)
    ns, nblk = 37, 23
    Wseq = rng.integers(0, 2, (ns, nblk)).astype(np.int32)
    Wseq[0] = 1
    Wseq[1] = 0
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, bs, ch)
    coef = (rng.uniform(-1, 1, coef_len) * 1e-2).astype(np.float32)
    a = ctx.synthesis(Wseq, coef_off, coef, pcm_off, pcm_len)
    b = o.synthesis(Wseq, coef_off, coef, pcm_off, pcm_len)
    assert_bits_equal(a, b, "decoded streams")
    # a single block finishes nothing
    one = ctx.synthesis(Wseq[:, :1], coef_off[:, :1], coef, pcm_off[:, :1], 8)
    assert not one.any()


def test_phaseA_host_path_multichunk(cfg, monkeypatch):
    """the pipelined host path (as vb200_encode_dsp's: 7 blocks per chunk give 10 ramped chunks over the four buffer
    sets), without taps and with every tap copied back chunk by chunk"""
    name, setup, ctx, o, enc, _ = cfg
    W = 0
    N, ch = setup.blocksize(W), setup.channels
    rng = np.random.default_rng(5)
    nb = 45
    pcm = rng.uniform(-0.7, 0.7, (nb, ch, N)).astype(np.float32)
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["blocktype"] = rng.integers(0, 2, nb)
    desc["ampmax"] = -12.0
    monkeypatch.setenv("VB200_CHUNK_BLOCKS", "7")
    a = ctx.phaseA(W, pcm, desc)
    at = ctx.phaseA(W, pcm, desc, taps=True)
    monkeypatch.delenv("VB200_CHUNK_BLOCKS")
    b = o.phaseA(W, pcm, desc, taps=True)
    for k in ("mdct", "logmdct", "logmask", "ampmax_out"):
        assert_bits_equal(a[k], b[k], "chunked " + k)
    for k in ("mdct_raw", "logfft", "noise", "tone", "logmdct", "logmask", "mdct", "ampmax_out"):
        assert_bits_equal(at[k], b[k], "chunked with taps " + k)


def test_decouple_vs_oracle(cfg):
    name, setup, ctx, o, _, _ = cfg
    ch = setup.channels
    rng = np.random.default_rng(8)
    for W in (0, 1):
        n = setup.blocksize(W) // 2
        res = rng.integers(-6, 7, (33, ch, n)).astype(np.float32)      # residue values are small ints,
        res[0] = 0.0                                                   # zeros and sign ties included
        assert_bits_equal(ctx.decouple(W, res), o.decouple(W, res), "decouple W%d" % W)


def test_phaseA_stream_mode_device(cfg):
    """device-resident stream mode: the ampmax chain of vorbis_analysis_blockout evaluated on the GPU"""
    import torch
    name, setup, ctx, o, _, _ = cfg
    W = 1
    N, ch = setup.blocksize(W), setup.channels
    ns, bps = 7, 9
    rng = np.random.default_rng(99)
    t = np.arange(N)
    amp = rng.choice([1e-3, 0.05, 0.5], (ns, bps, 1, 1))                # loud and quiet blocks: the chain matters
    pcm = (amp * (0.3 * rng.uniform(-1, 1, (ns, bps, ch, N)) +
                  0.6 * np.sin(2 * np.pi * 700 * t / setup.rate))).astype(np.float32).reshape(-1, ch, N)
    desc = np.zeros(ns * bps, abi.BLOCKDESC_DTYPE)
    desc["lW"] = 1; desc["nW"] = 1; desc["blocktype"] = 1
    amp0 = rng.choice([-9999.0, -20.0], ns).astype(np.float32)
    want = o.phaseA(W, pcm, desc, streams=(ns, bps), ampmax0=amp0)
    dev = torch.device("cuda", 0)
    d_pcm = torch.from_numpy(pcm).to(dev)
    d_desc = torch.from_numpy(desc.view(np.uint8).reshape(-1, 16).copy()).to(dev)
    outs = {k: torch.empty((ns * bps, ch, N // 2), device=dev) for k in ("mdct", "logmdct", "logmask")}
    d_amp = torch.empty(ns * bps, device=dev)
    d_amp0 = torch.from_numpy(amp0).to(dev)
    io = abi.PhaseAIO()
    io.pcm, io.desc = d_pcm.data_ptr(), d_desc.data_ptr()
    io.mdct, io.logmdct, io.logmask = (outs[k].data_ptr() for k in ("mdct", "logmdct", "logmask"))
    io.ampmax_out = d_amp.data_ptr()
    ctx.phaseA_dev(W, ns * bps, io, stream=torch.cuda.current_stream().cuda_stream, streams=(ns, bps),
                   d_ampmax0=d_amp0.data_ptr())
    torch.cuda.synchronize()
    for k in ("mdct", "logmdct", "logmask"):
        assert_bits_equal(outs[k].cpu().numpy(), want[k], "stream mode " + k)
    assert_bits_equal(d_amp.cpu().numpy(), want["ampmax_out"], "stream mode ampmax chain")


def test_phaseA_generic_kernel_path(cfg, monkeypatch):
    """the generic psy kernel (k_phaseA_psy, any n) kept as fallback for block sizes the
    register-resident kernel does not cover: same bits"""
    name, setup, ctx, o, enc, _ = cfg
    W = 1
    monkeypatch.setenv("VB200_PSY_V1", "1")
    out = ctx.phaseA(W, enc["L_pcm"], make_desc(enc, "L"), taps=True)
    monkeypatch.delenv("VB200_PSY_V1")
    for k, g in (("noise", "noise"), ("tone", "tone"), ("logmask", "logmask"), ("mdct", "mdct_m1")):
        assert_bits_equal(out[k], enc["L_" + g], "generic kernel " + k)


@pytest.mark.parametrize("W", [0, 1])
def test_phaseA_adversarial_inputs(cfg, W):
    """impulses, DC, full-scale square waves, denormals, huge and tiny amplitudes, exact zeros in one
    channel only: the CUDA chain must follow the reference arithmetic (oracle) bit for bit"""
    name, setup, ctx, o, enc, _ = cfg
    N, ch = setup.blocksize(W), setup.channels
    rng = np.random.default_rng(2718 + W)
    t = np.arange(N)
    cases = []
    imp = np.zeros((ch, N), np.float32); imp[:, N // 2] = 1.0; cases.append(imp)
    imp2 = np.zeros((ch, N), np.float32); imp2[0, 3] = -1.0; cases.append(imp2)
    cases.append(np.full((ch, N), 0.999, np.float32))
    sq = np.where((t // 16) % 2 == 0, 1.0, -1.0).astype(np.float32); cases.append(np.tile(sq, (ch, 1)))
    cases.append(np.full((ch, N), 1e-40, np.float32))                     # denormal PCM
    cases.append((rng.uniform(-1, 1, (ch, N)) * 1e-30).astype(np.float32))
    cases.append((rng.uniform(-1, 1, (ch, N)) * 1e6).astype(np.float32))  # far beyond full scale
    oz = rng.uniform(-0.5, 0.5, (ch, N)).astype(np.float32); oz[-1] = 0.0; cases.append(oz)
    cases.append(np.tile(np.sin(2 * np.pi * 1000.0 * t / setup.rate).astype(np.float32), (ch, 1)))
    cases.append(np.tile(np.float32(0.5) * np.sign(np.sin(2 * np.pi * 6000.0 * t / setup.rate)).astype(np.float32), (ch, 1)))
    pcm = np.stack(cases)
    nb = len(cases)
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["lW"] = (np.arange(nb) % 2) if W else 0
    desc["nW"] = ((np.arange(nb) // 2) % 2) if W else 0
    desc["blocktype"] = np.arange(nb) % 2
    desc["ampmax"] = np.where(np.arange(nb) % 3 == 0, -9999.0, -1.5).astype(np.float32)
    a = ctx.phaseA(W, pcm, desc, taps=True)
    b = o.phaseA(W, pcm, desc, taps=True)
    for k in ("mdct_raw", "logfft", "noise", "tone", "logmdct", "logmask", "mdct", "ampmax_out"):
        assert_bits_equal(a[k], b[k], "adversarial " + k)


@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_phaseA_pcm_ingest_from_stream_buffers(cfg, fmt):
    """SURVEY §8 f4: blocks cut on the device out of one contiguous buffer per stream (hop = N/2,
    lib/block.c:630-643), float planar or interleaved int16 (/32768.f, examples/encoder_example.c:196-201);
    must equal the block-layout path fed the same samples (checked against the oracle's stream mode)"""
    import torch
    name, setup, ctx, o, _, _ = cfg
    W = 1
    N, ch = setup.blocksize(W), setup.channels
    hop, ns, bps = N // 2, 5, 6
    stride = (bps - 1) * hop + N + 8
    rng = np.random.default_rng(123)
    t = np.arange(stride)
    s16 = np.clip(6000 * rng.standard_normal((ns, stride, ch)) +
                  12000 * np.sin(2 * np.pi * 523.0 * t / setup.rate)[None, :, None], -32768, 32767).astype(np.int16)
    f32 = (s16.astype(np.float32) / np.float32(32768.0))            # [ns][stride][ch]
    planar = np.ascontiguousarray(f32.transpose(0, 2, 1))           # [ns][ch][stride]
    blocks = np.stack([planar[s, :, k * hop:k * hop + N] for s in range(ns) for k in range(bps)])
    desc = np.zeros(ns * bps, abi.BLOCKDESC_DTYPE)
    desc["lW"] = 1; desc["nW"] = 1; desc["blocktype"] = 1
    want = o.phaseA(W, blocks, desc, streams=(ns, bps))
    dev = torch.device("cuda", 0)
    d_desc = torch.from_numpy(desc.view(np.uint8).reshape(-1, 16).copy()).to(dev)
    outs = {k: torch.empty((ns * bps, ch, N // 2), device=dev) for k in ("mdct", "logmdct", "logmask")}
    d_amp = torch.empty(ns * bps, device=dev)
    io = abi.PhaseAIO()
    io.desc = d_desc.data_ptr()
    io.mdct, io.logmdct, io.logmask = (outs[k].data_ptr() for k in ("mdct", "logmdct", "logmask"))
    io.ampmax_out = d_amp.data_ptr()
    if fmt == "s16":
        d_pcm = torch.from_numpy(s16).to(dev)
        ctx.phaseA_pcmstream_dev(W, ns, bps, d_pcm.data_ptr(), vlib.PCM_S16_INTERLEAVED, stride, hop, io,
                                 stream=torch.cuda.current_stream().cuda_stream)
    else:
        d_pcm = torch.from_numpy(planar).to(dev)
        ctx.phaseA_pcmstream_dev(W, ns, bps, d_pcm.data_ptr(), vlib.PCM_F32_PLANAR, stride, hop, io,
                                 stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for k in ("mdct", "logmdct", "logmask"):
        assert_bits_equal(outs[k].cpu().numpy(), want[k], "pcm ingest %s %s" % (fmt, k))
    assert_bits_equal(d_amp.cpu().numpy(), want["ampmax_out"], "pcm ingest ampmax")


def test_decode_int16_egress(cfg):
    """finished samples as interleaved int16: floor(x*32767.f+.5f), clipped (examples/decoder_example.c:250-262)"""
    import torch
    name, setup, ctx, o, _, dec = cfg
    bs = [setup.blocksize(0), setup.blocksize(1)]
    ch = setup.channels
    rng = np.random.default_rng(77)
    ns, nblk = 6, 9
    Wseq = rng.integers(0, 2, (ns, nblk)).astype(np.int32)
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, bs, ch)
    coef = (rng.uniform(-1, 1, coef_len) * 0.08).astype(np.float32)      # loud enough to clip sometimes
    ref_f = o.synthesis(Wseq, coef_off, coef, pcm_off, pcm_len)          # [ns][ch][len] float
    want = np.floor(ref_f * np.float32(32767.0) + np.float32(0.5))
    want = np.clip(want, -32768, 32767).astype(np.int16).transpose(0, 2, 1)   # [ns][len][ch]
    dev = torch.device("cuda", 0)
    d = {k: torch.from_numpy(v).to(dev) for k, v in
         (("W", Wseq), ("co", coef_off), ("c", coef), ("po", pcm_off))}
    out = torch.zeros((ns, pcm_len, ch), dtype=torch.int16, device=dev)
    ctx.synthesis_s16_dev(ns, nblk, d["W"].data_ptr(), d["co"].data_ptr(), d["c"].data_ptr(), d["po"].data_ptr(),
                          out.data_ptr(), pcm_len, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert (np.abs(want.astype(np.int32)) == 32767).any() or (want == -32768).any(), "test signal should clip"
    # only positions that blocks actually finish are written; the layout leaves no gaps
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------
# floor 1 (SURVEY §8 f1)
@pytest.mark.parametrize("tag", ["L", "S"])
def test_floor1_golden(cfg, tag):
    from test_oracle_golden import floor_expect
    name, setup, ctx, o, enc, _ = cfg
    W = 1 if tag == "L" else 0
    n = setup.blocksize(W) // 2
    fit, nz, encp = floor_expect(enc, tag)
    posts, got_nz = ctx.floor1_fit(W, enc[tag + "_logmdct"], enc[tag + "_logmask"])
    assert np.array_equal(got_nz, nz), "fit_nonzero"
    assert np.array_equal(posts, fit), "fit posts: %d diffs" % (posts != fit).sum()
    p2, ilog, nz2 = ctx.floor1_render(W, posts, got_nz)
    assert np.array_equal(p2[nz == 1], encp[nz == 1]), "encode posts"
    assert np.array_equal(ilog, enc[tag + "_ilogmask"].reshape(-1, n)), "ilogmask"
    assert np.array_equal(nz2, enc[tag + "_nonzero_in"].reshape(-1)), "nonzero"


@pytest.mark.parametrize("W", [0, 1])
def test_floor1_vs_oracle_random(cfg, W):
    """masks from the oracle's own Phase A on random PCM plus synthetic curves that force the
    corner cases: silence (NULL), flat curves, cliffs, everything inaudible, everything clipped."""
    name, setup, ctx, o, enc, _ = cfg
    N, ch = setup.blocksize(W), setup.channels
    n = N // 2
    rng = np.random.default_rng(4242 + W)
    nb = 24
    scale = 10.0 ** rng.uniform(-4, 0, (nb, 1, 1))
    pcm = (rng.uniform(-1, 1, (nb, ch, N)) * scale).astype(np.float32)
    t = np.arange(N)
    pcm[3] += (0.5 * np.sin(2 * np.pi * 0.013 * t)).astype(np.float32)
    pcm[5] = 0
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["lW"] = W; desc["nW"] = W; desc["blocktype"] = rng.integers(0, 2, nb); desc["ampmax"] = -9999.0
    pa = o.phaseA(W, pcm, desc)
    logmdct = [pa["logmdct"].reshape(-1, n)]
    logmask = [pa["logmask"].reshape(-1, n)]
    R = 12 * ch
    x = np.arange(n)
    syn_mask = rng.uniform(-140, 0, (R, n)).astype(np.float32)
    syn_mdct = (syn_mask + rng.normal(0, 12, (R, n))).astype(np.float32)
    syn_mask[0] = -60.0                                         # flat
    syn_mask[1] = np.where(x < n // 3, -20.0, -120.0)           # cliff
    syn_mdct[2] = -400.0                                        # nothing audible: every bin in the "b" sums
    syn_mask[3] = 20.0                                          # dBquant clips at 1023
    syn_mask[4] = -200.0                                        # dBquant clips at 0 -> NULL fit
    syn_mask[5] = (-30.0 - 80.0 * x / n).astype(np.float32)     # a straight line: no splits needed
    syn_mask[6] = np.where(rng.uniform(0, 1, n) < 0.1, -10.0, -139.9)  # sparse peaks
    logmdct.append(syn_mdct); logmask.append(syn_mask)
    logmdct = np.concatenate(logmdct); logmask = np.concatenate(logmask)
    a = ctx.floor1_fit(W, logmdct, logmask)
    b = o.floor1_fit(W, logmdct, logmask)
    assert np.array_equal(a[1], b[1]), "fit_nonzero"
    assert (b[1] == 0).any() and (b[1] == 1).any()
    assert np.array_equal(a[0], b[0]), "posts: %d diffs in rows %s" % ((a[0] != b[0]).sum(), np.unique(np.argwhere(a[0] != b[0])[:, 0])[:8])
    ra = ctx.floor1_render(W, a[0], a[1])
    rb = o.floor1_render(W, b[0], b[1])
    for k, what in enumerate(("posts", "ilogmask", "nonzero")):
        assert np.array_equal(ra[k], rb[k]), what
    # explicit floor selection (what one reference call does): rows of channel 0 only
    sel = setup.floor_of(W, 0)
    rows = np.arange(0, logmdct.shape[0], ch)
    a0 = ctx.floor1_fit(W, logmdct[rows], logmask[rows], floor_sel=sel)
    assert np.array_equal(a0[0], b[0][rows]) and np.array_equal(a0[1], b[1][rows])


@pytest.mark.parametrize("tag", ["L", "S"])
def test_encode_chain_on_device_golden(cfg, tag):
    """PCM -> Phase A -> floor1_fit -> floor render -> couple/quantise/normalise, every buffer
    resident on the device, equals what the reference's mapping0_forward produced."""
    import torch
    name, setup, ctx, o, enc, _ = cfg
    W = 1 if tag == "L" else 0
    N, ch = setup.blocksize(W), setup.channels
    n = N // 2
    for bt in (0, 1):
        sel = np.where(enc[tag + "_blocktype"] == bt)[0]
        if not len(sel):
            continue
        nb = len(sel)
        dev = torch.device("cuda")
        pcm = torch.from_numpy(np.ascontiguousarray(enc[tag + "_pcm"][sel])).to(dev)
        desc = torch.from_numpy(make_desc(enc, tag, sel).view(np.uint8).reshape(-1, 16).copy()).to(dev)
        mdct = torch.empty((nb, ch, n), dtype=torch.float32, device=dev)
        logmdct = torch.empty_like(mdct); logmask = torch.empty_like(mdct)
        amp = torch.empty(nb, dtype=torch.float32, device=dev)
        posts = torch.empty((nb * ch, abi.FLOOR1_STRIDE), dtype=torch.int32, device=dev)
        fnz = torch.empty(nb * ch, dtype=torch.int32, device=dev)
        iwork = torch.empty((nb, ch, n), dtype=torch.int32, device=dev)
        nz = torch.empty(nb * ch, dtype=torch.int32, device=dev)
        st = torch.cuda.current_stream().cuda_stream
        io = abi.PhaseAIO()
        io.pcm, io.desc = pcm.data_ptr(), desc.data_ptr()
        io.mdct, io.logmdct, io.logmask, io.ampmax_out = mdct.data_ptr(), logmdct.data_ptr(), logmask.data_ptr(), amp.data_ptr()
        ctx.phaseA_dev(W, nb, io, stream=st)
        ctx.floor1_fit_dev(W, nb * ch, logmdct.data_ptr(), logmask.data_ptr(), posts.data_ptr(), fnz.data_ptr(), stream=st)
        ctx.floor1_render_dev(W, nb * ch, posts.data_ptr(), fnz.data_ptr(), iwork.data_ptr(), nz.data_ptr(), stream=st)
        ctx.couple_quantize_normalize_dev(W, bt, 7, nb, mdct.data_ptr(), iwork.data_ptr(), nz.data_ptr(), stream=st)
        torch.cuda.synchronize()
        assert np.array_equal(iwork.cpu().numpy(), enc[tag + "_iwork_out"][sel]), "iwork"
        assert np.array_equal(nz.cpu().numpy().reshape(nb, ch), enc[tag + "_nonzero_out"][sel]), "nonzero"


def _enc_compare(got, want, what):
    for k in ("posts", "nonzero", "iwork"):
        assert np.array_equal(got[k], want[k]), "%s: %s" % (what, k)
    assert_bits_equal(got["ampmax_out"], want["ampmax_out"], what + ": ampmax_out")
    for k in ("mdct", "logmdct", "logmask"):
        if k in got:
            assert_bits_equal(got[k], want[k], "%s: %s" % (what, k))


@pytest.mark.parametrize("tag", ["L", "S"])
def test_encode_dsp_one_call_golden(cfg, tag):
    """vb200_encode_dsp (host buffers, one call for the whole chain of mapping0_forward) equals what
    the reference's mapping0_forward produced: quantised residue, nonzero, and - through the oracle -
    the floor posts; blocks of both blocktypes in ONE batch (per-block psy look)."""
    name, setup, ctx, o, enc, _ = cfg
    W = 1 if tag == "L" else 0
    nb = len(enc[tag + "_blocktype"])
    if not nb:
        pytest.skip("no such blocks in the fixture")
    sel = np.arange(nb)
    desc = make_desc(enc, tag, sel)
    got = ctx.encode_dsp(W, enc[tag + "_pcm"], desc, floats=True)
    assert np.array_equal(got["iwork"], enc[tag + "_iwork_out"]), "iwork vs reference"
    assert np.array_equal(got["nonzero"], enc[tag + "_nonzero_out"]), "nonzero vs reference"
    ep = enc[tag + "_enc_posts"].astype(np.int32).copy()
    ep[enc[tag + "_fit_posts"][..., 0] == -1] = 0                       # NULL fit: the API returns a zero row
    assert np.array_equal(got["posts"], ep), "posts vs reference (floor1_encode)"
    assert_bits_equal(got["mdct"], enc[tag + "_mdct_m1"], "mdct vs reference")
    assert_bits_equal(got["logmask"], enc[tag + "_logmask"], "logmask vs reference")
    _enc_compare(got, o.encode_dsp(W, enc[tag + "_pcm"], desc), "golden " + tag)


@pytest.mark.parametrize("fmt", ["blocks", "f32", "s16"])
@pytest.mark.parametrize("W", [0, 1])
def test_encode_dsp_streams_vs_oracle(cfg, W, fmt, monkeypatch):
    """streams of consecutive blocks cut on the device from contiguous PCM (int16 interleaved or float
    planar), ampmax chain per stream, mixed blocktypes, several pipeline chunks and a ragged last one"""
    name, setup, ctx, o, _, _ = cfg
    monkeypatch.setenv("VB200_CHUNK_BLOCKS", "12")
    N, ch = setup.blocksize(W), setup.channels
    hop, ns, bps = N // 2, 7, 5
    stride = (bps - 1) * hop + N + 4
    rng = np.random.default_rng(77 + W)
    t = np.arange(stride)
    s16 = np.clip(5000 * rng.standard_normal((ns, stride, ch)) * rng.uniform(0.02, 1.5, (ns, 1, 1)) +
                  9000 * np.sin(2 * np.pi * 660.0 * t / setup.rate)[None, :, None], -32768, 32767).astype(np.int16)
    s16[2] = 0                                                        # a silent stream: floor1_fit returns NULL
    planar = np.ascontiguousarray((s16.astype(np.float32) / np.float32(32768.0)).transpose(0, 2, 1))
    blocks = np.stack([planar[s, :, k * hop:k * hop + N] for s in range(ns) for k in range(bps)])
    desc = np.zeros(ns * bps, abi.BLOCKDESC_DTYPE)
    desc["lW"] = W; desc["nW"] = W
    desc["blocktype"] = rng.integers(0, 2, ns * bps)
    amp0 = rng.uniform(-40, -3, ns).astype(np.float32)
    want = o.encode_dsp(W, blocks, desc, streams=(ns, bps), ampmax0=amp0)
    if fmt == "blocks":
        got = ctx.encode_dsp(W, blocks, desc, nstreams=ns, ampmax0=amp0, independent=False, floats=True)
    elif fmt == "f32":
        got = ctx.encode_dsp(W, planar, desc, nstreams=ns, fmt=vlib.PCM_F32_PLANAR, hop=hop, ampmax0=amp0,
                             independent=False, floats=True)
    else:
        got = ctx.encode_dsp(W, s16, desc, nstreams=ns, fmt=vlib.PCM_S16_INTERLEAVED, hop=hop, ampmax0=amp0,
                             independent=False)
    _enc_compare(got, want, "streams %s W=%d" % (fmt, W))
    assert not got["nonzero"][2 * bps:3 * bps].any(), "silent stream must come back all-zero"


@pytest.mark.parametrize("ns", [30, 20])
def test_encode_dsp_many_chunks(cfg, ns, monkeypatch):
    """the host-buffer pipeline of vb200_encode_dsp with more chunks than buffer sets (the event chain
    H2D(k) -> kernels(k) -> D2H(k) -> H2D(k+4) is exercised), at 4 streams per chunk: 30 streams take the ramped
    chunk schedule (10 chunks), 20 streams the flat one (5 chunks)"""
    name, setup, ctx, o, _, _ = cfg
    monkeypatch.setenv("VB200_CHUNK_BLOCKS", "12")
    W = 1
    N, ch = setup.blocksize(W), setup.channels
    hop, bps = N // 2, 3
    stride = (bps - 1) * hop + N
    rng = np.random.default_rng(4242)
    s16 = np.clip(6000 * rng.standard_normal((ns, stride, ch)) * rng.uniform(0.05, 1.2, (ns, 1, 1)), -32768, 32767).astype(np.int16)
    planar = np.ascontiguousarray((s16.astype(np.float32) / np.float32(32768.0)).transpose(0, 2, 1))
    blocks = np.stack([planar[s, :, k * hop:k * hop + N] for s in range(ns) for k in range(bps)])
    desc = np.zeros(ns * bps, abi.BLOCKDESC_DTYPE)
    desc["lW"] = W; desc["nW"] = W
    desc["blocktype"] = rng.integers(0, 2, ns * bps)
    amp0 = rng.uniform(-40, -3, ns).astype(np.float32)
    want = o.encode_dsp(W, blocks, desc, streams=(ns, bps), ampmax0=amp0)
    for rep in range(2):                                             # the second call reuses the buffer sets
        got = ctx.encode_dsp(W, s16, desc, nstreams=ns, fmt=vlib.PCM_S16_INTERLEAVED, hop=hop, ampmax0=amp0,
                             independent=False)
        _enc_compare(got, want, "many chunks ns=%d rep=%d" % (ns, rep))


@pytest.mark.parametrize("fmt", ["s16", "blocks"])
@pytest.mark.parametrize("W", [0, 1])
def test_encode_dsp_managed_vs_oracle(cfg, W, fmt):
    """bitrate-managed mode (vb200_encode_dsp_managed): the 15 curves of every block - posts, nonzero flags and
    quantised residue of each - against the composed oracle (pinned on the reference's own functions in
    tests/test_oracle_vs_ref.py::test_managed_chain_vs_reference); streams with an ampmax chain, mixed block
    types, a silent stream (all 15 curves NULL) and a nearly silent one"""
    name, setup, ctx, o, _, _ = cfg
    N, ch = setup.blocksize(W), setup.channels
    hop, ns, bps = N // 2, 5, 3
    stride = (bps - 1) * hop + N
    rng = np.random.default_rng(555 + W)
    t = np.arange(stride)
    s16 = np.clip(5000 * rng.standard_normal((ns, stride, ch)) * rng.uniform(0.02, 1.5, (ns, 1, 1)) +
                  9000 * np.sin(2 * np.pi * 440.0 * t / setup.rate)[None, :, None], -32768, 32767).astype(np.int16)
    s16[1] = 0
    s16[3] = (s16[3] // 2000).astype(np.int16)
    planar = np.ascontiguousarray((s16.astype(np.float32) / np.float32(32768.0)).transpose(0, 2, 1))
    blocks = np.stack([planar[s, :, k * hop:k * hop + N] for s in range(ns) for k in range(bps)])
    desc = np.zeros(ns * bps, abi.BLOCKDESC_DTYPE)
    desc["lW"] = W; desc["nW"] = W
    desc["blocktype"] = rng.integers(0, 2, ns * bps)
    amp0 = rng.uniform(-40, -3, ns).astype(np.float32)
    want = o.encode_dsp_managed(W, blocks, desc, streams=(ns, bps), ampmax0=amp0)
    if fmt == "s16":
        got = ctx.encode_dsp_managed(W, s16, desc, nstreams=ns, fmt=vlib.PCM_S16_INTERLEAVED, hop=hop, ampmax0=amp0,
                                     independent=False)
    else:
        got = ctx.encode_dsp_managed(W, blocks, desc, nstreams=ns, ampmax0=amp0, independent=False)
    for k in ("posts", "nonzero", "iwork"):
        assert np.array_equal(got[k], want[k]), "%s: %d diffs" % (k, int((got[k] != want[k]).sum()))
    assert_bits_equal(got["ampmax_out"], want["ampmax_out"], "ampmax_out")
    assert not got["nonzero"][:, bps:2 * bps].any(), "the silent stream has no curve at any rate"
    # the middle curve is what the un-managed call produces
    one = ctx.encode_dsp(W, s16, desc, nstreams=ns, fmt=vlib.PCM_S16_INTERLEAVED, hop=hop, ampmax0=amp0, independent=False)
    mid = abi.PACKETBLOBS // 2
    for k in ("posts", "nonzero", "iwork"):
        assert np.array_equal(got[k][mid], one[k]), "curve 7 vs vb200_encode_dsp: " + k


def test_encode_dsp_device_pointers_and_errors(cfg):
    import torch
    name, setup, ctx, o, enc, _ = cfg
    W = 1
    N, ch = setup.blocksize(W), setup.channels
    n = N // 2
    nb = min(4, len(enc["L_blocktype"]))
    desc = make_desc(enc, "L", np.arange(nb))
    pcm = np.ascontiguousarray(enc["L_pcm"][:nb])
    want = o.encode_dsp(W, pcm, desc)
    dev = torch.device("cuda")
    t = {"pcm": torch.from_numpy(pcm).to(dev),
         "desc": torch.from_numpy(desc.view(np.uint8).reshape(-1, 16).copy()).to(dev),
         "posts": torch.zeros((nb, ch, abi.FLOOR1_STRIDE), dtype=torch.int32, device=dev),
         "nonzero": torch.zeros((nb, ch), dtype=torch.int32, device=dev),
         "iwork": torch.zeros((nb, ch, n), dtype=torch.int32, device=dev),
         "ampmax_out": torch.zeros(nb, device=dev)}
    io = abi.EncodeIO()
    for k, v in t.items():
        setattr(io, k, v.data_ptr())
    io.independent = 1
    ctx.encode_dsp_dev(W, nb, 1, io, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = {k: t[k].cpu().numpy() for k in ("posts", "nonzero", "iwork", "ampmax_out")}
    _enc_compare(got, want, "device pointers")
    io.pcm_fmt = 9
    with pytest.raises(vlib.VB200Error):
        ctx.encode_dsp_dev(W, nb, 1, io)
    io.pcm_fmt = vlib.PCM_S16_INTERLEAVED; io.hop = N // 2; io.stream_stride = N - 2
    with pytest.raises(vlib.VB200Error):
        ctx.encode_dsp_dev(W, nb, 1, io)
    io.pcm_fmt = 0; io.posts = None
    with pytest.raises(vlib.VB200Error):
        ctx.encode_dsp_dev(W, nb, 1, io)


@pytest.mark.parametrize("W", [0, 1])
def test_encode_dsp_int16_residue(cfg, W, monkeypatch):
    """VB200_IWORK_S16: the residue leaves as int16; equal to the int32 result where it fits, saturated and
    counted per block where it does not (PCM far outside [-1,1] makes |mdct|/floor exceed 32767)"""
    name, setup, ctx, o, _, _ = cfg                          # incl. the 6-channel setup (per-block counts by division)
    monkeypatch.setenv("VB200_CHUNK_BLOCKS", "5")
    N, ch = setup.blocksize(W), setup.channels
    rng = np.random.default_rng(5 + W)
    nb = 12
    pcm = (0.3 * rng.standard_normal((nb, ch, N))).astype(np.float32)
    pcm[3] *= 3e6                                                      # overflowing block
    pcm[8, 0] *= 1e6
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["lW"] = W; desc["nW"] = W; desc["blocktype"] = np.arange(nb) % 2; desc["ampmax"] = -10.0
    want = o.encode_dsp(W, pcm, desc)
    got = ctx.encode_dsp(W, pcm, desc, iwork_s16=True)
    assert got["iwork"].dtype == np.int16
    assert np.array_equal(got["iwork"], np.clip(want["iwork"], -32768, 32767).astype(np.int16))
    clipped = ((want["iwork"] > 32767) | (want["iwork"] < -32768)).reshape(nb, -1).sum(1)
    assert np.array_equal(got["overflow"], clipped)
    assert clipped[3] > 0 and clipped[0] == 0
    for k in ("posts", "nonzero"):
        assert np.array_equal(got[k], want[k]), k


def test_envelope_search_golden(cfg):
    """SURVEY §8 f2: the envelope / block-switch detector on the device equals the reference's
    _ve_envelope_search: marks and the carried filter state (lib/envelope.c:88-267)"""
    name, setup, ctx, o, _, _ = cfg
    env = load_npz("envelope", name)
    steps = int(env["steps"])
    ret, state = ctx.envelope_search(env["stream"][None], 0, steps)
    assert np.array_equal(ctx.envelope_marks(ret[0])[:steps + 2], env["marks"]), "marks vs reference"
    assert np.array_equal(state[0], env["state"]), "filter state vs reference"
    want_ret, want_state = o.envelope_search(env["stream"][None], 0, steps)
    assert np.array_equal(ret, want_ret)


@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_envelope_search_streams_vs_oracle(cfg, fmt):
    """many streams at once, int16 or float PCM, the search cut into two calls with the state carried"""
    import torch
    name, setup, ctx, o, _, _ = cfg
    ch = setup.channels
    ns, stride = 9, 64 * 90 + 128
    rng = np.random.default_rng(21)
    t = np.arange(stride)
    s16 = np.clip(4000 * rng.standard_normal((ns, stride, ch)) * rng.uniform(0.01, 2.0, (ns, 1, 1)) +
                  9000 * np.sin(2 * np.pi * 500.0 * t / setup.rate)[None, :, None], -32768, 32767).astype(np.int16)
    for s in range(ns):                                  # bursts and drop-outs at different places
        a = 300 + 517 * s
        s16[s, a:a + 400] //= 64
        s16[s, a + 400:a + 520] = rng.integers(-30000, 30000, (120, ch))
    s16[4] = 0                                           # digital silence
    planar = np.ascontiguousarray((s16.astype(np.float32) / np.float32(32768.0)).transpose(0, 2, 1))
    nsteps = 90
    want_ret, want_state = o.envelope_search(planar, 0, nsteps)
    src = planar if fmt == "f32" else s16
    f = vlib.PCM_F32_PLANAR if fmt == "f32" else vlib.PCM_S16_INTERLEAVED
    r1, s1 = ctx.envelope_search(src, 0, 37, fmt=f)
    r2, s2 = ctx.envelope_search(src, 37, nsteps - 37, state=s1, fmt=f)
    assert np.array_equal(np.concatenate([r1, r2], 1), want_ret), "trigger bits"
    assert np.array_equal(s2, want_state), "state"
    assert (want_ret != 0).any()
    # device pointers
    dev = torch.device("cuda")
    d_pcm = torch.from_numpy(src).to(dev)
    d_state = torch.zeros((ns, abi.ve_state_words(ch)), dtype=torch.int32, device=dev)
    d_ret = torch.zeros((ns, nsteps), dtype=torch.uint8, device=dev)
    ctx.envelope_search_dev(ns, d_pcm.data_ptr(), f, stride, 0, nsteps, d_state.data_ptr(), d_ret.data_ptr(),
                            stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_ret.cpu().numpy(), want_ret) and np.array_equal(d_state.cpu().numpy(), want_state)
    with pytest.raises(vlib.VB200Error):
        ctx.envelope_search(src, 80, 20, fmt=f)          # runs past the stream buffer


def _random_fit(rng, rows):
    posts = rng.integers(0, 140, (rows, abi.FLOOR1_STRIDE)).astype(np.int32)
    flag = rng.random(posts.shape) < 0.4
    flag[:, :2] = False
    posts[flag] |= 0x8000
    return posts


@pytest.mark.parametrize("W", [0, 1])
def test_floor1_inverse2_vs_oracle(cfg, W):
    """SURVEY §8 f3: the decode-side floor multiply (lib/floor1.c:1041-1086)"""
    name, setup, ctx, o, _, _ = cfg
    rng = np.random.default_rng(40 + W)
    n, rows = setup.blocksize(W) // 2, setup.channels * 9
    posts = _random_fit(rng, rows)
    posts[2, 7] = 400
    posts[5, 0] = 999
    present = (rng.random(rows) < 0.85).astype(np.int32)
    data = (rng.standard_normal((rows, n)) * 5).astype(np.float32)
    assert_bits_equal(ctx.floor1_inverse2(W, posts, present, data), o.floor1_inverse2(W, posts, present, data),
                      "floor1_inverse2")


@pytest.mark.parametrize("s16", [False, True])
def test_decode_dsp_one_call_vs_oracle(cfg, s16):
    """de-coupling + floor multiply + IMDCT + overlap-add in one call on packed mixed-size streams"""
    name, setup, ctx, o, _, _ = cfg
    ch = setup.channels
    bs = [setup.blocksize(0), setup.blocksize(1)]
    rng = np.random.default_rng(11)
    ns, nblk = 5, 9
    Wseq = rng.integers(0, 2, (ns, nblk)).astype(np.int32)
    Wseq[0] = 1
    Wseq[1] = 0
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, bs, ch)
    res = np.rint(rng.standard_normal(coef_len) * 3).astype(np.float32)        # residue backends leave integers
    posts = _random_fit(rng, ns * nblk * ch).reshape(ns, nblk, ch, -1)
    present = (rng.random((ns, nblk, ch)) < 0.9).astype(np.int32)
    want = o.decode_dsp(Wseq, coef_off, res, posts, present, pcm_off, pcm_len)
    got = ctx.decode_dsp(Wseq, coef_off, res, posts, present, pcm_off, pcm_len, s16=s16)
    if s16:
        w16 = np.clip(np.floor(want * np.float32(32767.0) + np.float32(0.5)), -32768, 32767).astype(np.int16)
        assert np.array_equal(got, w16.transpose(0, 2, 1))
    else:
        assert_bits_equal(got, want, "decode_dsp pcm")


def test_encode_then_decode_round_trip(cfg):
    """size-independent property: what vb200_encode_dsp hands to the entropy coder (posts + quantised,
    coupled residue), fed to vb200_decode_dsp as the entropy decoder would deliver it, reconstructs the
    PCM (lossy codec: the reconstruction must track the input closely, and equal the oracle's)"""
    name, setup, ctx, o, _, _ = cfg
    W = 1
    N, ch = setup.blocksize(W), setup.channels
    hop, ns, bps = N // 2, 3, 8
    stride = (bps - 1) * hop + N
    rng = np.random.default_rng(8)
    t = np.arange(stride)
    pcm = np.stack([[0.05 * rng.standard_normal(stride) + 0.4 * np.sin(2 * np.pi * (300 + 90 * c + 40 * s) * t / setup.rate)
                     for c in range(ch)] for s in range(ns)]).astype(np.float32)
    desc = np.zeros(ns * bps, abi.BLOCKDESC_DTYPE)
    desc["lW"] = 1; desc["nW"] = 1; desc["blocktype"] = 1
    enc = ctx.encode_dsp(W, pcm, desc, nstreams=ns, fmt=vlib.PCM_F32_PLANAR, hop=hop, independent=False)
    Wseq = np.ones((ns, bps), np.int32)
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, [setup.blocksize(0), N], ch)
    res = enc["iwork"].astype(np.float32).reshape(-1)
    assert res.size == coef_len
    present = (enc["posts"][..., 0] != 0) | (enc["posts"][..., 1] != 0) | (enc["nonzero"] != 0)
    got = ctx.decode_dsp(Wseq, coef_off, res, enc["posts"], present.astype(np.int32), pcm_off, pcm_len)
    want = o.decode_dsp(Wseq, coef_off, res, enc["posts"], present.astype(np.int32), pcm_off, pcm_len)
    assert_bits_equal(got, want, "round trip pcm")
    # block k (k >= 1) finishes the samples between the centres of blocks k-1 and k: output sample i
    # is stream sample N/2 + i (lib/block.c:767-823)
    m = pcm_len
    ref = pcm[:, :, N // 2:N // 2 + m]
    err = got[:, :, :ref.shape[2]] - ref
    snr = 10 * np.log10((ref ** 2).sum() / (err ** 2).sum())
    assert snr > 10.0, "reconstruction SNR %.1f dB" % snr


@pytest.mark.parametrize("W", [0, 1])
def test_residue_classify_vs_oracle(cfg, W):
    """SURVEY §8 f3: residue partition classification (lib/res0.c:412-532) per submap"""
    name, setup, ctx, o, enc, _ = cfg
    ch, n = setup.channels, setup.blocksize(W) // 2
    rng = np.random.default_rng(14 + W)
    nb = 40
    mag = np.exp(rng.uniform(-2, 3, (nb, ch, 1))) * np.exp(-np.arange(n) / (n / 4.0))[None, None, :]
    iwork = np.rint(rng.standard_normal((nb, ch, n)) * mag).astype(np.int32)
    nonzero = (rng.random((nb, ch)) < 0.8).astype(np.int32)
    nonzero[3] = 0
    assert ctx.residue_partvals(W) == o.residue_partvals(W) > 0
    got = ctx.residue_classify(W, iwork, nonzero)
    assert np.array_equal(got, o.residue_classify(W, iwork, nonzero))
    wide = ctx.residue_classify(W, iwork, nonzero, stride=ctx.residue_partvals(W) + 5)
    assert np.array_equal(wide[:, :, :got.shape[2]], got) and not wide[:, :, got.shape[2]:].any()
    with pytest.raises(vlib.VB200Error):
        ctx.residue_classify(W, iwork, nonzero, stride=ctx.residue_partvals(W) - 1)
    # on the reference's own residue vectors
    tag = "L" if W else "S"
    if len(enc[tag + "_blocktype"]):
        iw, nz = enc[tag + "_iwork_out"], enc[tag + "_nonzero_out"]
        assert np.array_equal(ctx.residue_classify(W, iw, nz), o.residue_classify(W, iw, nz))


def test_encode_dsp_with_classes(cfg, monkeypatch):
    """the one-call chain can hand back the partition classes too (int32 or int16 residue)"""
    name, setup, ctx, o, enc, _ = cfg
    monkeypatch.setenv("VB200_CHUNK_BLOCKS", "2")
    desc = make_desc(enc, "L")
    want = o.encode_dsp(1, enc["L_pcm"], desc)
    wcls = o.residue_classify(1, want["iwork"], want["nonzero"])
    got = ctx.encode_dsp(1, enc["L_pcm"], desc, classes=True)
    assert np.array_equal(got["classes"], wcls) and np.array_equal(got["iwork"], want["iwork"])
    if not (setup.channels & (setup.channels - 1)):
        got = ctx.encode_dsp(1, enc["L_pcm"], desc, classes=True, iwork_s16=True)
        assert np.array_equal(got["classes"], wcls)


def test_encode_dsp_class_stride_refused(cfg, monkeypatch):
    """the pipelined host form refuses a class_stride below partvals inside the first chunk's chain, after that
    chunk's copies in are queued; the same call on the same context with the right stride then gives what a fresh
    context gives"""
    name, setup, ctx, o, enc, _ = cfg
    monkeypatch.setenv("VB200_CHUNK_BLOCKS", "1")                      # one block per chunk: 2 to 5 chunks
    W, ch = 1, setup.channels
    n = setup.blocksize(W) // 2
    desc = make_desc(enc, "L")
    fresh = vlib.Context(setup)
    try:
        want = fresh.encode_dsp(W, enc["L_pcm"], desc, classes=True)
    finally:
        fresh.close()
    pv = ctx.residue_partvals(W)
    assert pv > 1
    io, ns, bps, keep = ctx._encode_io(W, enc["L_pcm"], desc, None, 0, 0, None, None)
    nb = ns * bps
    got = {"posts": np.zeros((nb, ch, abi.FLOOR1_STRIDE), np.int32), "nonzero": np.zeros((nb, ch), np.int32),
           "iwork": np.zeros((nb, ch, n), np.int32), "ampmax_out": np.zeros(nb, np.float32),
           "classes": np.full((nb, ch, pv), -1, np.int32)}
    for k, v in got.items():
        setattr(io, k, v.ctypes.data)
    io.class_stride = pv - 1
    assert ctx.L.vb200_encode_dsp(ctx.h, W, ns, bps, 7, C.byref(io)) == -131          # VB200_EINVAL
    assert "class_stride < partvals" in (ctx.L.vb200_last_error() or b"").decode()
    io.class_stride = pv
    assert ctx.L.vb200_encode_dsp(ctx.h, W, ns, bps, 7, C.byref(io)) == 0
    for k in ("posts", "nonzero", "iwork", "classes"):
        assert np.array_equal(got[k], want[k]), k
    assert_bits_equal(got["ampmax_out"], want["ampmax_out"], "ampmax_out")


def test_encode_dsp_dev_split_half_batches(cfg):
    """vb200_encode_dsp_dev from 2048 blocks up runs as two concurrent half-batches of whole streams (here 341 and
    342 streams of 3 blocks): int16 stream PCM in, the partition classes out, same results"""
    import torch
    name, setup, ctx, o, _, _ = cfg
    W = 1
    N, ch = setup.blocksize(W), setup.channels
    n, hop, ns, bps = N // 2, N // 2, 683, 3
    stride = (bps - 1) * hop + N
    rng = np.random.default_rng(31)
    s16 = np.clip(7000 * rng.standard_normal((ns, stride, ch)), -32768, 32767).astype(np.int16)
    planar = np.ascontiguousarray((s16.astype(np.float32) / np.float32(32768.0)).transpose(0, 2, 1))
    blocks = np.stack([planar[s, :, k * hop:k * hop + N] for s in range(ns) for k in range(bps)])
    desc = np.zeros(ns * bps, abi.BLOCKDESC_DTYPE)
    desc["lW"] = 1; desc["nW"] = 1; desc["blocktype"] = rng.integers(0, 2, ns * bps)
    amp0 = rng.uniform(-30, -3, ns).astype(np.float32)
    want = o.encode_dsp(W, blocks, desc, streams=(ns, bps), ampmax0=amp0)
    wcls = o.residue_classify(W, want["iwork"], want["nonzero"])
    dev = torch.device("cuda")
    nb = ns * bps
    t = {"pcm": torch.from_numpy(s16).to(dev),
         "desc": torch.from_numpy(desc.view(np.uint8).reshape(-1, 16).copy()).to(dev),
         "ampmax0": torch.from_numpy(amp0).to(dev),
         "posts": torch.zeros((nb, ch, abi.FLOOR1_STRIDE), dtype=torch.int32, device=dev),
         "nonzero": torch.zeros((nb, ch), dtype=torch.int32, device=dev),
         "iwork": torch.zeros((nb, ch, n), dtype=torch.int32, device=dev),
         "ampmax_out": torch.zeros(nb, device=dev),
         "classes": torch.zeros((nb, ch, ctx.residue_partvals(W)), dtype=torch.int32, device=dev)}
    io = abi.EncodeIO()
    for k, v in t.items():
        setattr(io, k, v.data_ptr())
    io.pcm_fmt, io.hop, io.stream_stride, io.class_stride = vlib.PCM_S16_INTERLEAVED, hop, stride, ctx.residue_partvals(W)
    ctx.encode_dsp_dev(W, ns, bps, io, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = {k: t[k].cpu().numpy() for k in ("posts", "nonzero", "iwork", "ampmax_out")}
    _enc_compare(got, want, "split halves")
    assert np.array_equal(t["classes"].cpu().numpy(), wcls)


# ---- whole streams through the batch path (SURVEY §8 a12, a15) -----------------------------------------------
def streams_signals(ch, rate, q):
    from test_plan_vs_ref import burst_signal
    return [probe_signal(ch, rate, 1.2, 11), burst_signal(ch, rate, 0.9, 5), burst_signal(ch, rate, 1.4, 9)]


@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_encode_streams_mixed_block_sizes(cfg, fmt):
    """vb200_encode_streams: envelope search, block planning (lib/block.c:556-615), both block sizes and the
    ampmax chain across sizes in ONE call.  f32: every block's W/lW/nW/blocktype/position, posts, nonzero and
    quantised residue must equal what the UNMODIFIED reference produced for the same streams through its public
    API (the timeline is the reference's own v->pcm: pre-extrapolated preamble, input, EOF tail; stored under
    tests/golden/ref by tests/golden/make_golden_ref.py).  s16: the same call on int16 timelines against the
    oracle's composition."""
    import refgold
    name, setup, ctx, o, _, _ = cfg
    rec = refgold.load("streams_" + name)
    caps = []
    for i, s in enumerate(streams_signals(*REF_ARGS[name])):
        p = "s%d_" % i
        c = {k: rec[p + k] for k in ("W", "lW", "nW", "blocktype", "nonzero_out", "enc_posts", "ampmax_out",
                                     "d_blocks", "d_iwork_blocks")}
        c["nblocks"], c["eof"], c["timeline"] = int(rec[p + "nblocks"]), int(rec[p + "eof"]), refgold.timeline(rec, s, p)
        caps.append(c)
    ch = setup.channels
    stride = (max(c["timeline"].shape[1] for c in caps) + 3) & ~3
    tl = np.zeros((len(caps), ch, stride), np.float32)
    for i, c in enumerate(caps):
        tl[i, :, :c["timeline"].shape[1]] = c["timeline"]
    pcm_len = np.array([c["timeline"].shape[1] for c in caps], np.int64)
    eof = np.array([c["eof"] for c in caps], np.int64)
    if fmt == "f32":
        got = ctx.encode_streams(tl, pcm_len, eof)
    else:
        s16 = np.clip(np.rint(tl * 32767.0), -32768, 32767).astype(np.int16)
        tl = s16.astype(np.float32) / np.float32(32768.0)
        got = ctx.encode_streams(np.ascontiguousarray(s16.transpose(0, 2, 1)), pcm_len, eof, fmt=vlib.PCM_S16_INTERLEAVED)
    nshort = 0
    for i, c in enumerate(caps):
        if fmt == "f32":
            k = c["nblocks"]
            want_plan = {nm: c[nm][:k] for nm in ("W", "lW", "nW", "blocktype")}
        else:
            wplan, wouts = o.encode_stream(tl[i], int(pcm_len[i]), int(eof[i]))
            k = len(wplan)
            want_plan = {nm: wplan[nm] for nm in ("W", "lW", "nW", "blocktype")}
        assert got["nblocks"][i] == k, "stream %d: %d blocks, want %d" % (i, got["nblocks"][i], k)
        plan = got["plan"][i, :k]
        for nm in ("W", "lW", "nW", "blocktype"):
            assert np.array_equal(plan[nm], want_plan[nm]), "stream %d %s" % (i, nm)
        if fmt == "f32":
            blocks = [tl[i][:, p:p + setup.blocksize(int(w))].ravel() for p, w in zip(plan["pos"], plan["W"])]
            refgold.assert_digest(np.concatenate(blocks), c["d_blocks"], "stream %d block positions" % i)
        for b in range(k):
            W, slot = int(plan[b]["W"]), int(plan[b]["slot"])
            n = setup.blocksize(W) // 2
            nshort += W == 0
            g = got[W]
            if fmt == "f32":
                assert np.array_equal(g["nonzero"][slot], c["nonzero_out"][b]), "stream %d block %d nonzero" % (i, b)
                for cc in range(ch):
                    if c["enc_posts"][b][cc][0] >= 0:
                        Pc = setup.floor_posts(W, setup.floor_of(W, cc))
                        assert np.array_equal(g["posts"][slot][cc][:Pc], c["enc_posts"][b][cc][:Pc]), "stream %d block %d posts" % (i, b)
                refgold.assert_digest(g["iwork"][slot], c["d_iwork_blocks"][b], "stream %d block %d residue" % (i, b))
                assert g["ampmax_out"][slot] == c["ampmax_out"][b]
            else:
                w = wouts[b]
                assert np.array_equal(g["posts"][slot], w["posts"][0]) and np.array_equal(g["nonzero"][slot], w["nonzero"][0])
                assert np.array_equal(g["iwork"][slot], w["iwork"][0]), "stream %d block %d residue" % (i, b)
    assert nshort >= 10                                       # the streams really mix the two sizes
    assert got["count"][0] == nshort


def test_plan_blocks_device_vs_oracle(cfg):
    """vb200_plan_blocks (k_plan_blocks) against the oracle's restatement on random mark patterns with and without EOF"""
    name, setup, ctx, o, _, _ = cfg
    rng = np.random.default_rng(77)
    ns, nsteps = 24, 900
    mark = (rng.uniform(0, 1, (ns, nsteps + 4)) < rng.uniform(0.0, 0.08, (ns, 1))).astype(np.int32)
    mark[:, nsteps:] = 0
    pcm_len = np.full(ns, 64 * (nsteps + 4), np.int64) + rng.integers(0, 64, ns)
    eof = np.where(np.arange(ns) % 3 == 0, 0, pcm_len - 3 * setup.blocksize(1) - rng.integers(0, 500, ns)).astype(np.int64)
    want, wn = o.plan_blocks(mark, nsteps, pcm_len, eof, max_blocks=600)
    got, gn = ctx.plan_blocks(mark, nsteps, pcm_len, eof, max_blocks=600)
    assert np.array_equal(gn, wn) and wn.min() > 20
    for s in range(ns):
        for nm in ("pos", "W", "lW", "nW", "blocktype", "slot"):
            assert np.array_equal(got[s, :wn[s]][nm], want[s, :wn[s]][nm]), "stream %d %s" % (s, nm)
