"""k_phaseA_transform at the four block sizes it has templated instances for (256, 512, 1024, 2048), fed from every
PCM source it reads: the block layout, planar float streams and interleaved int16 streams, each stream form also
from a start that is not 16-byte aligned (the scalar load path).  The raw MDCT, the log spectrum and the block's
ampmax are compared bit for bit with the CPU oracle, on 2000 rows per size with random window shapes."""
import numpy as np
import pytest

import refgold as G
from conftest import assert_bits_equal, load_setup
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu

SETUPS = {"44k_stereo_q5": lambda: load_setup("44k_stereo_q5"),            # 256 / 2048
          "ch2_22050_q0.9": lambda: G.load_setup(2, 22050, 0.9)}           # 512 / 1024
SIZES = [(256, "44k_stereo_q5", 0), (512, "ch2_22050_q0.9", 0), (1024, "ch2_22050_q0.9", 1),
         (2048, "44k_stereo_q5", 1)]
ROWS = 2000


@pytest.fixture(scope="module")
def contexts(oracle_lib, cuda_ok):
    made = {}
    for name, load in SETUPS.items():
        setup = load()
        assert setup.channels == 2
        made[name] = (setup, vlib.Context(setup), oracle_lib.Oracle(setup))
    yield made
    for _, ctx, _ in made.values():
        ctx.close()


def _desc(rng, nb, W):
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["lW"] = rng.integers(0, 2, nb) if W else 0
    desc["nW"] = rng.integers(0, 2, nb) if W else 0
    desc["blocktype"] = desc["lW"] & desc["nW"]
    desc["ampmax"] = np.where(rng.random(nb) < 0.3, -9999.0, rng.uniform(-40, 0, nb)).astype(np.float32)
    return desc


def _check(got, want, what):
    for k in ("mdct_raw", "logfft", "ampmax_out"):
        assert_bits_equal(got[k], want[k], "%s %s" % (what, k))


@pytest.mark.parametrize("N,name,W", SIZES, ids=[str(s[0]) for s in SIZES])
def test_block_layout(contexts, N, name, W):
    setup, ctx, o = contexts[name]
    assert setup.blocksize(W) == N
    rng = np.random.default_rng(N)
    nb = ROWS // 2
    pcm = rng.uniform(-1, 1, (nb, 2, N)).astype(np.float32)
    pcm[0] = 0.0                                       # silence
    pcm[1] *= 1e-30                                    # products in the denormal range
    pcm[2, :, ::2], pcm[2, :, 1::2] = 1.0, -1.0        # alternating full scale
    desc = _desc(rng, nb, W)
    _check(ctx.phaseA(W, pcm, desc, taps=True), o.phaseA(W, pcm, desc, taps=True), "N=%d blocks" % N)


@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("shift", [0, 1], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("N,name,W", SIZES, ids=[str(s[0]) for s in SIZES])
def test_stream_sources(contexts, N, name, W, fmt, shift):
    """blocks cut on the device out of one buffer per stream (hop N/2); shift = 1 starts every stream one sample
    (float) or one frame (int16) past a 16-byte boundary"""
    import torch
    setup, ctx, o = contexts[name]
    ch, hop, ns, bps = 2, N // 2, 20, ROWS // 40
    stride = (bps - 1) * hop + N + 8
    rng = np.random.default_rng(7 * N + shift)
    s16 = np.clip(9000 * rng.standard_normal((ns, stride, ch)), -32768, 32767).astype(np.int16)
    planar = np.ascontiguousarray((s16.astype(np.float32) / np.float32(32768.0)).transpose(0, 2, 1))
    blocks = np.stack([planar[s, :, k * hop:k * hop + N] for s in range(ns) for k in range(bps)])
    desc = _desc(rng, ns * bps, W)
    want = o.phaseA(W, blocks, desc, taps=True, streams=(ns, bps))
    dev = torch.device("cuda", 0)
    d_desc = torch.from_numpy(desc.view(np.uint8).reshape(-1, 16).copy()).to(dev)
    keys = ("mdct", "logmdct", "logmask", "mdct_raw", "logfft")
    outs = {k: torch.empty((ns * bps, ch, N // 2), device=dev) for k in keys}
    d_amp = torch.empty(ns * bps, device=dev)
    io = abi.PhaseAIO()
    io.desc = d_desc.data_ptr()
    io.mdct, io.logmdct, io.logmask = (outs[k].data_ptr() for k in ("mdct", "logmdct", "logmask"))
    io.tap_mdct_raw, io.tap_logfft = outs["mdct_raw"].data_ptr(), outs["logfft"].data_ptr()
    io.ampmax_out = d_amp.data_ptr()
    if fmt == "s16":
        buf = np.zeros((ns, stride + shift, ch), np.int16)
        buf[:, shift:] = s16
        d_pcm = torch.from_numpy(buf.reshape(-1)).to(dev)
        ptr = d_pcm.data_ptr() + 2 * ch * shift
        ctx.phaseA_pcmstream_dev(W, ns, bps, ptr, vlib.PCM_S16_INTERLEAVED, stride + shift, hop, io,
                                 stream=torch.cuda.current_stream().cuda_stream)
    else:
        buf = np.zeros((ns, ch, stride + 4), np.float32)
        buf[:, :, shift:shift + stride] = planar
        d_pcm = torch.from_numpy(buf.reshape(-1)).to(dev)
        ptr = d_pcm.data_ptr() + 4 * shift
        ctx.phaseA_pcmstream_dev(W, ns, bps, ptr, vlib.PCM_F32_PLANAR, stride + 4, hop, io,
                                 stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = {k: outs[k].cpu().numpy() for k in ("mdct_raw", "logfft")}
    got["ampmax_out"] = d_amp.cpu().numpy()
    _check(got, want, "N=%d %s shift %d" % (N, fmt, shift))
