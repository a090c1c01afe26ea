"""The LPC extrapolation of vorbis_analysis_wrote on the CPU (oracle/vb_oracle_lpc.c, the restatement that
vb200_encode_pcm_packets[_managed] and vb200_lpc_extrapolate are checked against):
  - the filter fit and the predictor equal the reference's vorbis_lpc_from_data and vorbis_lpc_predict bit for bit,
    in coefficients and output, at orders 16 and 32 on windows of 33 to 2^20 samples of silence (the epsilon exit),
    DC, a +-1 square wave, white noise, pure sines (near-singular), noise at the 1e-40 level and an impulse;
  - the timeline built from an input and its write schedule (the preamble from the write that crossed
    blocksizes[1], the tail from the drained planner's base) equals the v->pcm a stock encoder saw, for writes of 64,
    1000, 1024 and 4410 samples and all at once, on streams of 0 samples to two seconds.
Needs oracle/_ref (built where the reference sources exist)."""
import numpy as np
import pytest

import refgold as G
from conftest import probe_signal
from oracle import lpc
from oracle import pyoracle
from oracle import resume as R

ORDERS = (16, 32)
LENGTHS = (33, 64, 65, 1000, 4096, 44101, 1 << 20)
KINDS = ("silence", "dc", "square", "noise", "sine", "tiny", "impulse")
SETUPS = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2), (2, 44100, -0.1)]
WRITES = (64, 1000, 1024, 4410, 0)


def lpc_signal(kind, n, seed=0):
    rng = np.random.default_rng(seed + n)
    t = np.arange(n)
    if kind == "silence":
        x = np.zeros(n)
    elif kind == "dc":
        x = np.full(n, 0.375)
    elif kind == "square":
        x = np.where((t // 37) % 2, 1.0, -1.0)
    elif kind == "noise":
        x = rng.uniform(-1, 1, n)
    elif kind == "sine":
        x = 0.8 * np.sin(2 * np.pi * 0.0123 * t)
    elif kind == "tiny":
        x = rng.uniform(-1, 1, n) * 1e-40
    else:
        x = np.zeros(n)
        x[n // 3] = 1.0
    return x.astype(np.float32)


def _need_ref():
    if not (lpc.ref_available() and R.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("m", ORDERS)
def test_filter_and_predictor_equal_reference(m, kind):
    _need_ref()
    for n in LENGTHS:
        x = lpc_signal(kind, n)
        c0, y0 = lpc.ref_extrapolate(x, m, 3 * 2048)
        c1, y1 = lpc.extrapolate(x, m, 3 * 2048)
        assert np.array_equal(c0.view(np.uint32), c1.view(np.uint32)), "n=%d: coefficients" % n
        assert np.array_equal(y0.view(np.uint32), y1.view(np.uint32)), "n=%d: prediction" % n
    if kind == "silence":
        assert not c1.any() and not y1.any()


def _writes(n, w):
    if not w or not n:
        return [n] if n else []
    return [w] * (n // w) + ([n % w] if n % w else [])


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_timeline_equals_stock_encoder(ch, rate, q):
    _need_ref()
    setup = G.load_setup(ch, rate, q)
    bs = (setup.blocksize(0), setup.blocksize(1))
    ora = pyoracle.Oracle(setup)
    for n in (0, 1, 32, 33, 64, 65, bs[1], bs[1] + 1, 2 * rate):
        pcm = probe_signal(ch, rate, (n + 1000) / rate, seed=n)[:, :n]
        for w in WRITES:
            cap = R.ref_resume_capture(ch, rate, q, pcm, w or max(n, 1))
            tl, eof = lpc.timeline(ora, bs, pcm, _writes(n, w))
            want = cap["timeline"]
            assert eof == cap["eof"], "n=%d w=%d: eof" % (n, w)
            assert tl.shape == want.shape, "n=%d w=%d: length" % (n, w)
            assert np.array_equal(tl.view(np.uint32), want.view(np.uint32)), "n=%d w=%d: timeline" % (n, w)
