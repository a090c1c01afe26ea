"""The oracle's transforms at every block size the library accepts (64 ... 8192) against float64 direct formulas.

vorbisenc only produces 256/2048 and 512/4096 block pairs (and single-size setups).  Streams with hand-written setup
headers drive the reference at every size: tests/test_generated_setups_oracle.py pins the oracle's decode (inverse MDCT,
windows, overlap-add) to the stock decoder bit for bit from 64 to 8192.  Here the oracle's mdct_forward,
mdct_backward and drft_forward (float32, the reference's own arithmetic) are compared with the textbook transforms
evaluated in float64.  The error bound is calibrated at N = 2048, where the oracle is pinned to the reference bit for
bit: the float32 rounding error measured there, times a small factor, grows with log2 N.  An indexing or twiddle mistake
at any size gives errors of the order of the signal and fails by many orders of magnitude.
tests/test_gpu_long_blocks.py holds the device's transforms to the same bound (with the checks of
tests/setup_families.py)."""
import numpy as np
import pytest

from conftest import load_setup
from vorbis_b200 import abi

SIZES = [(64, 8192), (128, 4096), (256, 2048)]
SLACK = 4.0                                   # allowed multiple of the calibrated error, per log2 N / 11


def _decode_only_setup(bs0, bs1):
    """the 44.1 kHz mono setup reduced to what the transforms and a decoder need, with blocksizes (bs0, bs1)"""
    arrays = {k: v for k, v in load_setup("44k_mono_q4").arrays.items()
              if not k.startswith(("psy", "floor1_", "window", "residue_", "chmux", "submaps"))}
    arrays["blocksizes"] = np.array([bs0, bs1], np.int32)
    arrays["n_psy"] = np.int32(0)
    return abi.SetupHolder(arrays)


def _mdct_matrix(N):
    n = np.arange(N)[:, None]
    k = np.arange(N // 2)[None, :]
    return np.cos(2 * np.pi / N * (n + 0.5 + N / 4) * (k + 0.5))


def _fp64_mdct_forward(x):
    """[nvec][N] -> [nvec][N/2]; libvorbis scales the forward transform by 4/N"""
    N = x.shape[1]
    return (4.0 / N) * (x.astype(np.float64) @ _mdct_matrix(N))


def _fp64_mdct_backward(X):
    """[nvec][N/2] -> [nvec][N], unscaled"""
    return X.astype(np.float64) @ _mdct_matrix(2 * X.shape[1]).T


def _fp64_drft_forward(x):
    """FFTPACK's real forward transform layout: r0, r1, i1, r2, i2, ..., r(N/2)"""
    N = x.shape[1]
    F = np.fft.rfft(x.astype(np.float64), axis=1)
    out = np.empty((x.shape[0], N))
    out[:, 0] = F[:, 0].real
    out[:, 1:N - 1:2] = F[:, 1:N // 2].real
    out[:, 2:N - 1:2] = F[:, 1:N // 2].imag
    out[:, N - 1] = F[:, N // 2].real
    return out


def _rel_err(got, want):
    return float(np.abs(got.astype(np.float64) - want).max() / np.abs(want).max())


def _inputs(N, nvec=6, seed=0):
    rng = np.random.default_rng(seed + N)
    x = rng.uniform(-1, 1, (nvec, N)).astype(np.float32)
    y = rng.uniform(-1, 1, (nvec, N // 2)).astype(np.float32)
    return x, y


def _errors(xf, N, x, y, W):
    """relative max errors of (mdct_forward, mdct_backward, drft_forward) of the transform object xf at size W"""
    return (_rel_err(xf.mdct_forward(W, x), _fp64_mdct_forward(x)),
            _rel_err(xf.mdct_backward(W, y), _fp64_mdct_backward(y)),
            _rel_err(xf.drft_forward(W, x), _fp64_drft_forward(x)))


def _bounds(oracle_lib):
    """per transform: the oracle's error at N = 2048 (where it is pinned to the reference) times SLACK"""
    o = oracle_lib.Oracle(_decode_only_setup(256, 2048))
    cal = _errors(o, 2048, *_inputs(2048), 1)
    assert all(0 < e < 1e-5 for e in cal), cal
    return lambda N: [SLACK * e * np.log2(N) / 11.0 for e in cal]


@pytest.mark.parametrize("bs", SIZES, ids=lambda b: "%d_%d" % b)
def test_oracle_transforms_vs_fp64(oracle_lib, bs):
    bound = _bounds(oracle_lib)
    o = oracle_lib.Oracle(_decode_only_setup(*bs))
    for W in (0, 1):
        N = bs[W]
        errs = _errors(o, N, *_inputs(N), W)
        for name, e, b in zip(("mdct_forward", "mdct_backward", "drft_forward"), errs, bound(N)):
            assert e <= b, "%s N=%d: relative error %.3g over the bound %.3g" % (name, N, e, b)


def test_fp64_check_catches_an_indexing_error(oracle_lib):
    """the bound is far below what a wrong index gives: one swapped pair of outputs fails it"""
    bound = _bounds(oracle_lib)
    o = oracle_lib.Oracle(_decode_only_setup(64, 8192))
    x, y = _inputs(8192)
    got = o.mdct_forward(1, x)
    got[:, [100, 101]] = got[:, [101, 100]]
    assert _rel_err(got, _fp64_mdct_forward(x)) > 1000 * bound(8192)[0]
