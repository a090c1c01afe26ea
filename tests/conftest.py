import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")
CONFIG_NAMES = ["44k_stereo_q5", "44k_stereo_q1", "44k_mono_q4", "22k_mono_q3", "48k_6ch_q2"]
REF_ARGS = {  # the vorbis_encode_init_vbr arguments each fixture was generated with
    "44k_stereo_q5": (2, 44100, 0.5),
    "44k_stereo_q1": (2, 44100, 0.1),
    "44k_mono_q4": (1, 44100, 0.4),
    "22k_mono_q3": (1, 22050, 0.3),
    "48k_6ch_q2": (6, 48000, 0.2),
}


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def bits(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.float32:
        return a.view(np.uint32)
    return a


def assert_bits_equal(a, b, what=""):
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    bad = bits(a) != bits(b)
    if bad.any():
        idx = np.argwhere(bad)[0]
        raise AssertionError("%s: %d of %d values differ; first at %s: %r vs %r"
                             % (what, int(bad.sum()), a.size, tuple(idx), a[tuple(idx)], b[tuple(idx)]))


def load_setup(name):
    from vorbis_b200 import abi
    return abi.SetupHolder.load(os.path.join(GOLDEN, "setup_%s.npz" % name))


def load_npz(kind, name):
    with np.load(os.path.join(GOLDEN, "%s_%s.npz" % (kind, name))) as z:
        return {k: z[k] for k in z.files}


def make_desc(enc, tag, sel=None):
    from vorbis_b200 import abi
    n = len(enc[tag + "_W"])
    sel = np.arange(n) if sel is None else sel
    d = np.zeros(len(sel), abi.BLOCKDESC_DTYPE)
    d["lW"] = enc[tag + "_lW"][sel]
    d["nW"] = enc[tag + "_nW"][sel]
    d["blocktype"] = enc[tag + "_blocktype"][sel]
    d["ampmax"] = enc[tag + "_ampmax_in"][sel]
    return d


def probe_signal(ch, rate, secs, seed):
    rng = np.random.default_rng(seed)
    ns = int(rate * secs)
    t = np.arange(ns)
    pcm = np.stack([0.25 * rng.uniform(-1, 1, ns) + 0.5 * np.sin(2 * np.pi * (440 + 110 * c) * t / rate)
                    for c in range(ch)]).astype(np.float32)
    a = ns // 2
    pcm[:, a:a + 300] *= 0.01
    pcm[:, a + 300:a + 400] = rng.uniform(-0.9, 0.9, (ch, 100)).astype(np.float32)
    return pcm


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def cuda_ok():
    from vorbis_b200 import lib
    L = lib.load()
    if L.vb200_device_count() < 1:
        pytest.fail("gpu test selected but no CUDA device is visible")
    return True
