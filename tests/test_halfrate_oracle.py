"""Half-rate decode (vorbis_synthesis_halfrate, lib/synthesis.c:166-174): the oracle's mdct_backward at N/2 and
the overlap-add with the windows of the halved block sizes (oracle/vb_oracle_halfrate.c) against what the
reference's own decoder returns.  Bit-exact.  The inputs are the real streams behind tests/golden/decode_<cfg>.npz
(the spectra entering mdct_backward over a window of mixed long and short blocks); the reference's half-rate PCM
of the same blocks and its two half windows are stored in tests/golden/ref/halfrate/halfrate.npz
(tests/golden/make_golden_halfrate.py).  Where the reference is built it is also run live and must give the
stored results."""
import os
import sys

import numpy as np
import pytest

from conftest import CONFIG_NAMES, GOLDEN, assert_bits_equal, load_npz, load_setup
from oracle import halfrate
from vorbis_b200 import abi, lib as vlib

FIXTURE = os.path.join(GOLDEN, "ref", "halfrate", "halfrate.npz")


def load_halfrate(name):
    """the stored reference results of config `name`: W, pcm, halfrate_window0, halfrate_window1"""
    p = name + "__"
    with np.load(FIXTURE) as z:
        return {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def halfrate_setup(name):
    """the fixture's setup with the reference's half windows of blocksizes[w]/2 (SetupHolder.halfrate_windows)"""
    rec = load_halfrate(name)
    arrays = dict(load_setup(name).arrays)
    for w in (0, 1):
        arrays["halfrate_window%d" % w] = rec["halfrate_window%d" % w]
    return abi.SetupHolder(arrays), rec


def finished_halfrate(W, bs):
    """samples block k of the sequence W finishes at half rate: (bs[lW]/4 + bs[W]/4) >> 1 (lib/block.c:840-842)"""
    fin = np.zeros(len(W), np.int64)
    for k in range(1, len(W)):
        fin[k] = (bs[W[k - 1]] // 4 + bs[W[k]] // 4) >> 1
    return fin


def reference_halfrate(name):
    """Run the reference: encode the signal of tests/golden/make_golden.py, decode its packets after
    vorbis_synthesis_halfrate(vi, 1), and cut out the blocks of the fixture decode_<name>.npz."""
    sys.path.insert(0, GOLDEN)
    import make_golden
    ch, rate, q, secs = make_golden.CONFIGS[name][:4]
    pcm = make_golden.signal(ch, rate, secs, seed=1234)
    if name == "44k_mono_q4":
        pcm[:, :3000] = 0
    dec = load_npz("decode", name)
    bs = [int(b) for b in dec["bs"]]
    d = halfrate.ref_decode(halfrate.ref_encode(ch, rate, q, pcm), bs, ch, pcm.shape[1] + 4 * bs[1])
    Wd = d["W"]
    sh = np.where(Wd == 0)[0]
    k0 = max(0, int(sh[0]) - 3) if len(sh) else 0                # the window make_golden.py kept
    k1 = min(len(Wd), k0 + 14)
    assert np.array_equal(Wd[k0:k1], dec["W"]), "block flags of the fixture's window"
    fin = finished_halfrate(Wd, bs)
    start, stop = int(fin[:k0 + 1].sum()), int(fin[:k1].sum())
    return {"W": Wd[k0:k1], "pcm": d["pcm"][:, start:stop],
            "halfrate_window0": d["window0"], "halfrate_window1": d["window1"]}


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_oracle_halfrate_decode_equals_reference(name):
    setup, rec = halfrate_setup(name)
    dec = load_npz("decode", name)
    bs = [setup.blocksize(0), setup.blocksize(1)]
    assert set(dec["W"].tolist()) == {0, 1}, "the window mixes long and short blocks"
    assert np.array_equal(rec["W"], dec["W"])
    for w in (0, 1):
        assert rec["halfrate_window%d" % w].shape == (bs[w] // 4,)
    o = halfrate.Oracle.create(setup, setup.halfrate_windows())
    Wseq = dec["W"][None, :]
    coef_off, pcm_off, coef_len, pcm_len = vlib.synthesis_layout(Wseq, bs, setup.channels, halfrate=True)
    assert coef_len == dec["coef"].size
    got = o.synthesis(Wseq, coef_off, dec["coef"], pcm_off, pcm_len)[0]
    assert got.shape == rec["pcm"].shape and got.shape[1] == dec["pcm"].shape[1] // 2
    assert_bits_equal(got, rec["pcm"], "half-rate pcm")


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_reference_halfrate_live(name):
    """the stored half-rate results are what the reference computes (needs oracle/_ref)"""
    if not halfrate.ref_available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    _, rec = halfrate_setup(name)
    live = reference_halfrate(name)
    for k, v in live.items():
        assert_bits_equal(v, rec[k], k)


def decode_only_setup(bs0):
    """the 44.1 kHz mono setup reduced to what a decoder needs, with blocksizes (bs0, 512)"""
    arrays = {k: v for k, v in load_setup("44k_mono_q4").arrays.items()
              if not k.startswith(("psy", "floor1_", "window", "residue_", "chmux", "submaps"))}
    arrays["blocksizes"] = np.array([bs0, 512], np.int32)
    arrays["n_psy"] = np.int32(0)
    return abi.SetupHolder(arrays)


def test_oracle_halfrate_refuses_64_sample_blocks():
    """vorbis_synthesis_halfrate returns -1 when blocksizes[0] <= 64; 128 is the smallest it takes"""
    assert halfrate.Oracle.create(decode_only_setup(64)) is None
    o = halfrate.Oracle.create(decode_only_setup(128))
    assert o is not None
    assert o.mdct_backward(0, np.ones((1, 32), np.float32)).shape == (1, 64)
