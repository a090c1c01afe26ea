"""The bitrate manager's restatement in the CPU oracle (vbo_bitrate_addblock) against the reference's own
vorbis_bitrate_addblock / vorbis_bitrate_flushpacket (lib/bitrate.c): the packet kept, its final length and content,
and the state after every block, over thousands of random packet-size sequences with mixed block sizes.  The
reference runs where oracle/_ref was built; the fixture tests/golden/ref/bitrate.npz carries its results to where it
was not.  No GPU."""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import bitrate as B
from vorbis_b200 import abi

FIXTURE = os.path.join(ROOT, "tests", "golden", "ref", "bitrate.npz")

CONFIGS = B.CONFIGS
size_sequences = B.size_sequences


def oracle_run(info, rate, bs, lens, W, bits, branches):
    choice, nbytes, after = [], [], []
    t = 0
    for n in lens:
        c, b, a = B.vbo_bitrate_addblock(info, rate, bs, W[t:t + n], bits[t:t + n], branches=branches)
        choice.append(c), nbytes.append(b), after.append(a)
        t += n
    return np.concatenate(choice), np.concatenate(nbytes), np.concatenate(after)


def assert_same(got, want, what):
    c, b, a = got
    wc, wb, wa = want
    assert np.array_equal(c, wc), what + ": choice"
    assert np.array_equal(b, wb), what + ": bytes"
    for f in ("avg_reservoir", "minmax_reservoir", "avgfloat", "choice"):
        assert np.array_equal(a[f], wa[f]), what + ": state " + f


@pytest.mark.skipif(not B.ref_available(), reason="oracle/_ref not built (needs the reference sources at build time)")
def test_oracle_equals_reference_lib_bitrate():
    """per configuration 600 sequences (about 15 000 blocks): choice, final length, content (the kept blob's first bytes
    then zero bytes) and state after every block equal the reference's; every branch ran"""
    rng = np.random.default_rng(2024)
    branches = np.zeros(len(B.BRANCHES), np.int64)
    for name, cf in CONFIGS.items():
        info, bs = B.ref_bitrate_info(cf)
        lens, W, bits = size_sequences(rng, 600, bs, B.target_bits(info, bs, cf.rate))
        want = B.ref_bitrate_replay(cf, lens, W, bits, seed=7)
        assert want[2].all(), name + ": the reference's packet is not the kept blob's prefix and zero padding"
        mine = oracle_run(info, cf.rate, bs, lens, W, bits, branches)
        assert_same(mine, (want[0], want[1], want[3]), name)
    for i, b in enumerate(B.BRANCHES):
        assert branches[i] > 0, "branch not reached: " + b


def test_oracle_equals_fixture():
    """the same comparison against the reference's results stored in tests/golden/ref/bitrate.npz"""
    with np.load(FIXTURE) as z:
        f = {k: z[k] for k in z.files}
    names = [str(n) for n in f["names"]]
    assert set(names) == set(CONFIGS)
    branches = np.zeros(len(B.BRANCHES), np.int64)
    for i, name in enumerate(names):
        info = B.info_from_arrays(f["info_int"][i], f["info_float"][i])
        bs, rate = [int(v) for v in f["bs"][i]], int(f["rate"][i])
        lens, W, bits = f[name + "_lens"], f[name + "_W"], f[name + "_bits"]
        want = (f[name + "_choice"], f[name + "_bytes"],
                np.ascontiguousarray(f[name + "_state"]).view(abi.BITRATE_STATE_DTYPE).reshape(-1))
        assert_same(oracle_run(info, rate, bs, lens, W, bits, branches), want, name)
    for i, b in enumerate(B.BRANCHES):
        assert branches[i] > 0, "branch not reached: " + b


def test_oracle_cut_into_pieces_equals_one_run():
    """a stream's blocks cut into pieces that carry the state along give the result of one run"""
    rng = np.random.default_rng(5)
    cf = CONFIGS["cbr_small"]
    with np.load(FIXTURE) as z:
        i = [str(n) for n in z["names"]].index("cbr_small")
        info = B.info_from_arrays(z["info_int"][i], z["info_float"][i])
        bs = [int(v) for v in z["bs"][i]]
    lens, W, bits = size_sequences(rng, 1, bs, 3000, max_len=200)
    one = B.vbo_bitrate_addblock(info, cf.rate, bs, W, bits)
    cuts = np.sort(rng.choice(np.arange(1, len(W)), 4, replace=False))
    st = np.zeros(1, abi.BITRATE_STATE_DTYPE)
    st["avg_reservoir"] = st["minmax_reservoir"] = int(info.reservoir_bits * info.reservoir_bias)
    st["avgfloat"] = abi.PACKETBLOBS // 2
    parts = [B.vbo_bitrate_addblock(info, cf.rate, bs, W[a:b], bits[a:b], state=st)
             for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(W)])]
    assert_same(tuple(np.concatenate([p[j] for p in parts]) for j in range(3)), one, "pieces")
