"""Stored results of the reference for the tests that compare the oracle with it.

Written by tests/golden/make_golden_ref.py to tests/golden/ref/<group>[-<i>].npz, keys "<case>__<name>".
Oracle inputs are stored whole (block PCM as the stream buffer's extrapolated preamble and tail around the
test's own signal); arrays that are only compared are stored as a SHA-256 of dtype, shape and bytes."""
import hashlib
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REF = os.path.join(GOLDEN, "ref")
FIXTURE_OF = {(2, 44100, 0.5): "44k_stereo_q5", (2, 44100, 0.1): "44k_stereo_q1", (1, 44100, 0.4): "44k_mono_q4",
              (1, 22050, 0.3): "22k_mono_q3", (6, 48000, 0.2): "48k_6ch_q2"}


def case_id(ch, rate, q):
    return "ch%d_%d_q%g" % (ch, rate, q)


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(("%s%s" % (a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return h.hexdigest()


def assert_digest(got, want, what):
    assert digest(got) == str(want), "%s differs from the reference" % what


def load_setup(ch, rate, q):
    """the tables of vorbis_encode_init_vbr(ch, rate, q): a fixture of tests/golden, else stored with the results"""
    from vorbis_b200 import abi
    name = FIXTURE_OF.get((ch, rate, q))
    if name:
        return abi.SetupHolder.load(os.path.join(GOLDEN, "setup_%s.npz" % name))
    return abi.SetupHolder(load("setup_" + case_id(ch, rate, q)))


def load(name):
    """the stored results of case `<group>_<case>`"""
    group, case = name.split("_", 1)
    p = case + "__"
    for f in [group + ".npz"] + sorted(f for f in os.listdir(REF) if f.startswith(group + "-")):
        with np.load(os.path.join(REF, f)) as z:
            rec = {k[len(p):]: z[k] for k in z.files if k.startswith(p)}
        if rec:
            return rec
    raise KeyError(name)


def timeline(rec, pcm, prefix=""):
    """the reference's stream buffer v->pcm: preamble, the input, end-of-stream tail"""
    return np.concatenate([rec[prefix + "tl_pre"], pcm, rec[prefix + "tl_post"]], axis=1)


def blocks(rec, tl, bs, idx, prefix=""):
    """[len(idx)][ch][N] PCM of the blocks idx (all of one size) as the API loop handed them to mapping0_forward"""
    W, pos = rec[prefix + "W"], rec[prefix + "pos"]
    return np.stack([tl[:, pos[b]:pos[b] + bs[W[b]]] for b in idx]).astype(np.float32)


def desc(rec, idx, prefix=""):
    from vorbis_b200 import abi
    d = np.zeros(len(idx), abi.BLOCKDESC_DTYPE)
    for k in ("lW", "nW", "blocktype"):
        d[k] = rec[prefix + k][idx]
    d["ampmax"] = rec[prefix + "ampmax_in"][idx]
    return d
