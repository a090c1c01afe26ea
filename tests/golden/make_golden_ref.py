#!/usr/bin/env python
"""Record what the reference computes for the tests that compare the oracle with it
(tests/test_oracle_vs_ref.py, tests/test_plan_vs_ref.py, tests/test_gpu_parity.py::test_encode_streams_mixed_block_sizes)
into tests/golden/ref/<group>[-<i>].npz (format: tests/refgold.py).  Needs oracle/_ref/libvorbis_ref.so, i.e. the unmodified
reference sources compiled by oracle/Makefile.

usage:  python tests/golden/make_golden_ref.py
"""
import glob
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import REF_ARGS, probe_signal  # noqa: E402
from oracle import pyoracle, pyref  # noqa: E402
from refgold import FIXTURE_OF, REF, case_id, digest  # noqa: E402
from vorbis_b200 import abi, lib as vlib  # noqa: E402
import test_oracle_vs_ref as T  # noqa: E402
import test_plan_vs_ref as P  # noqa: E402

BIG = ("mdct_raw", "logfft", "noise", "tone", "logmdct", "logmask", "mdct_m1", "ilogmask", "iwork_out")


GROUPS = {}
MAX_FILE = 640 << 10          # a group larger than this is written as <group>.npz, <group>-1.npz, ... (whole cases)


def save(name, d):
    group, case = name.split("_", 1)
    GROUPS.setdefault(group, {}).update({"%s__%s" % (case, k): v for k, v in d.items()})


def save_setup(args, r):
    if args not in FIXTURE_OF:
        save("setup_" + case_id(*args), r.setup().arrays)


def capture(args, pcm, fields=None, prefix=""):
    """encode `pcm` through the reference's API loop; returns (stored dict, raw capture, reference)"""
    ch, rate, q = args
    r = pyref.Ref(ch, rate, q)
    save_setup(args, r)
    cap = r.encode_capture(pcm, timeline=True) if fields is None else r.encode_capture(pcm, fields=fields, timeline=True)
    tl, k, half = cap["timeline"], cap["nblocks"], r.bs[1] // 2
    assert np.array_equal(tl[:, half:half + pcm.shape[1]], pcm), "input region of the stream buffer"
    o = pyoracle.Oracle(r.setup())
    mark, nsteps = o.timeline_marks(tl[None])
    plan, nb = o.plan_blocks(mark, nsteps, [tl.shape[1]], [cap["eof"]])
    assert nb[0] == k
    pos = plan[0, :k]["pos"].astype(np.int64)
    for b in range(k):
        N = r.bs[cap["W"][b]]
        assert np.array_equal(cap["pcm"][b][:, :N], tl[:, pos[b]:pos[b] + N]), "block %d position" % b
    rec = {"tl_pre": tl[:, :half], "tl_post": tl[:, half + pcm.shape[1]:], "eof": np.int64(cap["eof"]),
           "nblocks": np.int64(k), "bytes": np.int64(cap["bytes"]), "pos": pos}
    for nm in ("W", "lW", "nW", "blocktype", "ampmax_in", "ampmax_out", "nonzero_in", "nonzero_out",
               "fit_posts", "enc_posts"):
        rec[nm] = cap[nm][:k]
    rec["d_blocks"] = digest(np.concatenate([cap["pcm"][b][:, :r.bs[cap["W"][b]]].ravel() for b in range(k)]))
    for W in (0, 1):
        idx = np.where(cap["W"] == W)[0]
        n = r.bs[W] // 2
        for nm in BIG:
            if nm in cap:
                rec["d_%s_W%d" % (nm, W)] = digest(cap[nm][idx][:, :, :n])
    return {prefix + k_: v for k_, v in rec.items()}, cap, r


def pair_cases():
    for args in T.GRID:
        ch, rate, q = args
        pcm = T.pair_signal(ch, rate)
        rec, cap, r = capture(args, pcm)
        rng = np.random.default_rng(7)
        for W in (0, 1):
            for which in (0, 1, 2, 3):
                rec["d_table_W%d_%d" % (W, which)] = digest(r.table(W, which))
            x, y, lW, nW = T.transform_inputs(r.bs[W], rng)
            rec["d_mdct_forward_W%d" % W] = digest(r.mdct_forward(W, x))
            rec["d_mdct_backward_W%d" % W] = digest(r.mdct_backward(W, y))
            rec["d_drft_forward_W%d" % W] = digest(r.drft_forward(W, x))
            rec["d_window_W%d" % W] = digest(r.apply_window(W, x, lW, nW))
            idx = np.where(cap["W"] == W)[0]
            n = r.bs[W] // 2
            if len(idx):
                desc = np.zeros(len(idx), abi.BLOCKDESC_DTYPE)
                for k in ("lW", "nW", "blocktype"):
                    desc[k] = cap[k][idx]
                desc["ampmax"] = cap["ampmax_in"][idx]
                m, lmd, lmk, amp = r.phaseA_batch(W, cap["pcm"][idx][:, :, :r.bs[W]], desc)
                rec["d_batch_logmask_W%d" % W] = digest(lmk)
                rec["d_batch_mdct_W%d" % W] = digest(m)
            for bt in (0, 1):
                sel = np.where((cap["W"] == W) & (cap["blocktype"] == bt))[0]
                rec["d_iwork_out_W%d_bt%d" % (W, bt)] = digest(cap["iwork_out"][sel][:, :, :n])
        d = r.decode_capture(cap["nblocks"] + 4, pcm.shape[1] + 8192)
        Wseq = d["W"][None, :]
        pcm_len = vlib.synthesis_layout(Wseq, r.bs, ch)[3]
        m = min(d["pcm"].shape[1], pcm_len)
        rec["dec_W"] = d["W"]
        rec["dec_coef"] = np.concatenate([d["dec_coef"][k][:, :r.bs[d["W"][k]] // 2].reshape(-1)
                                          for k in range(len(d["W"]))])
        rec["dec_m"] = np.int64(m)
        rec["d_dec_pcm"] = digest(d["pcm"][:, :m])
        save("pair_" + case_id(*args), rec)
        r.close()


def floor1_cases():
    for args in T.FLOOR1_ARGS:
        rec, cap, r = capture(args, T.floor1_signal(*args))
        save("floor1_" + case_id(*args), rec)
        r.close()


def chain_cases():
    for args in T.CHAIN_ARGS:
        rec, cap, r = capture(args, T.chain_signal(*args))
        r2 = pyref.Ref(*args)
        for W in (0, 1):
            idx = np.where(cap["W"] == W)[0]
            if not len(idx):
                continue
            b = r2.encode_dsp_batch(W, np.ascontiguousarray(cap["pcm"][idx][:, :, :r.bs[W]]), _desc(cap, idx))
            for k in ("posts", "nonzero", "iwork"):
                rec["d_batch_%s_W%d" % (k, W)] = digest(b[k])
            rec["batch_ampmax_out_W%d" % W] = b["ampmax_out"]
        save("chain_" + case_id(*args), rec)
        r.close()
        r2.close()


def managed_cases():
    for args in T.MANAGED_ARGS:
        rec, cap, r = capture(args, T.managed_signal(*args))
        r2 = pyref.Ref(*args)
        for W in (0, 1):
            idx = np.where(cap["W"] == W)[0][:10]
            if not len(idx):
                continue
            b = r2.encode_dsp_managed_batch(W, np.ascontiguousarray(cap["pcm"][idx][:, :, :r.bs[W]]), _desc(cap, idx))
            for k in ("posts", "nonzero", "iwork"):
                rec["d_managed_%s_W%d" % (k, W)] = digest(b[k])
            rec["managed_ampmax_out_W%d" % W] = b["ampmax_out"]
        save("managed_" + case_id(*args), rec)
        r.close()
        r2.close()


def envelope_cases():
    for args in T.ENVELOPE_ARGS:
        r = pyref.Ref(*args)
        save_setup(args, r)
        pcm = T.envelope_signal(*args)
        marks, steps, st, stream = r.envelope_marks(pcm)
        half = r.bs[1] // 2
        assert np.array_equal(stream[:, half:], pcm)
        save("envelope_" + case_id(*args), {"marks": marks, "steps": np.int64(steps), "state": st,
                                              "stream_pre": stream[:, :half]})
        r.close()


def inverse2_cases():
    for args in T.INVERSE2_ARGS:
        r = pyref.Ref(*args)
        save_setup(args, r)
        rec = {}
        for W, (posts, present, data) in T.inverse2_inputs(args[0], r.bs):
            rec["d_inverse2_W%d" % W] = digest(r.floor1_inverse2(W, posts, present, data))
        save("inverse2_" + case_id(*args), rec)
        r.close()


def residue_cases():
    for args in T.RESIDUE_ARGS:
        r = pyref.Ref(*args)
        save_setup(args, r)
        o = pyoracle.Oracle(r.setup())
        rec = {}
        for W, (iwork, nonzero) in T.residue_inputs(args[0], r.bs):
            rec["d_classes_W%d" % W] = digest(r.residue_classify(W, iwork, nonzero, o.residue_partvals(W)))
        save("residue_" + case_id(*args), rec)
        r.close()


def plan_cases():
    for args in P.GRID:
        for mode in ("probe", "bursts"):
            rec, cap, r = capture(args, P.plan_signal(*args, mode), fields=("pcm",))
            save("plan_%s_%s" % (mode, case_id(*args)), rec)
            r.close()
    rec, cap, r = capture((1, 44100, .4), P.config1_signal(), fields=("pcm",))
    save("plan_config1", rec)
    r.close()


def streams_cases():
    import test_gpu_parity as G
    for name, args in REF_ARGS.items():
        rec = {}
        for i, s in enumerate(G.streams_signals(*args)):
            part, cap, r = capture(args, s, fields=("pcm", "iwork_out"), prefix="s%d_" % i)
            part["s%d_d_iwork_blocks" % i] = np.array([digest(cap["iwork_out"][b][:, :r.bs[cap["W"][b]] // 2])
                                                       for b in range(cap["nblocks"])])
            rec.update(part)
            r.close()
        save("streams_" + name, rec)


def _desc(cap, idx):
    desc = np.zeros(len(idx), abi.BLOCKDESC_DTYPE)
    for k in ("lW", "nW", "blocktype"):
        desc[k] = cap[k][idx]
    desc["ampmax"] = cap["ampmax_in"][idx]
    return desc


def main():
    if not pyref.available():
        sys.exit("oracle/_ref/libvorbis_ref.so is missing: build it with oracle/Makefile (target ref)")
    os.makedirs(REF, exist_ok=True)
    for f in (pair_cases, floor1_cases, chain_cases, managed_cases, envelope_cases, inverse2_cases, residue_cases,
              plan_cases, streams_cases):
        f()
        print(f.__name__, "done")
    for group, arrays in GROUPS.items():
        cases = {}
        for k, v in arrays.items():
            cases.setdefault(k.split("__", 1)[0], {})[k] = v
        # cases already stored stay in their files, which must hold exactly what was just computed; new cases go
        # to new files after the group's last one, so that adding a case never rewrites a stored fixture
        files = sorted(glob.glob(os.path.join(REF, group + ".npz")) + glob.glob(os.path.join(REF, group + "-*.npz")))
        for f in files:
            with np.load(f) as z:
                stored = {k: z[k] for k in z.files}
            for case in {k.split("__", 1)[0] for k in stored}:
                got = cases.pop(case, None)
                assert got is not None, "%s: case %s is no longer computed" % (f, case)
                want = {k: v for k, v in stored.items() if k.split("__", 1)[0] == case}
                assert got.keys() == want.keys() and all(np.array_equal(got[k], want[k]) for k in want), \
                    "%s: case %s changed" % (f, case)
        shards, cur = [], {}
        for c in cases.values():
            buf = io.BytesIO()
            np.savez_compressed(buf, **cur, **c)
            if cur and buf.tell() > MAX_FILE:
                shards.append(cur)
                cur = {}
            cur.update(c)
        first = len(files)
        for i, s in enumerate(shards + [cur] if cur else []):
            np.savez_compressed(os.path.join(REF, group + ("-%d" % (first + i) if first + i else "") + ".npz"), **s)


if __name__ == "__main__":
    main()
