"""The carried block planner on the CPU (oracle/vb_oracle_resume.c, the restatement of what
vb200_encode_streams_packets[_managed]_resume carry from call to call):
  - any cut of a timeline into calls, at any sample (inside a 64-sample step, calls with no new samples, calls cut by
    max_blocks), gives the one-shot planner's blocks, its final envelope state, and carried mark windows equal to the
    one-shot marks;
  - driven the way a stock encoder's write / blockout loop runs, the carry equals the unmodified reference's
    vorbis_dsp_state after every vorbis_analysis_blockout (base, ve->current, ve->cursor, ve->curmark, pcm_current,
    centerW, W, lW and the block's nW and blocktype), for write chunks of 64, 1000, 1024 and 4410 samples and the whole
    input.  This part needs oracle/_ref (built where the reference sources exist)."""
import numpy as np
import pytest

import refgold as G
from oracle import pyoracle
from oracle import resume as R
from test_plan_vs_ref import GRID, burst_signal, plan_signal

FIELDS = ("W", "lW", "nW", "blocktype")


def _random_timeline(ch, rate, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(rate // 20, 2 * rate))
    pcm = burst_signal(ch, rate, max(n / rate, 0.2), seed)[:, :n] if n > rate // 4 else \
        rng.uniform(-0.5, 0.5, (ch, n)).astype(np.float32)
    half = 1024
    tl = np.zeros((ch, half + n + 4 * half), np.float32)
    tl[:, half:half + n] = pcm[:, :n]
    return tl, half + n


def _cuts(rng, eof, rate):
    """increasing buffer ends up to eof: 1 sample to several seconds apart, repeats (no new samples) and cuts a few
    samples apart (inside a 64-sample step)"""
    ends, e = [], 0
    while e < eof:
        r = rng.random()
        e += 0 if r < 0.15 else int(rng.integers(1, 64)) if r < 0.4 else int(rng.integers(64, 3 * rate))
        ends.append(min(e, eof))
    return ends


def _one_shot(o, tl, eof):
    mark, nsteps = o.timeline_marks(tl[None])
    plan, nb = o.plan_blocks(mark, nsteps, [tl.shape[1]], [eof])
    _, env = o.envelope_search(tl[None], 0, nsteps)
    return plan[0, :nb[0]], mark[0], env


def _pieced(o, bs, tl, eof, ends, rng, mark):
    ch, L = tl.shape
    P = R.Planner(bs, ch)
    rows = []
    for end in ends + [L] * 200:
        if P.c.done:
            break
        base = P.c.base
        mb = int(rng.choice([1, 2, 1 << 20])) if end < L else 1 << 20
        got = P.feed(o, tl[:, base:end], end - base, eof if end == L else 0, mb)
        for b in got:
            rows.append((base + int(b["pos"]),) + tuple(int(b[f]) for f in FIELDS))
        if not P.c.done:
            # the window entries no later step can change equal the one-shot marks of the same timeline steps
            fin = max(P.c.current // 64 - 1, 0)
            assert P.c.base % 64 == 0
            s0 = P.c.base // 64
            assert np.array_equal(P.window[:fin], (mark[s0:s0 + fin] != 0).astype(np.uint8))
    assert P.c.done
    return rows, P.env


def _rows(plan):
    return [(int(b["pos"]),) + tuple(int(b[f]) for f in FIELDS) for b in plan]


def _check_cuts(args, tl, eof, seed, trials=6):
    setup = G.load_setup(*args)
    o = pyoracle.Oracle(setup)
    bs = (setup.blocksize(0), setup.blocksize(1))
    plan, mark, env = _one_shot(o, tl, eof)
    want = _rows(plan)
    rng = np.random.default_rng(seed)
    for _ in range(trials):
        rows, penv = _pieced(o, bs, tl, eof, _cuts(rng, eof, args[1]), rng, mark)
        assert rows == want
        assert np.array_equal(penv, env)


@pytest.mark.parametrize("mode", ["probe", "bursts"])
@pytest.mark.parametrize("ch,rate,q", GRID)
def test_cuts_equal_one_shot_on_plan_cases(ch, rate, q, mode):
    rec = G.load("plan_%s_%s" % (mode, G.case_id(ch, rate, q)))
    tl = G.timeline(rec, plan_signal(ch, rate, q, mode))
    _check_cuts((ch, rate, q), tl, int(rec["eof"]), seed=ch * rate)


@pytest.mark.parametrize("seed", range(6))
def test_cuts_equal_one_shot_on_random_signals(seed):
    ch, rate, q = GRID[seed % len(GRID)]
    tl, eof = _random_timeline(ch, rate, 100 + seed)
    _check_cuts((ch, rate, q), tl, eof, seed=seed, trials=4)


REF_CASES = [(2, 44100, .5, "bursts"), (1, 22050, .3, "probe"), (6, 48000, .2, "bursts")]


@pytest.mark.parametrize("chunk", [64, 1000, 1024, 4410, 0])
@pytest.mark.parametrize("ch,rate,q,mode", REF_CASES)
def test_carry_equals_reference_after_every_blockout(ch, rate, q, mode, chunk):
    if not R.ref_available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    pcm = plan_signal(ch, rate, q, mode)[:, :int(rate * 0.8)]
    cap = R.ref_resume_capture(ch, rate, q, pcm, chunk or pcm.shape[1])
    rec, tl, ends = cap["rec"], cap["timeline"], cap["write_end"]
    setup = G.load_setup(ch, rate, q)
    o = pyoracle.Oracle(setup)
    P = R.Planner((setup.blocksize(0), setup.blocksize(1)), ch)
    k = 0
    for w, end in enumerate(ends):
        eof = cap["eof"] if w == len(ends) - 1 else 0
        if not eof and end - setup.blocksize(1) // 2 <= setup.blocksize(1):
            continue        # vorbis_analysis_wrote has not extrapolated the preamble yet: no timeline to pass
        while not P.c.done:
            base = P.c.base
            got = P.feed(o, tl[:, base:end], int(end) - base, eof, 1)
            if not len(got):
                break
            assert rec["write"][k] == w, "block %d: planned after write %d, the reference after %d" % (k, w, rec["write"][k])
            now = {"base": P.c.base, "current": P.c.current, "cursor": P.c.cursor, "curmark": P.c.curmark,
                   "kept": P.c.kept, "centerW": P.c.centerW, "W": P.c.W, "lW": P.c.lW, "nW": int(got[0]["nW"]),
                   "blocktype": int(got[0]["blocktype"])}
            for f, v in now.items():
                assert v == rec[f][k], "block %d: %s %d, the reference %d" % (k, f, v, rec[f][k])
            k += 1
    assert P.c.done and k == len(rec["write"]) and (np.array(rec["W"]) == 0).sum() >= 1
