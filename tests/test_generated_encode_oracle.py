"""The encode side on generated Vorbis setups (tests/vorbis_gen.py), against the reference's own encoder functions on
the same headers (oracle/gen_encode.py), without a GPU:
- every corpus setup lies inside the set where libvorbis's encoder stays inside its own arrays (the checker refuses
  the rest), and the checker's books match the headers' parse (dim, entries, minval, delta, quantvals);
- the CPU oracle's floor1_fit, floor1_render and residue_classify equal floor1_fit, floor1_encode and the residue
  class functions bit for bit, on random rows and on silence, clipped rows, cliffs and rows flat to the fit's
  threshold;
- the corpus reaches what vorbisenc's setups never do (listed in test_corpus_coverage), counted in the reference's own
  run.

The corpus goes past vorbisenc's floors and books: floor multipliers 1 and 3, 2 and 65 posts, class dimensions 5-8,
non-whole, negative and huge fit thresholds, residue cascades of 8 stages, 1 and 64 partitions, stage books of dimension 1-8 with
delta > 1 and unused lattice entries."""
import numpy as np
import pytest

import vorbis_gen as G
from oracle import gen_encode as ge

# per floor: maxover, maxunder, maxerr, twofitweight, twofitatten (encoder fields the headers do not carry)
VORBISENC = (60., 30., 500., 1., 18.)


def _classmetric(rng, r):
    """classmetric1 / classmetric2 of a residue description: rising thresholds, some -1 (no limit for type 1's entropy
    test; never met for type 2's angle test)"""
    P = len(r["cascade"])
    cm = np.full((2, 64), -1, np.int32)
    cm[0, :P] = np.sort(rng.integers(0, 12, P)) * rng.integers(1, 4)
    cm[1, :P] = np.where(rng.random(P) < 0.3, -1, np.sort(rng.integers(0, 300, P)))
    return cm


def _lat(g, specs):
    """lattice stage books of (dim, quantvals, delta, sparse)"""
    return [g.lattice(*s) for s in specs]


def _e64_128_mono():
    g = G.Gen(200, (64, 128), 1)
    sb = _lat(g, [(1, 5, 1, 0.4), (2, 5, 2, 0.3), (3, 5, 3, 0.2)])
    f0 = g.floor(32, mult=1, partitions=0)                                    # 2 posts
    r0 = g.residue(1, 3, 29, 1, 3, ppw=3, stage_books=sb, cascade=[0b1, 0b11, 0b111])
    f1 = g.floor(64, mult=3, partitions=5, dims=[1, 2, 3, 4, 5], subs=[0, 1, 2, 3, 1], minus_one=True)
    sb1 = _lat(g, [(2, 3, 1, 0.3), (4, 3, 5, 0.3), (1, 9, 2, 0.5)])
    r1 = g.residue(1, 5, 61, 4, 8, ppw=2, stage_books=sb1, cascade=[0xff, 0x81, 0b1, 0b1010, 0x7f, 0, 0b11, 0x40])
    g.modes(g.mapping([f0], [r0]), g.mapping([f1], [r1]))
    return g, [(12.5, 7.25, 80., 2.5, 9.), (70000., 65536., 2000., 0., 40.)]


def _e256_2048_stereo():
    g = G.Gen(201, (256, 2048), 2)
    sb = _lat(g, [(4, 3, 4, 0.4), (5, 3, 2, 0.2), (8, 3, 1, 0.0)])
    f0 = g.floor(64, mult=2, partitions=3, dims=[6, 7, 8], subs=[3, 2, 1])    # n = 64 of a 128-line half block
    r0 = g.residue(2, 6, 250, 8, 64, ppw=1, stage_books=sb)
    f1 = g.floor(1024, mult=4, partitions=8, dims=[8, 7], subs=[3, 0], minus_one=True, pclass=[0] * 7 + [1])
    sb1 = _lat(g, [(1, 7, 3, 0.3), (2, 5, 7, 0.5), (3, 3, 1, 0.2), (4, 5, 2, 0.3), (8, 3, 2, 0.0)])
    r1 = g.residue(1, 100, 1000, 32, 5, ppw=2, stage_books=sb1, cascade=[0b101, 0b11, 0xff, 0b1, 0x90])
    g.modes(g.mapping([f0], [r0]), g.mapping([f1], [r1], coupling=[(0, 1)]))
    return g, [(20.75, -2.5, 150.5, 1.5, 3.5), VORBISENC]


def _e128_8192_3ch():
    g = G.Gen(202, (128, 8192), 3)
    sb = _lat(g, [(2, 3, 2, 0.3), (3, 5, 1, 0.3), (6, 3, 1, 0.1)])
    fa = g.floor(64, mult=2, partitions=3, dims=[2], subs=[1])
    ra = g.residue(2, 2, 126, 6, 4, ppw=3, stage_books=sb)                   # the bundle of channels 0 and 2
    fb = g.floor(64, mult=1, partitions=2, dims=[3, 4], subs=[0, 2])
    rb = g.residue(1, 0, 64, 16, 6, ppw=1, stage_books=sb)
    m0 = g.mapping([fa, fb], [ra, rb], chmux=[0, 1, 0])
    sb1 = _lat(g, [(1, 5, 4, 0.2), (2, 7, 1, 0.4), (4, 3, 3, 0.3), (7, 3, 1, 0.2)])
    fc = g.floor(4096, mult=3, partitions=6, dims=[5, 6], subs=[2, 3], minus_one=True)
    rc = g.residue(1, 37, 4000, 28, 7, ppw=2, stage_books=sb1)
    fd = g.floor(2048, mult=4, partitions=4, dims=[4, 1], subs=[1, 0])      # n = 2048 of a 4096-line half block
    rd = g.residue(2, 11, 4090, 32, 3, ppw=1, stage_books=sb1)
    fe = g.floor(4096, mult=1, partitions=2, dims=[8], subs=[3])
    re = g.residue(1, 0, 4096, 24, 12, ppw=1, stage_books=sb1)
    m1 = g.mapping([fc, fd, fe], [rc, rd, re], chmux=[2, 0, 1])
    g.modes(m0, m1)
    return g, [(4.5, 9.75, 30., 3., 6.), (60., 30., 500., 1., 18.), (100000.5, 0.5, 1e6, 6., 0.),
               (65535., 65535., 700., 0.5, 24.), (33., 66., 250., 1., 12.)]


def _e64_64_8ch():
    g = G.Gen(203, (64, 64), 8)
    sb = _lat(g, [(1, 3, 1, 0.3), (2, 3, 2, 0.3), (4, 3, 1, 0.4), (8, 3, 1, 0.0)])
    fl, rs = [], []
    for s in range(4):
        fl.append(g.floor(32, mult=s + 1, partitions=s + 1, dims=[1 + s, 8 - s], subs=[s, 3 - s]))
        t = 2 if s % 2 else 1
        rs.append(g.residue(t, s, 64 - 2 * s if t == 2 else 32 - s, 2 * (s + 1) if t == 2 else 8,
                            [1, 2, 5, 3][s], ppw=[1, 2, 1, 3][s], stage_books=sb))
    m0 = g.mapping(fl, rs, chmux=[c % 4 for c in range(8)])
    m1 = g.mapping(fl[::-1], rs[::-1], chmux=[(c + 1) % 4 for c in range(8)])
    g.modes(m0, m1)
    return g, [(8.5, 8.5, 40., 1., 18.), VORBISENC, (65536., 70000.25, 900., 2., 10.), (-0.5, 1.75, 3., 0., 30.)]


ENC = {"e64_128_mono": _e64_128_mono, "e256_2048_stereo": _e256_2048_stereo, "e128_8192_3ch": _e128_8192_3ch,
       "e64_64_8ch": _e64_64_8ch}
NAMES = sorted(ENC)

_CACHE = {}


def corpus(name):
    """(description, header packets, floor fields [floors][5], classmetric [residues][2][64]) of one setup"""
    if name not in _CACHE:
        g, ff = ENC[name]()
        d = g.d
        rng = np.random.default_rng(300 + NAMES.index(name))
        cm = np.stack([_classmetric(rng, r) for r in d["residues"]])
        hdr = (G.ident_header(d), G.comment_header(), G.setup_header(d))
        _CACHE[name] = (d, hdr, np.array(ff, np.float32), cm)
    return _CACHE[name]


def need():
    if not ge.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def encoder(name):
    d, hdr, ff, cm = corpus(name)
    return ge.Encoder(*hdr, ff, cm)


def floors_of(d, W):
    """[(submap, floor description, floor index)] of mode W"""
    m = d["mappings"][d["modes"][W][1]]
    return [(s, d["floors"][m["floor"][s]], m["floor"][s]) for s in range(m["submaps"])]


def fit_rows(rng, n, atten, rows=48):
    """(logmdct, logmask) rows for floor1_fit: random, then silence (NULL fit), everything clipped, cliffs, rows whose
    logmdct + twofitatten equals logmask (the fit's >= test on the edge) and rows just below it"""
    mask = rng.uniform(-140, 0, (rows, n)).astype(np.float32)
    mdct = (mask + rng.normal(0, 12, (rows, n))).astype(np.float32)
    mask[1] = -200.                                           # dBquant 0 everywhere: floor1_fit returns NULL
    mask[2], mdct[2] = 300., 300.                             # clipped to 1023
    x = np.arange(n)
    for r, cut in ((3, n // 3), (4, 2 * n // 3), (5, 1)):
        mask[r] = np.where(x < cut, -20., -130.)
        mdct[r] = mask[r] + np.where(x % 3 == 0, 5., -40.)
    mask[6] = rng.choice([-60., -59.5], n)
    mdct[6] = mask[6] - np.float32(atten)                     # exactly on the threshold
    mdct[7] = np.nextafter(mask[6] - np.float32(atten), np.float32(-1e9))
    mask[7] = mask[6]
    mask[8] = np.linspace(-140, -1, n)
    mdct[8] = mask[8] + np.where(x % 2, 40., -40.)
    mask[9, : n // 2], mdct[9] = -200., -200.                 # a silent half
    return mdct.astype(np.float32), mask.astype(np.float32)


def residue_rows(rng, nb, ch, n):
    """heavy-tailed quantised residue with zero runs and silent channels, and nonzero with channels left out"""
    t = rng.standard_t(1.5, (nb, ch, n)) * rng.choice([1, 4, 30], (nb, ch, 1))
    iwork = np.clip(np.round(t), -3000, 3000).astype(np.int32)
    iwork[rng.random((nb, ch, n)) < 0.3] = 0
    iwork[rng.random((nb, ch)) < 0.1] = 0
    nonzero = (rng.random((nb, ch)) < 0.7).astype(np.int32)
    nonzero[0] = 0                                            # a block with nothing to classify
    nonzero[1] = 1
    return iwork, nonzero


def post_rows(rng, d, W, nb):
    """posts at the quantised scale per (block, channel) for the channel's floor, 30% flagged unused, some silent"""
    ch = d["channels"]
    m = d["mappings"][d["modes"][W][1]]
    posts = np.zeros((nb, ch, ge.FLOOR1_STRIDE), np.int32)
    for c in range(ch):
        f = d["floors"][m["floor"][m["chmux"][c]]]
        P = 2 + sum(f["cdim"][k] for k in f["pclass"])
        v = rng.integers(0, G.QUANT_Q[f["mult"] - 1], (nb, P))
        flag = (rng.random((nb, P)) < 0.3) & (np.arange(P) >= 2)
        posts[:, c, :P] = v | (flag * 0x8000)
    posts[rng.random((nb, ch)) < 0.15] = 0
    return posts


def packet_inputs(rng, d, W, nb):
    n = d["bs"][W] // 2
    desc = np.zeros((nb, 2), np.int32)
    if W:
        desc[:] = rng.integers(0, 2, (nb, 2))
    iwork, nonzero = residue_rows(rng, nb, d["channels"], n)
    return desc, post_rows(rng, d, W, nb), nonzero, iwork


# ---- the checker and its preconditions --------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_checker_accepts_and_matches_headers(name):
    need()
    d, hdr, ff, cm = corpus(name)
    e = ge.Encoder(*hdr, ff, cm)
    try:
        assert e.refused == 0, [w for b, w in ge.REFUSED.items() if e.refused & b]
        back = G.read_setup(hdr[0], hdr[2])
        es = e.entropy()
        assert es.nbooks == len(back["books"]) and es.modebits == e.modebits == 1
        for i, b in enumerate(back["books"]):
            dim, entries, minval, delta, qv = e.book(i)
            assert (dim, entries) == (b["dim"], b["entries"]) == (es.books[i].dim, es.books[i].entries), i
            assert (minval, delta, qv) == (es.books[i].minval, es.books[i].delta, es.books[i].quantvals), i
            if b["maptype"] == 1:
                assert qv == G.maptype1_quantvals(dim, entries), i
        stage = {x for r in back["residues"] for row in r["books"] for x in row if x >= 0}
        for i in stage:                                          # the lattices the corpus writes, read back as written
            desc = d["books"][i]
            dim, entries, minval, delta, qv = e.book(i)
            assert qv ** dim == entries and qv % 2 == 1
            assert delta == desc["delta"][1] and minval == -(qv >> 1) * delta
        s = e.setup.c
        for W in (0, 1):
            for sm, f, fi in floors_of(back, W):
                F = s.floor1[W][sm]
                assert F.posts == 2 + sum(f["cdim"][k] for k in f["pclass"]) and F.mult == f["mult"]
                assert [F.maxover, F.maxunder, F.maxerr, F.twofitweight, F.twofitatten] == list(ff[fi])
                m = back["mappings"][back["modes"][W][1]]
                r, R = back["residues"][m["residue"][sm]], s.residue[W][sm]
                assert (R.type, R.begin, R.end, R.grouping, R.partitions) == \
                    (r["type"], r["begin"], r["end"], r["grouping"], len(r["cascade"]))
                assert list(R.classmetric1) == list(cm[m["residue"][sm], 0])
                assert list(R.classmetric2) == list(cm[m["residue"][sm], 1])
    finally:
        e.close()


def test_checker_refuses_outside_its_preconditions():
    """books off the lattice, a dimension-8 book with unused entries and a floor wider than the block are refused"""
    need()
    for what, bit in (("even", 4), ("walk8", 8), ("delta0", 2), ("floor", 16)):
        g, ff = _e64_128_mono()
        d = g.d
        stage = d["residues"][0]["books"][0][0]
        if what == "even":
            d["books"][stage] = G.lattice_book(g.rng, 2, 4, 1)
            d["books"][stage]["min"] = (1, 2, 788)
        elif what == "walk8":
            d["books"][stage] = G.lattice_book(g.rng, 8, 3, 1, sparse=0.1)
        elif what == "delta0":
            d["books"][stage]["delta"] = (0, 1, 786)                 # 0.25: rint gives 0
        else:
            d["floors"][0]["rangebits"] = 7                          # a 128-line floor on a 32-line half block
        cm = np.stack([_classmetric(np.random.default_rng(1), r) for r in d["residues"]])
        e = ge.Encoder(G.ident_header(d), G.comment_header(), G.setup_header(d), np.array(ff, np.float32), cm)
        try:
            assert e.refused & bit, (what, e.refused)
        finally:
            e.close()


# ---- the CPU oracle against the reference ------------------------------------------------------------------------
@pytest.fixture(scope="module", params=NAMES)
def pair(request, oracle_lib):
    need()
    e = encoder(request.param)
    assert e.refused == 0
    yield request.param, e, oracle_lib.Oracle(e.setup)
    e.close()


def test_oracle_floor_fit_and_render(pair):
    name, e, o = pair
    d = corpus(name)[0]
    for W in (0, 1):
        n = d["bs"][W] // 2
        for sm, f, fi in floors_of(d, W):
            rng = np.random.default_rng(1000 * W + 10 * sm + NAMES.index(name))
            mdct, mask = fit_rows(rng, n, corpus(name)[2][fi][4])
            want, wnz = e.fit(W, sm, mdct, mask)
            got, gnz = o.floor1_fit(W, mdct, mask, floor_sel=sm)
            assert np.array_equal(gnz, wnz), (name, W, sm)
            assert np.array_equal(got, want), (name, W, sm, np.argwhere(got != want)[:5])
            assert wnz.any() and not wnz.all()
            ref = want * wnz[:, None]
            rposts, rilog, rret, _ = e.encode(W, sm, ref)
            gposts, gilog, gnz2 = o.floor1_render(W, want, wnz, floor_sel=sm)
            assert np.array_equal(gnz2, rret), (name, W, sm)
            assert np.array_equal(gilog, rilog), (name, W, sm)
            live = rret == 1
            assert np.array_equal(gposts[live], rposts[live]), (name, W, sm)


def test_oracle_residue_classify(pair):
    name, e, o = pair
    d = corpus(name)[0]
    for W in (0, 1):
        rng = np.random.default_rng(2000 + W + 10 * NAMES.index(name))
        iwork, nonzero = residue_rows(rng, 24, d["channels"], d["bs"][W] // 2)
        stride = o.residue_partvals(W)
        want = e.classify(W, iwork, nonzero, stride)
        got = o.residue_classify(W, iwork, nonzero, stride)       # the oracle's rows start at 0, the checker's at -1
        live = want >= 0
        assert np.array_equal(got[live], want[live]), (name, W, np.argwhere((got != want) & live)[:5])
        assert not got[~live].any(), (name, W, "the oracle classified what the reference leaves out")
        assert (want >= 0).any() and (want == -1).any()


# ---- coverage ---------------------------------------------------------------------------------------------------
def _coverage():
    c = {"bs": set(), "mult": set(), "posts": set(), "narrow": 0, "cdim": set(), "subs": set(), "minus1": 0,
         "small_sub": 0, "frac": 0, "huge": 0, "maxerr": set(), "tw": set(), "ta": set(), "res_types": set(),
         "off_edge": 0, "grouping": set(), "parts": set(), "ppw": set(), "stages": 0, "stage_dims": set(),
         "delta_gt1": 0, "sparse_stage": 0, "cm_minus1": 0, "submaps": set(), "channels": set(),
         "fallback": 0, "dropped": 0, "nullfit": 0, "float_fits": 0}
    for name in NAMES:
        d, hdr, ff, cm = corpus(name)
        back = G.read_setup(hdr[0], hdr[2])
        c["bs"] |= set(back["bs"])
        c["channels"].add(back["channels"])
        e = encoder(name)
        try:
            for W in (0, 1):
                m = back["mappings"][back["modes"][W][1]]
                c["submaps"].add(m["submaps"])
                n = back["bs"][W] // 2
                for sm, f, fi in floors_of(back, W):
                    q = G.QUANT_Q[f["mult"] - 1]
                    c["mult"].add(f["mult"])
                    c["posts"].add(2 + len(f["xlist"]))
                    c["narrow"] += (1 << f["rangebits"]) < n
                    for k in set(f["pclass"]):
                        c["cdim"].add(f["cdim"][k])
                        c["subs"].add(f["csubs"][k])
                        c["minus1"] += -1 in f["subbook"][k]
                        c["small_sub"] += any(b >= 0 and back["books"][b]["entries"] < q for b in f["subbook"][k])
                    mo, mu, me, tw, ta = (float(x) for x in ff[fi])
                    whole = mo == int(mo) and mu == int(mu)
                    c["frac"] += not whole
                    c["huge"] += max(abs(mo), abs(mu)) >= 65536
                    c["maxerr"].add(me)
                    c["tw"].add(tw)
                    c["ta"].add(ta)
                    rng = np.random.default_rng(7 + sm)
                    mdct, mask = fit_rows(rng, n, ta)
                    _, nz = e.fit(W, sm, mdct, mask)
                    if not (whole and max(abs(mo), abs(mu)) < 65536):
                        c["float_fits"] += int(nz.sum())
                    r = back["residues"][m["residue"][sm]]
                    bundle = sum(1 for x in m["chmux"] if x == sm)
                    c["res_types"].add(r["type"])
                    c["off_edge"] += r["begin"] > 0 and r["end"] < n * (bundle if r["type"] == 2 else 1)
                    c["grouping"].add(r["grouping"])
                    c["parts"].add(len(r["cascade"]))
                    c["ppw"].add(back["books"][r["groupbook"]]["dim"])
                    c["stages"] = max(c["stages"], max(G.ilog(x) for x in r["cascade"]))
                    c["cm_minus1"] += bool((cm[m["residue"][sm], :, :len(r["cascade"]) - 1] == -1).any())
                    for row in r["books"]:
                        for b in row:
                            if b >= 0:
                                B = back["books"][b]
                                c["stage_dims"].add(B["dim"])
                                c["delta_gt1"] += e.book(b)[3] > 1
                                c["sparse_stage"] += B["sparse"]
                rng = np.random.default_rng(50 + W)
                e.packets(W, *packet_inputs(rng, back, W, 40))
            for k, v in e.counts().items():
                c[k] += v
        finally:
            e.close()
    return c


def test_corpus_coverage():
    need()
    c = _coverage()
    want = [("block sizes 64, 128, 256, 2048, 8192", c["bs"] >= {64, 128, 256, 2048, 8192}),
            ("floor multipliers 1-4", c["mult"] >= {1, 2, 3, 4}), ("floors of 2 and 65 posts", c["posts"] >= {2, 65}),
            ("a floor narrower than the half block", c["narrow"] > 0),
            ("class dimensions 1-8", c["cdim"] >= set(range(1, 9))), ("subclass bits 0-3", c["subs"] >= {0, 1, 2, 3}),
            ("a -1 subbook", c["minus1"] > 0), ("a subbook smaller than the floor's range", c["small_sub"] > 0),
            ("non-whole maxover / maxunder", c["frac"] > 0), ("maxover / maxunder >= 65536", c["huge"] > 0),
            ("maxerr other than 500", len(c["maxerr"] - {500.}) > 0),
            ("twofitweight other than 1 and 3", len(c["tw"] - {1., 3.}) > 0),
            ("twofitatten other than 18", len(c["ta"] - {18.}) > 0),
            ("residue types 1 and 2", c["res_types"] >= {1, 2}), ("begin and end off the block edges", c["off_edge"] > 0),
            ("grouping 1 and 32", c["grouping"] >= {1, 32}), ("1 and 64 partitions", c["parts"] >= {1, 64}),
            ("1-3 partitions per word", c["ppw"] >= {1, 2, 3}), ("a cascade of 8 stages", c["stages"] == 8),
            ("stage books of dimension 1-8", c["stage_dims"] >= set(range(1, 9))),
            ("a stage book with delta > 1", c["delta_gt1"] > 0), ("a sparse stage book", c["sparse_stage"] > 0),
            ("a classmetric of -1", c["cm_minus1"] > 0), ("several submaps", len(c["submaps"] - {1}) >= 2),
            ("1, 2, 3 and 8 channels", c["channels"] >= {1, 2, 3, 8}),
            ("fallback walks in the reference", c["fallback"] > 0),
            ("floor values the reference drops", c["dropped"] > 0),
            ("NULL fits in the reference", c["nullfit"] > 0),
            ("fits on the non-integer threshold form", c["float_fits"] > 0)]
    missing = [what for what, ok in want if not ok]
    assert not missing, "missing %s; reached %s" % (missing, c)
