"""Couple / quantise / normalise (_vp_couple_quantize_normalize, lib/psy.c:1014-1213) on coupling maps vorbisenc never
writes, against the reference's own function, and the maps vb200_ctx_create refuses.

vorbisenc writes three maps: none, stereo (0,1) and the 5.1 map.  A vb200_setup may hold any map of up to
VB200_MAX_COUPLING steps, and so may a parsed stream.  Each row below starts from a vorbisenc setup, so that psy, the
point limits, sliding_lowpass and the point amplitudes are real, and rewrites its map on the reference encoder
(pyref.Ref.set_coupling) and so in the setup the device context is built from.  Every row exists for one structural
property of the device path, asserted in test_row_structure:

- k_cqn_fast<2> runs stereo with at most one step; the magnitude may be channel 1 (slots swapped);
- k_cqn runs everything else: two channels with two steps, any channel count up to 79 (its shared-memory columns),
  channels that are an angle in one step and a magnitude in a later one (the later step reads what the point-stereo
  branch left), repeated steps and magnitudes, long chains;
- k_cqn_nonzero propagates nonzero flags in step order (lib/psy.c:1204-1212), so a late step can reach an early pair;
- the bitrate-managed chain takes k_cqn_fast_curves<2> for stereo (1,0) and one k_cqn per curve otherwise.

CPU part (no GPU): the row structure, the CPU oracle against the reference on the stage inputs of every row, and the
refusals of vb200_ctx_create.  GPU part: the stage, the block chain and the managed chain bit for bit against the CPU
oracle and, where oracle/_ref has ref_set_coupling, against the remapped reference; the 80-channel refusal with
coupling; packets and decoding end to end.  Every part but the structure and the refusals needs oracle/_ref; the
oracle test and the end-to-end test need its coupling hooks and skip without them."""
import ctypes as C

import numpy as np
import pytest

from conftest import assert_bits_equal, load_setup, probe_signal
from oracle import pyref
from vorbis_b200 import abi, lib as vlib

EIMPL, EINVAL = -130, -131
NB = abi.PACKETBLOBS


def _chain(ch):
    return [(k, k + 1) for k in range(ch - 1)]


STEREO, MULTI3, MULTI5, MULTI8, MANY = (2, 44100, 0.5), (3, 44100, 0.4), (5, 44100, 0.9), (8, 48000, 0.3), \
    (79, 44100, 0.4)
# id, vorbisenc setup, map of W = 0, map of W = 1, the properties the row exists for
ROWS = [
    ("2ch-swapped", STEREO, [(1, 0)], [(1, 0)], {"fast2_swapped"}),
    ("2ch-two-steps", STEREO, [(0, 1), (1, 0)], [(0, 1), (1, 0)], {"kcqn_2ch", "ang_then_mag"}),
    ("2ch-repeated-step", STEREO, [(0, 1), (0, 1)], [(0, 1), (0, 1)], {"kcqn_2ch", "repeated_step"}),
    ("2ch-per-W", STEREO, [], [(1, 0)], {"per_W", "fast2_swapped"}),
    ("3ch-ang-then-mag", MULTI3, [(0, 1), (1, 2)], [(0, 1), (1, 2)], {"ang_then_mag"}),
    ("3ch-gen-a", MULTI3, [(0, 2), (2, 1)], [(0, 2), (2, 1)], {"ang_then_mag", "generated"}),
    ("3ch-gen-b", MULTI3, [(2, 0), (0, 1)], [(2, 0), (0, 1)], {"ang_then_mag", "generated"}),
    ("5ch-chain-repeated-mag", MULTI5, _chain(5) + [(1, 3)], _chain(5) + [(1, 3)], {"odd_stride", "repeated_mag"}),
    ("8ch-reverse-chain", MULTI8, _chain(8)[::-1], _chain(8)[::-1], {"reverse_chain"}),
    ("79ch-chain", MANY, _chain(79), _chain(79), {"smem_limit"}),
]
IDS = [r[0] for r in ROWS]


# ---- the structure of each row --------------------------------------------------------------------------------------
def _cqn_smem(ch):
    """shared memory of k_cqn (vb200.cu cqn_smem): 4 warps x (5 columns x 32 lines + 1 flag) per channel"""
    return 4 * (5 * ch * 32 * 4 + ch * 4)


def _ang_then_mag(m):
    return any(a == m[t][0] for s, (_, a) in enumerate(m) for t in range(s + 1, len(m)))


PROPS = {
    # k_cqn_fast<2> with the magnitude in slot 1: c0 = 1, c1 = 0
    "fast2_swapped": lambda ch, m: ch == 2 and m[1] == [(1, 0)],
    # two channels, more than one step: cqn_launch's steps <= 1 test fails, k_cqn runs at ch = 2
    "kcqn_2ch": lambda ch, m: ch == 2 and all(len(s) > 1 for s in m),
    "repeated_step": lambda ch, m: all(len(set(s)) < len(s) for s in m),
    # W = 0 uncoupled, W = 1 coupled: the maps are per block size
    "per_W": lambda ch, m: m[0] == [] and len(m[1]) > 0,
    # a channel is the angle of one step and the magnitude of a later one
    "ang_then_mag": lambda ch, m: all(_ang_then_mag(s) for s in m if s),
    # maps of the generated corpus (tests/vorbis_gen.py)
    "generated": lambda ch, m: m[1] in ([(0, 2), (2, 1)], [(2, 0), (0, 1)]),
    # an odd channel count: the shared-memory columns of k_cqn are ch * 32 words apart
    "odd_stride": lambda ch, m: ch % 2 == 1 and ch > 3,
    "repeated_mag": lambda ch, m: all(len({a for a, _ in s}) < len(s) for s in m),
    # a chain over every channel, last pair first: the nonzero flags of the last step reach step 0
    "reverse_chain": lambda ch, m: ch >= 8 and all(s == _chain(ch)[::-1] for s in m),
    # the most channels k_cqn takes (200 KiB of shared memory), with the longest chain they allow
    "smem_limit": lambda ch, m: ch == 79 and _cqn_smem(79) <= 200 * 1024 < _cqn_smem(80) and all(
        s == _chain(ch) for s in m),
}


@pytest.mark.parametrize("row", ROWS, ids=IDS)
def test_row_structure(row):
    _, args, m0, m1, props = row
    ch = args[0]
    for W, m in enumerate((m0, m1)):
        assert all(0 <= a < ch and 0 <= b < ch and a != b for a, b in m), "W=%d: a map mapping0_unpack refuses" % W
    for p in props:
        assert PROPS[p](ch, [m0, m1]), p


# ---- inputs ---------------------------------------------------------------------------------------------------------
FROMDB = np.exp(np.linspace(np.log(1.0649863e-07), 0.0, 256))   # floor1_fromdB_LOOKUP, close enough for scaling
BLOCKS_PER_CALL = 64


def stage_inputs(seed, nb, ch, n, steps):
    """(mdct, iwork, nonzero) of nb blocks: iwork holds floor indices shaped like a rendered ilogmask (piecewise linear
    and falling, clipped to 0..255, with rows all 0 and rows all 255), the MDCT is heavy-tailed around the floor with
    exact zeros, and block b's nonzero flags are all on, all off, one channel of one pair, or random (b % 4)"""
    rng = np.random.default_rng(seed)
    rows = nb * ch
    K = 8
    xs = np.sort(rng.random((rows, K)), axis=1)
    xs[:, 0], xs[:, -1] = 0.0, 1.0
    vals = rng.uniform(150, 330, (rows, 1)) - np.cumsum(rng.uniform(-25, 60, (rows, K)), axis=1)
    x = (np.arange(n) + 0.5) / n
    iw = np.stack([np.interp(x, xs[r], vals[r]) for r in range(rows)])
    iw = np.clip(np.rint(iw), 0, 255).astype(np.int32)
    pick = rng.random(rows)
    iw[pick < 0.04] = 0
    iw[pick > 0.96] = 255
    t = rng.standard_t(2.5, (rows, n)) * rng.choice([0.2, 1.0, 4.0], (rows, 1))
    mdct = (FROMDB[iw] * t).astype(np.float32)
    mdct[rng.random((rows, n)) < 0.15] = 0.0
    mdct[rng.random(rows) < 0.03] = 0.0
    nonzero = np.ones((nb, ch), np.int32)
    for b in range(nb):
        kind = b % 4
        if kind == 1:
            nonzero[b] = 0
        elif kind == 2:
            nonzero[b] = 0
            if steps:
                s = steps[rng.integers(len(steps))]
                nonzero[b, s[rng.integers(2)]] = 1
            else:
                nonzero[b, rng.integers(ch)] = 1
        elif kind == 3:
            nonzero[b] = rng.integers(0, 2, ch)
    return mdct.reshape(nb, ch, n), iw.reshape(nb, ch, n), nonzero


def chain_blocks(args, W, N, nb, seed):
    """nb independent blocks of size N cut from the probe signal (channel 1 mostly a copy of channel 0, some channels
    silent in some blocks, every channel silent in blocks 2, 7, ..) with random window flags, block types and
    ampmax"""
    ch, rate, _ = args
    rng = np.random.default_rng(seed)
    pcm = probe_signal(ch, rate, max(0.25, ((nb + 1) * N // 2 + 16) / rate), seed)
    if ch >= 2:
        pcm[1] = (0.7 * pcm[0] + 0.3 * pcm[1]).astype(np.float32)
    blocks = np.stack([pcm[:, b * N // 2:b * N // 2 + N] for b in range(nb)]).astype(np.float32)
    for b in range(nb):
        for c in range(ch):
            if (3 * b + c) % 7 == 0 or b % 5 == 2:
                blocks[b, c] = 0.0
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    if W:
        desc["lW"], desc["nW"] = rng.integers(0, 2, nb), rng.integers(0, 2, nb)
    desc["blocktype"] = rng.integers(0, 2, nb)
    desc["ampmax"] = rng.uniform(-40, -2, nb).astype(np.float32)
    return np.ascontiguousarray(blocks), desc


# ---- the remapped reference and its setup ---------------------------------------------------------------------------
def _need_ref():
    if not pyref.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def _map(setup, W):
    s = setup.c
    return [(int(s.coupling_mag[W][k]), int(s.coupling_ang[W][k])) for k in range(s.coupling_steps[W])]


def _need_hooks():
    _need_ref()
    if not pyref.coupling_hooks_available():
        pytest.skip("oracle/_ref was built from a ref_driver.c without ref_set_coupling / ref_get_headers: rebuild it")


def _set_map(setup, maps):
    s = setup.c
    for W in (0, 1):
        s.coupling_steps[W] = len(maps[W])
        for k, (m, a) in enumerate(maps[W]):
            s.coupling_mag[W][k], s.coupling_ang[W][k] = m, a


def remapped(args, maps):
    """(reference encoder, setup) of the vorbisenc setup args with the maps rewritten.  Where the reference library has
    ref_set_coupling the map is rewritten in the encoder, whose setup must then carry it; elsewhere the encoder is None
    and only the setup holds the map (what the device and the CPU oracle take)."""
    _need_ref()
    r = pyref.Ref(*args)
    if pyref.coupling_hooks_available():
        for W in (0, 1):
            r.set_coupling(W, maps[W])
        setup = r.setup()
    else:
        setup = r.setup()
        r.close()
        r = None
        _set_map(setup, maps)
    for W in (0, 1):
        assert _map(setup, W) == list(maps[W]), "W=%d: the setup does not carry the new map" % W
    return r, setup


@pytest.fixture(scope="module", params=ROWS, ids=IDS)
def row(request, oracle_lib):
    name, args, m0, m1, _ = request.param
    r, setup = remapped(args, (m0, m1))
    o = oracle_lib.Oracle(setup)
    yield {"name": name, "args": args, "maps": (m0, m1), "ref": r, "oracle": o, "setup": setup, "ch": args[0],
           "bs": [setup.blocksize(0), setup.blocksize(1)]}
    o.close()
    if r is not None:
        r.close()


def _wants(rw, method, *a):
    """[(name, result)] of the CPU oracle and, where the reference encoder carries the map, of the reference"""
    out = [("oracle", getattr(rw["oracle"], method)(*a))]
    if rw["ref"] is not None:
        out.append(("reference", getattr(rw["ref"], {"encode_dsp": "encode_dsp_batch",
                                                     "encode_dsp_managed": "encode_dsp_managed_batch"}.get(method, method))(*a)))
    return out


def _stage_cases(rw):
    """(W, blocktype, blobno, inputs) of every stage call of a row: both W, both block types, every blob"""
    ch, nb = rw["ch"], BLOCKS_PER_CALL
    for W in (0, 1):
        n = rw["bs"][W] // 2
        for bt in (0, 1):
            inputs = stage_inputs(1000 * W + 100 * bt + ch, nb, ch, n, rw["maps"][W])
            for blob in range(NB):
                yield W, bt, blob, inputs


def _check_stage(got, want, what):
    assert_bits_equal(got[0], want[0], "%s: iwork" % what)
    assert np.array_equal(got[1], want[1]), "%s: nonzero" % what


# ---- CPU: the oracle on the same rows -------------------------------------------------------------------------------
def test_oracle_stage_vs_reference(row):
    """the CPU oracle's couple/quantise/normalise equals the reference's on every row, W, block type and blob (the
    device is compared with both, so the oracle's pin reaches these maps)"""
    _need_hooks()
    o = row["oracle"]
    for W, bt, blob, (mdct, iw, nz) in _stage_cases(row):
        what = "%s W=%d bt=%d blob=%d" % (row["name"], W, bt, blob)
        _check_stage(o.couple_quantize_normalize(W, bt, blob, mdct, iw, nz),
                     row["ref"].couple_quantize_normalize(W, bt, blob, mdct, iw, nz), what)


# ---- CPU: maps the stock decoder refuses get no context -------------------------------------------------------------
REFUSED = [
    ("mag-equals-channels", "44k_stereo_q5", 1, [(2, 0)]),
    ("ang-negative", "44k_stereo_q5", 0, [(0, -1)]),
    ("mag-equals-ang", "44k_stereo_q5", 1, [(1, 1)]),
    ("valid-then-ang-equals-channels", "44k_stereo_q5", 1, [(0, 1), (0, 2)]),
    ("6ch-mag-negative", "48k_6ch_q2", 0, [(-1, 2)]),
    ("6ch-valid-then-mag-equals-ang", "48k_6ch_q2", 1, [(0, 3), (1, 2), (4, 4)]),
]


@pytest.mark.parametrize("name,setup_name,W,steps", REFUSED, ids=[r[0] for r in REFUSED])
def test_create_refuses_invalid_map(name, setup_name, W, steps):
    """the checks of mapping0_unpack (lib/mapping0.c:110-118): vb200_ctx_create returns VB200_EINVAL with
    "coupling map" and no handle, before it touches a device (so this runs anywhere the library loads)"""
    L = vlib.load()
    setup = load_setup(setup_name)
    s = setup.c
    s.coupling_steps[W] = len(steps)
    for k, (m, a) in enumerate(steps):
        s.coupling_mag[W][k], s.coupling_ang[W][k] = m, a
    h = C.c_void_p()
    rc = L.vb200_ctx_create(C.byref(s), 0, C.byref(h))
    if rc == 0:
        L.vb200_ctx_destroy(h)
    assert rc == EINVAL, "%s: rc %d" % (name, rc)
    assert h.value is None, name
    assert b"coupling map" in L.vb200_last_error()


# ---- GPU: the device against the oracle and the reference --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx(row, cuda_ok):
    c = vlib.Context(row["setup"])
    yield c
    c.close()


@pytest.mark.gpu
def test_stage_vs_reference(row, ctx):
    """vb200_couple_quantize_normalize equals the CPU oracle and the reference's _vp_couple_quantize_normalize bit for
    bit for both W, both block types and every blob (each blob has its own point limit, low-pass and point
    amplitudes)"""
    for W, bt, blob, (mdct, iw, nz) in _stage_cases(row):
        got = ctx.couple_quantize_normalize(W, bt, blob, mdct, iw, nz)
        for who, want in _wants(row, "couple_quantize_normalize", W, bt, blob, mdct, iw, nz):
            _check_stage(got, want, "%s W=%d bt=%d blob=%d vs %s" % (row["name"], W, bt, blob, who))


def _chain_counts(ch, W):
    if ch > 8:
        return (6, 3)[W]
    return (24, 12)[W]


@pytest.mark.gpu
def test_chain_vs_reference(row, ctx):
    """vb200_encode_dsp (Phase A, floor fit and render, couple/quantise/normalise) equals the CPU oracle's chain and the
    reference's own functions in mapping0_forward's order on probe blocks of both sizes: posts, nonzero and iwork"""
    for W in (0, 1):
        blocks, desc = chain_blocks(row["args"], W, row["bs"][W], _chain_counts(row["ch"], W), 40 + W)
        got = ctx.encode_dsp(W, blocks, desc)
        for who, want in _wants(row, "encode_dsp", W, blocks, desc):
            for k in ("posts", "nonzero", "iwork"):
                assert_bits_equal(got[k], want[k], "%s W=%d %s vs %s" % (row["name"], W, k, who))
        assert (got["nonzero"] == 0).any() and (got["nonzero"] == 1).any()


@pytest.mark.gpu
def test_managed_chain_vs_reference(row, ctx):
    """vb200_encode_dsp_managed equals the CPU oracle and the reference's managed mapping0_forward order for all 15
    curves: stereo (1,0) takes k_cqn_fast_curves<2>, the other rows the per-curve k_cqn fallback with its row
    offsets"""
    for W in (0, 1):
        nb = max(2, _chain_counts(row["ch"], W) // 2)
        blocks, desc = chain_blocks(row["args"], W, row["bs"][W], nb, 60 + W)
        got = ctx.encode_dsp_managed(W, blocks, desc)
        for who, want in _wants(row, "encode_dsp_managed", W, blocks, desc):
            for k in ("posts", "nonzero", "iwork"):
                assert_bits_equal(got[k], want[k], "%s W=%d managed %s vs %s" % (row["name"], W, k, who))


E2E = [("2ch-swapped", STEREO, [(1, 0)]), ("3ch-ang-then-mag", MULTI3, [(0, 1), (1, 2)])]


@pytest.mark.gpu
@pytest.mark.parametrize("name,args,steps", E2E, ids=[e[0] for e in E2E])
def test_packets_and_decode_end_to_end(cuda_ok, name, args, steps):
    """the remapped reference encoder writes the map into its setup header; vb200_encode_dsp and vb200_encode_entropy
    on its blocks give its audio packets byte for byte, and a context from vb200_vorbis_headers_parse of its headers
    decodes them as the stock decoder does, bit for bit"""
    import test_gpu_encode_packets as EP
    from oracle import decode
    from oracle.decode import Packets, META
    from test_gpu_generated_setups import _resume
    _need_hooks()
    if not decode.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ch, rate, q = args
    pcm = probe_signal(ch, rate, 0.5, seed=11)
    stock = EP._capture(ch, rate, q, pcm)[1]
    r, setup = remapped(args, (steps, steps))
    cap = r.encode_capture(pcm, fields=("pcm",))
    hdr, want = r.headers(), r.packets()
    r.close()
    pk = hdr + want
    assert len(want) == cap["nblocks"]
    assert want != stock, "the map changed nothing in the packets"
    heads = vlib.vorbis_headers(*hdr)
    for W in (0, 1):
        assert _map(heads, W) == steps, "W=%d: the setup header does not carry the map" % W
    # the entropy setup holds books, floors and residues only (struct vb200_encode_entropy_setup), none of which the
    # coupling map changes, so the driver's for the same vorbisenc arguments is the remapped encoder's
    d = EP._driver(ch, rate, q)
    ctx = vlib.Context(setup)
    try:
        es, keep = d.setup_copy()
        ctx.encode_entropy_setup(es)
        for W in (0, 1):
            sel = cap["W"] == W
            assert sel.any()
            blocks = np.ascontiguousarray(cap["pcm"][sel][:, :, :ctx.bs[W]])
            desc = EP._desc(cap, sel)
            chain = ctx.encode_dsp(W, blocks, desc)
            got = ctx.encode_entropy(W, desc, chain["posts"], chain["nonzero"], chain["iwork"])
            assert got["packets"] == [p for p, s in zip(want, sel) if s], "%s W=%d packets" % (name, W)
    finally:
        ctx.close()
        d.close()
    meta = np.zeros((len(pk), META), np.int64)
    meta[:, 1] = [len(p) for p in pk]
    meta[1:, 0] = np.cumsum(meta[:-1, 1])
    meta[3:, 2] = -1
    meta[:, 4] = np.arange(len(pk))
    p = Packets(np.frombuffer(b"".join(pk), np.uint8).copy(), meta)
    ref_pcm = decode.stock_decode(p, channels=ch)
    dctx = heads.context()
    try:
        out = _resume(dctx, p, False)
    finally:
        dctx.close()
    assert ref_pcm.shape[1] > 0 and out.shape == ref_pcm.shape
    assert_bits_equal(out, ref_pcm, "%s decode" % name)


class _Sentinel:
    """numpy, except that zeros and full hand back buffers filled with 0xA5 bytes and remember them: the outputs that
    the wrappers of vorbis_b200.lib allocate"""

    def __init__(self):
        self.made = []

    def __getattr__(self, k):
        return getattr(np, k)

    def zeros(self, shape, dtype=float, **kw):
        a = np.empty(shape, dtype)
        a.reshape(-1).view(np.uint8)[...] = 0xA5
        self.made.append(a)
        return a

    def full(self, shape, value, dtype=None, **kw):
        return self.zeros(shape, dtype if dtype is not None else np.asarray(value).dtype)

    def untouched(self):
        return all((a.reshape(-1).view(np.uint8) == 0xA5).all() for a in self.made)


@pytest.mark.gpu
def test_80_channels_coupled_refused(cuda_ok, monkeypatch):
    """80 channels with a coupling chain: k_cqn's shared memory does not reach, so every encode call returns
    VB200_EIMPL before it writes an output"""
    _need_ref()
    try:
        r = pyref.Ref(80, 44100, 0.4)
    except RuntimeError as e:
        pytest.skip("vorbisenc builds no 80-channel setup: %s" % e)
    setup = r.setup()
    r.close()
    _set_map(setup, (_chain(80), _chain(80)))
    ctx = vlib.Context(setup)
    try:
        ch, W = 80, 1
        N = ctx.bs[W]
        blocks, desc = chain_blocks((80, 44100, 0.4), W, N, 2, 80)
        mdct, iw0, nz0 = stage_inputs(80, 2, ch, N // 2, _chain(80))

        def cqn():
            iw, nz = vlib.np.zeros(iw0.shape, np.int32), vlib.np.zeros(nz0.shape, np.int32)
            ctx._chk(ctx.L.vb200_couple_quantize_normalize(ctx.h, W, 0, 7, 2, vlib._ptr(mdct), vlib._ptr(iw),
                                                           vlib._ptr(nz)))
        calls = {"couple_quantize_normalize": cqn,
                 "encode_dsp": lambda: ctx.encode_dsp(W, blocks, desc),
                 "encode_dsp_managed": lambda: ctx.encode_dsp_managed(W, blocks, desc)}
        for name, call in calls.items():
            sent = _Sentinel()
            monkeypatch.setattr(vlib, "np", sent)
            try:
                with pytest.raises(vlib.VB200Error, match="too many channels") as e:
                    call()
            finally:
                monkeypatch.setattr(vlib, "np", np)
            assert "error %d" % EIMPL in str(e.value), name
            assert sent.made and sent.untouched(), "%s wrote an output" % name
    finally:
        ctx.close()
