"""The device's floor fit, floor render, residue classification and entropy coder on generated Vorbis setups
(test_generated_encode_oracle.py's corpus), bit for bit and byte for byte against the reference's own floor1_fit,
floor1_encode, residue class functions and mapping0_forward packet writing on the same headers (oracle/gen_encode.py).

Each setup's context is made from the checker's vb200_setup (the header fields plus the encoder fields), and its
entropy setup is the product's vb200ms_entropy_setup_build of the reference's encoder.  Beyond the bit checks: the
device's packets of each setup decode to the stock decoder's PCM on a context from vb200_vorbis_headers_parse of the
same headers, the _dev forms equal the host forms, and a floor wider than the block or a residue that does not match
the context's classification setup is refused with VB200_EINVAL."""
import ctypes as C

import numpy as np
import pytest

import vorbis_gen as G
from oracle import decode
from test_generated_encode_oracle import NAMES, corpus, encoder, fit_rows, floors_of, need, packet_inputs, \
    residue_rows
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
EINVAL = -131


@pytest.fixture(scope="module", params=NAMES)
def case(request, cuda_ok):
    need()
    e = encoder(request.param)
    assert e.refused == 0
    ctx = lib.Context(e.setup)
    ctx.encode_entropy_setup(e.entropy())
    yield request.param, corpus(request.param)[0], e, ctx
    ctx.close()
    e.close()


def test_floor_fit_and_render(case):
    """vb200_floor1_fit's posts, and vb200_floor1_render's posts, ilogmask and nonzero from the reference's posts and
    from the device's own"""
    name, d, e, ctx = case
    ff = corpus(name)[2]
    for W in (0, 1):
        n = d["bs"][W] // 2
        for sm, f, fi in floors_of(d, W):
            rng = np.random.default_rng(4000 + 10 * W + sm)
            mdct, mask = fit_rows(rng, n, ff[fi][4], rows=64)
            want, wnz = e.fit(W, sm, mdct, mask)
            got, gnz = ctx.floor1_fit(W, mdct, mask, floor_sel=sm)
            what = "%s W=%d submap %d" % (name, W, sm)
            assert np.array_equal(gnz, wnz), what
            assert np.array_equal(got, want), (what, np.argwhere(got != want)[:5])
            rposts, rilog, rret, _ = e.encode(W, sm, want * wnz[:, None])
            live = rret == 1
            for src in (want, got):
                posts, ilog, nz = ctx.floor1_render(W, src, gnz, floor_sel=sm)
                assert np.array_equal(nz, rret), what
                assert np.array_equal(ilog, rilog), what
                assert np.array_equal(posts[live], rposts[live]), what


def test_residue_classify(case):
    """classes of every submap, with channels left out by nonzero inside a submap"""
    name, d, e, ctx = case
    for W in (0, 1):
        rng = np.random.default_rng(5000 + W)
        iwork, nonzero = residue_rows(rng, 32, d["channels"], d["bs"][W] // 2)
        got = ctx.residue_classify(W, iwork, nonzero)
        want = e.classify(W, iwork, nonzero, got.shape[2])      # -1: nothing classified, where the device writes 0
        live = want >= 0
        assert np.array_equal(got[live], want[live]), (name, W, np.argwhere((got != want) & live)[:5])
        assert not got[~live].any(), (name, W)
        assert live.any() and (~live).any()


def test_entropy_packets(case):
    """vb200_encode_entropy's packets and bit counts for both block sizes: heavy-tailed residue, silent channels,
    posts with unused flags, varied lW / nW"""
    name, d, e, ctx = case
    for W in (0, 1):
        rng = np.random.default_rng(6000 + W)
        desc, posts, nonzero, iwork = packet_inputs(rng, d, W, 120)
        want, left = e.packets(W, desc, posts, nonzero, iwork.copy())
        bd = np.zeros(len(desc), abi.BLOCKDESC_DTYPE)
        bd["lW"], bd["nW"] = desc[:, 0], desc[:, 1]
        got = ctx.encode_entropy(W, bd, left, nonzero, iwork)
        for i in range(len(desc)):
            assert got["packets"][i] == want[i], "%s W=%d block %d" % (name, W, i)
            assert (got["pkt_bits"][i] + 7) // 8 == len(want[i])
        assert max(len(p) for p in want) <= ctx.packet_bound(W)


def test_round_trip_decodes_like_stock(case):
    """the device's packets, in a stream of both block sizes, decode on a context from vb200_vorbis_headers_parse of
    the same headers to the stock decoder's PCM"""
    from test_gpu_generated_setups import _resume
    name, d, e, ctx = case
    rng = np.random.default_rng(7000)
    nblk = 24
    flags = [int(x) for x in rng.integers(0, 2, nblk)]
    pk = [None] * nblk
    for W in (0, 1):
        idx = [k for k in range(nblk) if flags[k] == W]
        if not idx:
            continue
        _, posts, nonzero, iwork = packet_inputs(rng, d, W, len(idx))
        bd = np.zeros(len(idx), abi.BLOCKDESC_DTYPE)
        for j, k in enumerate(idx):
            bd["lW"][j] = flags[k - 1] if k else 0
            bd["nW"][j] = flags[k + 1] if k + 1 < nblk else W
        _, posts = e.packets(W, bd, posts, nonzero, iwork.copy())
        got = ctx.encode_entropy(W, bd, posts, nonzero, iwork)
        for j, k in enumerate(idx):
            pk[k] = got["packets"][j]
    p = G.stream(d, pk, granule=False)
    want = decode.stock_decode(p, channels=d["channels"])
    hdr = corpus(name)[1]
    h = lib.vorbis_headers(*hdr)
    dctx = h.context()
    try:
        out = _resume(dctx, p, False)
        assert out.shape == want.shape and want.shape[1] > 0, name
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), name
    finally:
        dctx.close()


def test_dev_forms_equal_host_forms(cuda_ok):
    """vb200_floor1_fit_dev, vb200_residue_classify_dev and vb200_encode_entropy_dev on one setup equal the host forms"""
    import torch
    need()
    name = "e128_8192_3ch"
    d = corpus(name)[0]
    e = encoder(name)
    ctx = lib.Context(e.setup)
    try:
        ctx.encode_entropy_setup(e.entropy())
        W, ch = 1, d["channels"]
        n = d["bs"][W] // 2
        rng = np.random.default_rng(8000)
        mdct, mask = fit_rows(rng, n, 18., rows=5 * ch)
        hp, hz = ctx.floor1_fit(W, mdct, mask)
        t = {k: torch.from_numpy(v).cuda() for k, v in (("mdct", mdct), ("mask", mask))}
        dp = torch.zeros((mdct.shape[0], abi.FLOOR1_STRIDE), dtype=torch.int32, device="cuda")
        dz = torch.zeros(mdct.shape[0], dtype=torch.int32, device="cuda")
        ctx.floor1_fit_dev(W, mdct.shape[0], t["mdct"].data_ptr(), t["mask"].data_ptr(), dp.data_ptr(), dz.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(dp.cpu().numpy(), hp) and np.array_equal(dz.cpu().numpy(), hz)

        desc, posts, nonzero, iwork = packet_inputs(rng, d, W, 40)
        stride = ctx.residue_partvals(W)
        host_cls = ctx.residue_classify(W, iwork, nonzero)
        di, dn = torch.from_numpy(iwork).cuda(), torch.from_numpy(nonzero).cuda()
        dc = torch.full((len(desc), ch, stride), -1, dtype=torch.int32, device="cuda")
        ctx.residue_classify_dev(W, len(desc), di.data_ptr(), dn.data_ptr(), dc.data_ptr(), stride)
        torch.cuda.synchronize()
        assert np.array_equal(dc.cpu().numpy(), host_cls)

        bd = np.zeros(len(desc), abi.BLOCKDESC_DTYPE)
        bd["lW"], bd["nW"] = desc[:, 0], desc[:, 1]
        _, left = e.packets(W, bd, posts, nonzero, iwork.copy())
        host = ctx.encode_entropy(W, bd, left, nonzero, iwork)
        from test_gpu_encode_packets import _dev_entropy
        rc, data, bits = _dev_entropy(ctx, W, bd, left, nonzero, iwork)
        assert rc == 0 and np.array_equal(bits, host["pkt_bits"])
        for i in range(len(desc)):
            assert bytes(data[i, :(bits[i] + 7) // 8]) == host["packets"][i]
    finally:
        ctx.close()
        e.close()


def test_refusals(cuda_ok):
    """a floor wider than the block: vb200_ctx_create gives VB200_EINVAL and no context; an entropy setup whose residue
    differs from the context's classification setup: VB200_EINVAL, and the context keeps coding with the setup it had"""
    need()
    name = "e64_128_mono"
    d = corpus(name)[0]
    e = encoder(name)
    try:
        wide = abi.Setup()
        C.memmove(C.addressof(wide), C.addressof(e.setup.c), C.sizeof(wide))
        F = wide.floor1[0][0]
        F.n = F.postlist[1] = d["bs"][0]                    # twice the half block
        h = C.c_void_p()
        L = lib.load()
        assert L.vb200_ctx_create(C.byref(wide), 0, C.byref(h)) == EINVAL
        assert not h.value

        ctx = lib.Context(e.setup)
        try:
            ctx.encode_entropy_setup(e.entropy())
            rng = np.random.default_rng(9000)
            W = 1
            desc, posts, nonzero, iwork = packet_inputs(rng, d, W, 20)
            bd = np.zeros(len(desc), abi.BLOCKDESC_DTYPE)
            bd["lW"], bd["nW"] = desc[:, 0], desc[:, 1]
            want, left = e.packets(W, bd, posts, nonzero, iwork.copy())
            es = abi.EncodeEntropySetup()
            C.memmove(C.addressof(es), C.addressof(e.entropy()), C.sizeof(es))
            es.residue[W][0].begin += 1                       # no longer the context's classification setup
            assert L.vb200_encode_entropy_setup(ctx.h, C.byref(es)) == EINVAL
            got = ctx.encode_entropy(W, bd, left, nonzero, iwork)
            assert got["packets"] == want
        finally:
            ctx.close()
    finally:
        e.close()
