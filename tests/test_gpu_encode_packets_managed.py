"""The entropy coding of bitrate-managed mapping0_forward on the device (vb200_encode_entropy_managed_dev,
vb200_encode_packets_managed and the managed multi-stream driver's device path): all 15 packets of every block against
the reference's own floor1_encode and residue class / forward on that curve's posts, nonzero flags and residue, byte for
byte.  Needs oracle/_ref (built where the reference sources exist; the libraries travel)."""
import numpy as np
import pytest

from conftest import load_setup, probe_signal
from oracle import pyref
from test_gpu_encode_packets import SETUPS, _capture, _desc, _driver, _fuzz_inputs, _need, \
    _stage0_books_with_unused_entries
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

NB, MID = abi.PACKETBLOBS, abi.PACKETBLOBS // 2
VB200_EINVAL = -131


def _dev_managed(ctx, W, desc, posts, nonzero, iwork, stride=None):
    """vb200_encode_entropy_managed_dev through torch device buffers on curve-major inputs [15][blob_blocks][...]
    (blob_blocks >= len(desc)): (rc, strided data uint8 [15][nb][stride], pkt_bits [15][nb])"""
    import torch
    nb, blob = len(desc), posts.shape[1]
    stride = ctx.packet_bound(W) if stride is None else stride
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
         (("desc", desc.view(np.uint8)), ("posts", posts), ("nz", nonzero), ("iw", iwork))}
    bits = torch.zeros(NB * nb, dtype=torch.int32, device="cuda")
    data = torch.zeros(NB * nb * stride, dtype=torch.uint8, device="cuda")
    rc = ctx.encode_entropy_managed_dev(W, nb, blob, t["desc"].data_ptr(), t["posts"].data_ptr(), t["nz"].data_ptr(),
                                        t["iw"].data_ptr(), stride, bits.data_ptr(), data.data_ptr(), check=False)
    torch.cuda.synchronize()
    return rc, data.cpu().numpy().reshape(NB, nb, stride), bits.cpu().numpy().reshape(NB, nb)


def _unpack(data, bits):
    return [[bytes(data[k, i, :(bits[k, i] + 7) // 8]) for i in range(bits.shape[1])] for k in range(NB)]


def _ref_curves(ch, rate, q, W, desc, posts, nonzero, iwork):
    """ref_packets on every curve of the first len(desc) blocks: ([15][nb] packets, the posts floor1_encode leaves
    [15][nb][ch][FLOOR1_STRIDE], stage-0 unused-entry hits)"""
    ep = _need()
    nb, n = len(desc), iwork.shape[-1]
    want, post_pass, hits = ep.ref_packets(ch, rate, q, W, np.concatenate([desc] * NB),
                                           np.ascontiguousarray(posts[:, :nb]).reshape(NB * nb, ch, abi.FLOOR1_STRIDE),
                                           np.ascontiguousarray(nonzero[:, :nb]).reshape(NB * nb, ch),
                                           np.array(iwork[:, :nb]).reshape(NB * nb, ch, n))
    return [want[k * nb:(k + 1) * nb] for k in range(NB)], post_pass.reshape(NB, nb, ch, abi.FLOOR1_STRIDE), hits


def _poisoned(x, blob, value):
    """curve-major x [15][nb][...] in a [15][blob][...] layout whose rows past nb hold value"""
    out = np.full((NB, blob) + x.shape[2:], value, x.dtype)
    out[:, :x.shape[1]] = x
    return out


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_stage_parity_captured_blocks(cuda_ok, ch, rate, q):
    """vb200_encode_dsp_managed then vb200_encode_entropy_managed_dev, and vb200_encode_packets_managed alone, on the
    stock encoder's blocks: every (curve, block) packet is the reference's on that curve; the middle curve is the stock
    encoder's audio packet and vb200_encode_packets'; pkt_bits rounds up to the length; no packet exceeds the bound"""
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        pcm = probe_signal(ch, rate, 0.5, seed=11)
        cap, want = _capture(ch, rate, q, pcm)
        for W in (0, 1):
            sel = cap["W"] == W
            if not sel.any():
                continue
            blocks = np.ascontiguousarray(cap["pcm"][sel][:, :, :ctx.bs[W]])
            desc = _desc(cap, sel)
            wp = [p for p, s in zip(want, sel) if s]
            m = ctx.encode_dsp_managed(W, blocks, desc)
            rc, data, bits = _dev_managed(ctx, W, desc, m["posts"], m["nonzero"], m["iwork"])
            assert rc == 0
            got = _unpack(data, bits)
            ref, _, _ = _ref_curves(ch, rate, q, W, desc, m["posts"], m["nonzero"], m["iwork"])
            for k in range(NB):
                assert got[k] == ref[k], "W=%d curve %d" % (W, k)
            assert got[MID] == wp
            assert got[MID] == ctx.encode_packets(W, blocks, desc)["packets"]
            assert all((bits[k, i] + 7) // 8 == len(got[k][i]) for k in range(NB) for i in range(len(desc)))
            assert max(len(p) for c in got for p in c) <= ctx.packet_bound(W)
            fused = ctx.encode_packets_managed(W, blocks, desc)
            assert fused["packets"] == got
            assert np.array_equal(fused["pkt_bits"], bits)
            assert np.array_equal(fused["ampmax_out"], m["ampmax_out"])
    finally:
        d.close()


def _fuzz_curves(rng, es, W, nb, ch, n):
    """random curves per block as _fuzz_inputs builds them, with whole curves NULL for some blocks: the 7 below the
    middle (low fit NULL), the 7 above it (high fit NULL), or all 15 (middle fit NULL)"""
    desc = None
    posts, nonzero, iwork = [], [], []
    for k in range(NB):
        dk, p, z, w = _fuzz_inputs(rng, es, W, nb, ch, n)
        desc = dk if desc is None else desc
        posts.append(p), nonzero.append(z), iwork.append(w)
    posts, nonzero, iwork = np.stack(posts), np.stack(nonzero), np.stack(iwork)
    kind = rng.integers(0, 6, nb)
    for b in range(nb):
        curves = {0: range(0, MID), 1: range(MID + 1, NB), 2: range(NB)}.get(int(kind[b]), ())
        for k in curves:
            posts[k, b], nonzero[k, b], iwork[k, b] = 0, 0, 0
    return desc, posts, nonzero, iwork


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_fuzz_against_reference_functions(cuda_ok, ch, rate, q):
    """random curves with NULL curve runs, in a layout with blob_blocks > nblocks whose pad rows hold garbage: every
    packet equals the reference's on its curve, and the fallback search of local_book_besterror ran"""
    d = _driver(ch, rate, q)
    try:
        es, keep = d.setup_copy()
        rng = np.random.default_rng(200 + ch)
        hits = 0
        for W in (0, 1):
            nb = 40 if W == 0 else 20
            desc, posts, nonzero, iwork = _fuzz_curves(rng, es, W, nb, ch, d.ctx.bs[W] // 2)
            ref, post_pass, h = _ref_curves(ch, rate, q, W, desc, posts, nonzero, iwork)
            hits += h
            blob = nb + 7
            rc, data, bits = _dev_managed(d.ctx, W, desc, _poisoned(post_pass, blob, 0x7fff7fff),
                                          _poisoned(nonzero, blob, 1), _poisoned(iwork, blob, 1 << 30))
            assert rc == 0
            got = _unpack(data, bits)
            for k in range(NB):
                for i in range(nb):
                    assert got[k][i] == ref[k][i], "W=%d curve %d block %d" % (W, k, i)
            assert max(len(p) for c in ref for p in c) <= d.ctx.packet_bound(W)
        if _stage0_books_with_unused_entries(es):
            assert hits > 0, "no residue vector landed on an unused lattice entry"
    finally:
        d.close()


def test_whole_streams(cuda_ok):
    """vb200_encode_streams_managed on 4 burst streams, then vb200_encode_entropy_managed_dev per size with
    blob_blocks = cap[W] and the pad rows poisoned: every (curve, slot) packet is the reference's, and curve 7 reordered
    by plan[].slot is every stream's stock (un-managed) packets"""
    from test_plan_vs_ref import burst_signal
    ch, rate, q = 2, 44100, 0.4
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        caps, wants = [], []
        for i in range(4):
            pcm = burst_signal(ch, rate, 0.7, 40 + i)
            ref = pyref.Ref(ch, rate, q)
            c = ref.encode_capture(pcm, fields=(), timeline=True)
            pk = ref.packets()
            ref.close()
            caps.append(c)
            wants.append(pk[len(pk) - c["nblocks"]:])
        stride = (max(c["timeline"].shape[1] for c in caps) + 3) & ~3
        tl = np.zeros((len(caps), ch, stride), np.float32)
        for i, c in enumerate(caps):
            tl[i, :, :c["timeline"].shape[1]] = c["timeline"]
        pcm_len = np.array([c["timeline"].shape[1] for c in caps], np.int64)
        eof = np.array([c["eof"] for c in caps], np.int64)
        got = ctx.encode_streams_managed(tl, pcm_len, eof)
        plans = [got["plan"][i, :got["nblocks"][i]] for i in range(len(caps))]
        pk = {}
        for W in (0, 1):
            cnt = got["count"][W]
            assert cnt > 0
            desc = np.zeros(cnt, abi.BLOCKDESC_DTYPE)
            for p in plans:
                for b in p[p["W"] == W]:
                    desc["lW"][b["slot"]], desc["nW"][b["slot"]] = b["lW"], b["nW"]
            g, blob = got[W], cnt + 5
            rc, data, bits = _dev_managed(ctx, W, desc, _poisoned(g["posts"], blob, 0x7fff7fff),
                                          _poisoned(g["nonzero"], blob, 1), _poisoned(g["iwork"], blob, 1 << 30))
            assert rc == 0
            mine = _unpack(data, bits)
            ref, _, _ = _ref_curves(ch, rate, q, W, desc, g["posts"], g["nonzero"], g["iwork"])
            for k in range(NB):
                assert mine[k] == ref[k], "W=%d curve %d" % (W, k)
            pk[W] = mine[MID]
        for i, p in enumerate(plans):
            assert [pk[int(b["W"])][int(b["slot"])] for b in p] == wants[i], "stream %d" % i
    finally:
        d.close()


def test_forms_bounds_and_errors(cuda_ok):
    """_dev equals the host form, whose offsets are the running sum of the lengths; a small data_cap gives
    VB200_EINVAL with pkt_bits filled; a bad pkt_stride, blob_blocks < nblocks and an unregistered context give
    VB200_EINVAL; vb200_encode_packets_managed makes vb200_encode_dsp_managed's launches plus four"""
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        cap, _ = _capture(ch, rate, q, probe_signal(ch, rate, 0.5, seed=3))
        W = 1
        sel = cap["W"] == W
        blocks, desc = np.ascontiguousarray(cap["pcm"][sel][:, :, :ctx.bs[W]]), _desc(cap, sel)
        host = ctx.encode_packets_managed(W, blocks, desc)
        m = ctx.encode_dsp_managed(W, blocks, desc)
        rc, data, bits = _dev_managed(ctx, W, desc, m["posts"], m["nonzero"], m["iwork"])
        assert rc == 0 and np.array_equal(bits, host["pkt_bits"])
        assert _unpack(data, bits) == host["packets"]
        lens = ((host["pkt_bits"] + 7) // 8).ravel()
        assert np.array_equal(host["pkt_off"].ravel(), np.concatenate([[0], np.cumsum(lens)[:-1]]))
        small = ctx.encode_packets_managed(W, blocks, desc, data_cap=10, check=False)
        assert small["rc"] == VB200_EINVAL and np.array_equal(small["pkt_bits"], host["pkt_bits"])
        bound = ctx.packet_bound(W)
        args = (ctx, W, desc, m["posts"], m["nonzero"], m["iwork"])
        assert _dev_managed(*args, stride=bound - 4)[0] == VB200_EINVAL
        assert _dev_managed(*args, stride=bound + 2)[0] == VB200_EINVAL
        assert _dev_managed(ctx, W, desc, m["posts"][:, :-1], m["nonzero"][:, :-1], m["iwork"][:, :-1])[0] == VB200_EINVAL
        plain = lib.Context(load_setup("44k_stereo_q5"))
        assert plain.L.vb200_encode_entropy_managed_dev(plain.h, 0, 1, 1, None, None, None, None, 4096, None, None,
                                                        None) == VB200_EINVAL
        assert plain.L.vb200_encode_packets_managed(plain.h, 0, 1, 1, None, None, None, None, 0) == VB200_EINVAL
        plain.close()
        per = []
        for k in (3, len(desc)):
            l0 = ctx.launch_count()
            ctx.encode_dsp_managed(W, blocks[:k], desc[:k])
            l1 = ctx.launch_count()
            ctx.encode_packets_managed(W, blocks[:k], desc[:k])
            per.append((l1 - l0, ctx.launch_count() - l1))
        assert all(b == a + 4 for a, b in per), per
    finally:
        d.close()


@pytest.mark.parametrize("ch,rate,max_br,nominal,min_br", [(2, 44100, -1, 128000, -1), (1, 44100, -1, 64000, -1),
                                                           (2, 44100, 144000, -1, 112000)])
def test_managed_driver_device_path(cuda_ok, ch, rate, max_br, nominal, min_br):
    """7 streams through the managed multi-stream driver: with the device coder (reported on) and with the host path
    forced, every stream's packets (count, bytes, hash) equal the stock managed encoder's; launches per round stay
    within the managed driver's bound"""
    from oracle import encode_managed, managed
    from test_gpu_managed_dropin import _signals
    if not (managed.available() and encode_managed.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ns = 7
    pcm = _signals(ch, rate, ns, 0.8)
    want = [managed.stock_summary(ch, rate, max_br, nominal, min_br, pcm[i])[1:] for i in range(ns)]
    for host in (False, True):
        blocks, rounds, launches, got, on_device = encode_managed.ms_encode(ch, rate, max_br, nominal, min_br, pcm,
                                                                            host_entropy=host)
        assert on_device == (not host)
        print("managed driver %s path: %d blocks, %d rounds, %.2f launches per round"
              % ("host" if host else "device", blocks, rounds, launches / rounds))
        for i in range(ns):
            assert got[i] == want[i], "stream %d (host path forced: %s)" % (i, host)
        assert launches <= 30 * rounds, "%d launches in %d rounds" % (launches, rounds)
