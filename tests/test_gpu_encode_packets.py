"""The entropy coding of mapping0_forward on the device (vb200_encode_entropy[_dev], vb200_encode_packets and the
multi-stream driver's device path) against the reference's own floor1_encode and residue class / forward: every packet
byte for byte.  Needs oracle/_ref (built where the reference sources exist; the libraries travel)."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_setup, probe_signal
from oracle import pyref
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

SETUPS = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2), (2, 44100, 0.1), (2, 32000, 0.0)]


def _need():
    from oracle import encode_packets as ep
    if not (pyref.available() and ep.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    return ep


def _driver(ch, rate, q):
    ep = _need()
    d = ep.Driver(ch, rate, q)
    assert d.on_device
    return d


def _capture(ch, rate, q, pcm):
    """the stock encoder's blocks (PCM, flags, ampmax on entry) and its audio packets"""
    ref = pyref.Ref(ch, rate, q)
    cap = ref.encode_capture(pcm, fields=("pcm",))
    pk = ref.packets()
    ref.close()
    nb = cap["nblocks"]
    assert len(pk) - nb in (0, 3)
    return cap, pk[len(pk) - nb:]


def _desc(cap, sel):
    d = np.zeros(int(sel.sum()), abi.BLOCKDESC_DTYPE)
    for k in ("lW", "nW", "blocktype"):
        d[k] = cap[k][sel]
    d["ampmax"] = cap["ampmax_in"][sel]
    return d


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_stage_parity_captured_blocks(cuda_ok, ch, rate, q):
    """vb200_encode_dsp then vb200_encode_entropy, and vb200_encode_packets alone, on the stock encoder's blocks give
    its audio packets byte for byte; pkt_bits rounds up to the packet's length; no packet exceeds the bound"""
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        pcm = probe_signal(ch, rate, 0.5, seed=11)
        cap, want = _capture(ch, rate, q, pcm)
        for W in (0, 1):
            sel = cap["W"] == W
            if not sel.any():
                continue
            N = ctx.bs[W]
            blocks = np.ascontiguousarray(cap["pcm"][sel][:, :, :N])
            desc = _desc(cap, sel)
            wp = [p for p, s in zip(want, sel) if s]
            chain = ctx.encode_dsp(W, blocks, desc)
            got = ctx.encode_entropy(W, desc, chain["posts"], chain["nonzero"], chain["iwork"])
            assert got["packets"] == wp
            assert all((b + 7) // 8 == len(p) for b, p in zip(got["pkt_bits"], wp))
            assert max(len(p) for p in wp) <= ctx.packet_bound(W)
            fused = ctx.encode_packets(W, blocks, desc)
            assert fused["packets"] == wp
            assert np.array_equal(fused["pkt_bits"], got["pkt_bits"])
            assert np.array_equal(fused["ampmax_out"], chain["ampmax_out"])
    finally:
        d.close()


def _fuzz_inputs(rng, es, W, nb, ch, n):
    posts_max = max(2 + sum(f.class_dim[f.partitionclass[i]] for i in range(f.partitions))
                    for f in es.floor[W] if f.type == 1)
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    if W:
        desc["lW"], desc["nW"] = rng.integers(0, 2, nb), rng.integers(0, 2, nb)
    posts = np.zeros((nb, ch, abi.FLOOR1_STRIDE), np.int32)
    v = rng.integers(0, 64, (nb, ch, posts_max))
    flag = (rng.random((nb, ch, posts_max)) < 0.3) & (np.arange(posts_max) >= 2)
    posts[:, :, :posts_max] = v | (flag * 0x8000)
    posts[rng.random((nb, ch)) < 0.15] = 0                       # silent channels
    nonzero = (rng.random((nb, ch)) < 0.8).astype(np.int32)
    t = rng.standard_t(1.5, (nb, ch, n)) * rng.choice([1, 4, 30], (nb, ch, 1))
    iwork = np.clip(np.round(t), -3000, 3000).astype(np.int32)  # heavy tails: clamped and unused lattice entries
    iwork[rng.random((nb, ch, n)) < 0.3] = 0
    iwork[rng.random((nb, ch)) < 0.05] = 0
    return desc, posts, nonzero, iwork


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_fuzz_against_reference_functions(cuda_ok, ch, rate, q):
    """random quantised posts with random unused flags, silent rows, random nonzero patterns and heavy-tailed residue:
    the device's bytes and bit counts equal the reference's, and the fallback search of local_book_besterror ran"""
    ep = _need()
    d = _driver(ch, rate, q)
    try:
        es, keep = d.setup_copy()
        rng = np.random.default_rng(100 + ch)
        hits = 0
        for W in (0, 1):
            nb = 300 if W == 0 else 150
            desc, posts, nonzero, iwork = _fuzz_inputs(rng, es, W, nb, ch, d.ctx.bs[W] // 2)
            want, post_pass, h = ep.ref_packets(ch, rate, q, W, desc, posts, nonzero, iwork.copy())
            hits += h
            got = d.ctx.encode_entropy(W, desc, post_pass, nonzero, iwork)
            for i in range(nb):
                assert got["packets"][i] == want[i], "W=%d block %d" % (W, i)
                assert (got["pkt_bits"][i] + 7) // 8 == len(want[i])
            assert max(len(p) for p in want) <= d.ctx.packet_bound(W)
        if _stage0_books_with_unused_entries(es):
            assert hits > 0, "no residue vector landed on an unused lattice entry"
    finally:
        d.close()


def _stage0_books_with_unused_entries(es):
    """whether a stage-0 residue book of the setup has entries without a codeword (the fallback search can run)"""
    books = set(r.stagebook[c][0] for w in range(2) for r in es.residue[w] if r.type > 0 for c in range(r.partitions))
    for b in books - {-1}:
        B = es.books[b]
        if B.entries and (np.ctypeslib.as_array((C.c_uint8 * B.entries).from_address(B.length)) == 0).any():
            return True
    return False


def _dev_entropy(ctx, W, desc, posts, nonzero, iwork, stride=None):
    """vb200_encode_entropy_dev through torch device buffers: (strided data uint8 [nb][stride], pkt_bits)"""
    import torch
    nb = len(desc)
    stride = ctx.packet_bound(W) if stride is None else stride
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
         (("desc", desc.view(np.uint8)), ("posts", posts), ("nz", nonzero), ("iw", iwork))}
    bits = torch.zeros(nb, dtype=torch.int32, device="cuda")
    data = torch.zeros(nb * stride, dtype=torch.uint8, device="cuda")
    rc = ctx.encode_entropy_dev(W, nb, t["desc"].data_ptr(), t["posts"].data_ptr(), t["nz"].data_ptr(),
                                t["iw"].data_ptr(), stride, bits.data_ptr(), data.data_ptr(), check=False)
    torch.cuda.synchronize()
    return rc, data.cpu().numpy().reshape(nb, stride), bits.cpu().numpy()


def test_whole_streams(cuda_ok):
    """vb200_encode_streams, then vb200_encode_entropy_dev per block size, reordered by plan[].slot: every stream's
    packets are the stock encoder's for that stream (burst signals, both block sizes)"""
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
        got = ctx.encode_streams(tl, pcm_len, eof)
        plans = [got["plan"][i, :got["nblocks"][i]] for i in range(len(caps))]
        pk = {}
        for W in (0, 1):
            cnt = 1 + max([int(b["slot"]) for p in plans for b in p if b["W"] == W] + [-1])
            assert cnt > 0
            desc = np.zeros(cnt, abi.BLOCKDESC_DTYPE)
            for p in plans:
                for b in p[p["W"] == W]:
                    desc["lW"][b["slot"]], desc["nW"][b["slot"]] = b["lW"], b["nW"]
            g = got[W]
            rc, data, bits = _dev_entropy(ctx, W, desc, g["posts"][:cnt], g["nonzero"][:cnt], g["iwork"][:cnt])
            assert rc == 0
            pk[W] = [bytes(data[s, :(bits[s] + 7) // 8]) for s in range(cnt)]
        for i, p in enumerate(plans):
            mine = [pk[int(b["W"])][int(b["slot"])] for b in p]
            assert mine == wants[i], "stream %d" % i
    finally:
        d.close()


def test_forms_bounds_and_errors(cuda_ok):
    """_dev equals the host form and the packed layout the strided one; a small data_cap gives VB200_EINVAL with
    pkt_bits filled; a small or unaligned pkt_stride and an unregistered context give VB200_EINVAL; hand-edited setups
    give VB200_EINVAL / VB200_EIMPL; vb200_encode_packets makes a fixed number of launches"""
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        es, keep = d.setup_copy()
        rng = np.random.default_rng(7)
        W = 1
        desc, posts, nonzero, iwork = _fuzz_inputs(rng, es, W, 40, ch, ctx.bs[W] // 2)
        host = ctx.encode_entropy(W, desc, posts, nonzero, iwork)
        rc, data, bits = _dev_entropy(ctx, W, desc, posts, nonzero, iwork)
        assert rc == 0 and np.array_equal(bits, host["pkt_bits"])
        for i in range(len(desc)):
            assert bytes(data[i, :(bits[i] + 7) // 8]) == host["packets"][i]
        assert host["pkt_off"][0] == 0
        assert np.array_equal(np.diff(host["pkt_off"]), ((host["pkt_bits"] + 7) // 8)[:-1])
        small = ctx.encode_entropy(W, desc, posts, nonzero, iwork, data_cap=10, check=False)
        assert small["rc"] == -131 and np.array_equal(small["pkt_bits"], host["pkt_bits"])
        bound = ctx.packet_bound(W)
        assert bound % 4 == 0 and max(len(p) for p in host["packets"]) <= bound
        assert _dev_entropy(ctx, W, desc, posts, nonzero, iwork, stride=bound - 4)[0] == -131
        assert _dev_entropy(ctx, W, desc, posts, nonzero, iwork, stride=bound + 2)[0] == -131
        # an unregistered context
        plain = lib.Context(load_setup("44k_stereo_q5"))
        assert plain.L.vb200_encode_packet_bound(plain.h, 0) == -131
        assert plain.L.vb200_encode_entropy(plain.h, 0, 1, None, None, None, None, None, None, None, 0) == -131
        plain.close()

        def reg(edit):
            e, bk = d.setup_copy()
            edit(e, bk)
            return ctx.L.vb200_encode_entropy_setup(ctx.h, C.byref(e))

        stage = next(es.residue[1][0].stagebook[c][s] for c in range(64) for s in range(8)
                     if es.residue[1][0].stagebook[c][s] >= 0)
        used_cls = es.floor[1][0].partitionclass[0]
        longer = np.full(keep[0].entries, 33, np.uint8)
        cases = [
            (-131, lambda e, b: setattr(e.residue[1][0], "groupbook", e.nbooks)),
            (-131, lambda e, b: b[stage].__setattr__("dim", 9)),
            (-131, lambda e, b: b[stage].__setattr__("quantvals", 0)),
            (-131, lambda e, b: b[0].__setattr__("length", longer.ctypes.data)),
            (-131, lambda e, b: setattr(e.residue[1][0], "end", 1 << 20)),
            (-131, lambda e, b: e.floor[1][0].class_dim.__setitem__(used_cls, 9)),
            (-131, lambda e, b: e.floor[1][0].class_subs.__setitem__(used_cls, 4)),
            (-130, lambda e, b: setattr(e.residue[0][0], "type", 0)),
            (-130, lambda e, b: setattr(e.floor[0][0], "type", 0)),
        ]
        for want_rc, edit in cases:
            assert reg(edit) == want_rc
        e, bk = d.setup_copy()                              # the driver's own setup registers again
        ctx.encode_entropy_setup(e)
        # launches per vb200_encode_packets: those of vb200_encode_dsp on one batch plus four, for any batch size
        cap, _ = _capture(ch, rate, q, probe_signal(ch, rate, 0.5, seed=3))
        sel = cap["W"] == 1
        blocks, desc = np.ascontiguousarray(cap["pcm"][sel][:, :, :ctx.bs[1]]), _desc(cap, sel)
        per = []
        for k in (3, len(desc)):
            l0 = ctx.launch_count()
            ctx.encode_dsp(1, blocks[:k], desc[:k])
            l1 = ctx.launch_count()
            ctx.encode_packets(1, blocks[:k], desc[:k])
            per.append((l1 - l0, ctx.launch_count() - l1))
        assert per[0] == per[1] and per[0][1] == per[0][0] + 4, per
    finally:
        d.close()


@pytest.mark.parametrize("ch,rate,q", SETUPS[:3])
def test_multistream_driver_device_path(cuda_ok, ch, rate, q):
    """7 streams through the multi-stream driver: on the device path and with the host path forced, every stream's
    packets (count, bytes, hash) equal the stock encoder's"""
    from test_plan_vs_ref import burst_signal
    ep = _need()
    ns, secs = 7, 0.6
    n = int(rate * secs)
    sig = [probe_signal(ch, rate, secs, seed=60 + i)[:, :n] if i % 2 == 0 else burst_signal(ch, rate, secs, 70 + i)[:, :n]
           for i in range(ns)]
    pcm = np.ascontiguousarray(np.stack(sig), np.float32)
    L = pyref.lib()
    L.ref_stock_encode_summary.restype = C.c_long
    want = []
    for i in range(ns):
        h, b, c = C.c_uint64(0), C.c_long(0), C.c_long(0)
        p = np.ascontiguousarray(pcm[i])
        L.ref_stock_encode_summary(ch, C.c_long(rate), C.c_float(q), p.ctypes.data_as(C.c_void_p), C.c_long(n),
                                   C.byref(h), C.byref(b), C.byref(c))
        want.append((c.value, b.value, h.value))
    for host in (False, True):
        blocks, got, on_device = ep.ms_encode(pcm, ch, rate, q, host_entropy=host)
        assert on_device == (not host)
        assert blocks > 0
        for i in range(ns):
            assert got[i] == want[i], "stream %d (host path forced: %s)" % (i, host)
