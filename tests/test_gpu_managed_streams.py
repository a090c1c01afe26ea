"""Bitrate-managed mode for whole streams (vb200_encode_streams_managed[_dev]) and the one-launch couple/quantise/
normalise of all 15 curves (k_cqn_fast_curves) that it shares with vb200_encode_dsp_managed.  Bit-exact against the
oracle's per-block managed composition with the ampmax chain carried along each stream."""
import ctypes as C

import numpy as np
import pytest

from conftest import CONFIG_NAMES, REF_ARGS, assert_bits_equal, load_setup, probe_signal
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu

NB, MID = abi.PACKETBLOBS, abi.PACKETBLOBS // 2
VB200_EINVAL = -131                                       # include/vorbis_b200.h


@pytest.fixture(scope="module", params=CONFIG_NAMES)
def cfg(request, oracle_lib, cuda_ok):
    name = request.param
    setup = load_setup(name)
    return name, setup, vlib.Context(setup), oracle_lib.Oracle(setup)


class _ManagedChain:
    """an Oracle whose encode_dsp is encode_dsp_managed: Oracle.encode_stream's composition (marks -> block plan ->
    every block in order with the ampmax decay chain carried across block sizes) with the 15 curves per block"""

    def __init__(self, o):
        self.o = o

    def __getattr__(self, name):
        return getattr(self.o, name)

    def encode_dsp(self, W, pcm, desc, blobno=None):
        return self.o.encode_dsp_managed(W, pcm, desc)


def managed_stream(o, tl, pcm_len, eof):
    return type(o).encode_stream(_ManagedChain(o), tl, pcm_len, eof)


def stream_timelines(name):
    """the timelines of test_gpu_parity.py::test_encode_streams_mixed_block_sizes (the reference's own stream
    buffers), plus a silent stream as long as the first"""
    import refgold
    from test_gpu_parity import streams_signals
    rec = refgold.load("streams_" + name)
    tls, eofs = [], []
    for i, s in enumerate(streams_signals(*REF_ARGS[name])):
        p = "s%d_" % i
        tls.append(refgold.timeline(rec, s, p))
        eofs.append(int(rec[p + "eof"]))
    tls.append(np.zeros_like(tls[0]))
    eofs.append(eofs[0])
    ch = tls[0].shape[0]
    stride = (max(t.shape[1] for t in tls) + 3) & ~3
    tl = np.zeros((len(tls), ch, stride), np.float32)
    for i, t in enumerate(tls):
        tl[i, :, :t.shape[1]] = t
    pcm_len = np.array([t.shape[1] for t in tls], np.int64)
    return tl, pcm_len, np.array(eofs, np.int64)


@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_encode_streams_managed_vs_oracle(cfg, fmt):
    name, setup, ctx, o = cfg
    tl, pcm_len, eof = stream_timelines(name)
    ch = setup.channels
    if fmt == "f32":
        args = (tl, pcm_len, eof)
        kw = {}
    else:
        s16 = np.clip(np.rint(tl * 32767.0), -32768, 32767).astype(np.int16)
        tl = s16.astype(np.float32) / np.float32(32768.0)
        args = (np.ascontiguousarray(s16.transpose(0, 2, 1)), pcm_len, eof)
        kw = {"fmt": vlib.PCM_S16_INTERLEAVED}
    got = ctx.encode_streams_managed(*args, **kw)
    one = ctx.encode_streams(*args, **kw, blobno=MID)
    assert got["count"] == one["count"]
    assert np.array_equal(got["nblocks"], one["nblocks"])
    assert np.array_equal(got["plan"], one["plan"]), "the plan is the un-managed call's"
    for W in (0, 1):
        g, u = got[W], one[W]
        assert g["posts"].shape[:2] == (NB, got["count"][W])
        for k in ("posts", "nonzero", "iwork"):
            assert np.array_equal(g[k][MID], u[k]), "W=%d curve %d %s vs vb200_encode_streams" % (W, MID, k)
        assert_bits_equal(g["ampmax_out"], u["ampmax_out"], "ampmax_out vs vb200_encode_streams")
    nshort = 0
    silent = len(pcm_len) - 1
    for i in range(len(pcm_len)):
        wplan, wouts = managed_stream(o, tl[i], pcm_len[i], eof[i])
        k = len(wplan)
        assert got["nblocks"][i] == k, "stream %d: %d blocks, want %d" % (i, got["nblocks"][i], k)
        plan = got["plan"][i, :k]
        for nm in ("W", "lW", "nW", "blocktype"):
            assert np.array_equal(plan[nm], wplan[nm]), "stream %d %s" % (i, nm)
        for b in range(k):
            W, slot = int(plan[b]["W"]), int(plan[b]["slot"])
            nshort += W == 0
            g, w = got[W], wouts[b]
            for nm in ("posts", "nonzero", "iwork"):
                assert np.array_equal(g[nm][:, slot], w[nm][:, 0]), "stream %d block %d %s" % (i, b, nm)
            assert_bits_equal(g["ampmax_out"][slot:slot + 1], w["ampmax_out"], "stream %d block %d ampmax" % (i, b))
            if i == silent:
                assert not g["nonzero"][:, slot].any(), "the silent stream has no curve at any rate"
    assert nshort >= 10                                       # the streams really mix the two sizes
    assert got["count"][0] == nshort


def _streams_io(ctx, pcm, pcm_len, eof, caps, max_blocks):
    """host vb200_streams_io with cap-strided managed outputs"""
    ch = ctx.channels
    io = abi.StreamsIO()
    io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = pcm.ctypes.data, vlib.PCM_F32_PLANAR, max_blocks, pcm.shape[2]
    io.pcm_len, io.eof = pcm_len.ctypes.data, eof.ctypes.data
    keep = {"plan": np.zeros((pcm.shape[0], max_blocks), abi.STREAM_BLOCK_DTYPE), "nb": np.zeros(pcm.shape[0], np.int32)}
    io.plan, io.nblocks = keep["plan"].ctypes.data, keep["nb"].ctypes.data
    for w in range(2):
        cw, n = max(int(caps[w]), 1), ctx.bs[w] // 2
        io.cap[w] = int(caps[w])
        keep[w] = [np.zeros(NB * cw * ch * abi.FLOOR1_STRIDE, np.int32), np.zeros(NB * cw * ch, np.int32),
                   np.zeros(NB * cw * ch * n, np.int32), np.zeros(cw, np.float32)]
        io.posts[w], io.nonzero[w], io.iwork[w], io.ampmax_out[w] = (a.ctypes.data for a in keep[w])
    return io, keep


def test_encode_streams_managed_cap(cfg):
    """count > cap: VB200_EINVAL with count[] holding the need; a size with cap 0 and no blocks succeeds"""
    name, setup, ctx, o = cfg
    tl, pcm_len, eof = stream_timelines(name)
    want = ctx.encode_streams_managed(tl, pcm_len, eof)
    mb = tl.shape[2] // (ctx.bs[0] // 2) + 8
    io, keep = _streams_io(ctx, tl, pcm_len, eof, (want["count"][0] - 1, want["count"][1]), mb)
    rc = ctx.L.vb200_encode_streams_managed(ctx.h, tl.shape[0], C.byref(io))
    assert rc == VB200_EINVAL
    assert [io.count[0], io.count[1]] == want["count"]
    # one short stream that ends before a long block could start: only short blocks
    n0 = ctx.bs[1] // 2 + ctx.bs[0]
    short = np.zeros((1, setup.channels, (n0 + 2 * ctx.bs[1] + 3) & ~3), np.float32)
    short[0, :, ctx.bs[1] // 2:n0] = probe_signal(setup.channels, setup.rate, 1.0, 3)[:, :n0 - ctx.bs[1] // 2]
    slen, seof = np.array([short.shape[2]], np.int64), np.array([n0], np.int64)
    plan, nb = o.plan_blocks(*o.timeline_marks(short), slen, seof)
    assert nb[0] > 0 and not (plan[0, :nb[0]]["W"] == 1).any()
    wantm = ctx.encode_streams_managed(short, slen, seof, cap=[64, 1])
    io, keep = _streams_io(ctx, short, slen, seof, (64, 0), 64)
    assert ctx.L.vb200_encode_streams_managed(ctx.h, 1, C.byref(io)) == 0
    assert [io.count[0], io.count[1]] == [wantm["count"][0], 0] and io.count[0] > 0
    cnt, rows = io.count[0], io.count[0] * setup.channels
    nz = keep[0][1].reshape(NB, 64 * setup.channels)[:, :rows]
    assert np.array_equal(nz, wantm[0]["nonzero"].reshape(NB, rows))


def test_encode_streams_managed_dev_equals_host(cfg):
    """the _dev form on torch device buffers (cap-strided curves) equals the host form"""
    import torch
    name, setup, ctx, o = cfg
    tl, pcm_len, eof = stream_timelines(name)
    s16 = np.ascontiguousarray(np.clip(np.rint(tl * 32767.0), -32768, 32767).astype(np.int16).transpose(0, 2, 1))
    ns, stride, ch = s16.shape
    mb = stride // (ctx.bs[0] // 2) + 8
    caps = [ns * mb, ns * (stride // (ctx.bs[1] // 2) + 8)]
    want = ctx.encode_streams_managed(s16, pcm_len, eof, fmt=vlib.PCM_S16_INTERLEAVED, max_blocks=mb, cap=caps)
    dev = torch.device("cuda:0")
    t = {"pcm": torch.from_numpy(s16).to(dev), "pcm_len": torch.from_numpy(pcm_len).to(dev),
         "eof": torch.from_numpy(eof).to(dev),
         "plan": torch.zeros((ns, mb, abi.STREAM_BLOCK_DTYPE.itemsize // 4), dtype=torch.int32, device=dev),
         "nblocks": torch.zeros(ns, dtype=torch.int32, device=dev)}
    io = abi.StreamsIO()
    io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = t["pcm"].data_ptr(), vlib.PCM_S16_INTERLEAVED, mb, stride
    io.pcm_len, io.eof, io.plan, io.nblocks = (t[k].data_ptr() for k in ("pcm_len", "eof", "plan", "nblocks"))
    out = {}
    for w in range(2):
        n = ctx.bs[w] // 2
        io.cap[w] = caps[w]
        out[w] = {"posts": torch.full((NB, caps[w], ch, abi.FLOOR1_STRIDE), -1, dtype=torch.int32, device=dev),
                  "nonzero": torch.full((NB, caps[w], ch), -1, dtype=torch.int32, device=dev),
                  "iwork": torch.full((NB, caps[w], ch, n), -1, dtype=torch.int32, device=dev),
                  "ampmax_out": torch.zeros(caps[w], dtype=torch.float32, device=dev)}
        io.posts[w], io.nonzero[w] = out[w]["posts"].data_ptr(), out[w]["nonzero"].data_ptr()
        io.iwork[w], io.ampmax_out[w] = out[w]["iwork"].data_ptr(), out[w]["ampmax_out"].data_ptr()
    ctx._chk(ctx.L.vb200_encode_streams_managed_dev(ctx.h, ns, C.byref(io), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert [io.count[0], io.count[1]] == want["count"]
    assert np.array_equal(t["nblocks"].cpu().numpy(), want["nblocks"])
    assert np.array_equal(t["plan"].cpu().numpy().view(abi.STREAM_BLOCK_DTYPE).reshape(ns, mb), want["plan"])
    for w in range(2):
        cnt = io.count[w]
        for k in ("posts", "nonzero", "iwork"):
            g = out[w][k].cpu().numpy()
            assert np.array_equal(g[:, :cnt], want[w][k]), "W=%d %s" % (w, k)
            assert (g[:, cnt:] == -1).all(), "W=%d %s: rows past count are not written" % (w, k)
        assert_bits_equal(out[w]["ampmax_out"].cpu().numpy()[:cnt], want[w]["ampmax_out"], "ampmax_out")


@pytest.mark.parametrize("W", [0, 1])
def test_encode_dsp_managed_many_tasks_per_warp(cfg, W):
    """vb200_encode_dsp_managed on a batch large enough that every warp of k_cqn_fast_curves walks several tasks
    (the next task's first curve is prefetched during the last curve); the 6-channel setup takes the per-curve
    k_cqn path"""
    name, setup, ctx, o = cfg
    N, ch = setup.blocksize(W), setup.channels
    nb = (6000 if W == 0 else 2000) if ch <= 2 else 150
    rng = np.random.default_rng(900 + W)
    t = np.arange(N)
    amp = rng.uniform(0.0, 0.6, (nb, 1, 1)).astype(np.float32)
    amp[rng.uniform(size=nb) < 0.05] = 0                               # silent blocks: every curve NULL
    blocks = (amp * (0.3 * rng.standard_normal((nb, ch, N)) +
                     np.sin(2 * np.pi * rng.uniform(100, 8000, (nb, 1, 1)) * t / setup.rate))).astype(np.float32)
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["lW"] = W; desc["nW"] = W
    desc["blocktype"] = rng.integers(0, 2, nb)
    desc["ampmax"] = rng.uniform(-60, -3, nb)
    want = o.encode_dsp_managed(W, blocks, desc)
    got = ctx.encode_dsp_managed(W, blocks, desc)
    for k in ("posts", "nonzero", "iwork"):
        assert np.array_equal(got[k], want[k]), "%s: %d diffs" % (k, int((got[k] != want[k]).sum()))
    assert_bits_equal(got["ampmax_out"], want["ampmax_out"], "ampmax_out")
    assert got["nonzero"].any() and not got["nonzero"].all()
