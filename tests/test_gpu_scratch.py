"""The context's device scratch: the arenas of different call families never overlap, the host forms stage through
a pool of their own, and the debug cycle counters survive other calls.

- A host decode call between two reads of the cycle counters leaves them as they were.
- One context runs the host forms of every encode family in two orders, each at a larger and a smaller size, and
  every output equals the same call on a fresh context.
- vb200_encode_dsp_dev and vb200_encode_streams_dev issued alternately on two streams equal serial runs.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import probe_signal
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

SETUP = (2, 44100, 0.5)


def _same(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _same(a[k], b[k], "%s[%r]" % (what, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s[%d]" % (what, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape, what
        assert a.tobytes() == b.tobytes(), what
    else:
        assert a == b, what


def _encode_driver():
    from oracle import encode_packets as ep
    from oracle import pyref
    if not (pyref.available() and ep.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    d = ep.Driver(*SETUP)
    assert d.on_device
    return d


def _blocks(ctx, nb, seed):
    rng = np.random.default_rng(seed)
    ch, N = ctx.channels, ctx.bs[1]
    pcm = (0.3 * rng.standard_normal((nb, ch, N))).astype(np.float32)
    desc = np.zeros(nb, abi.BLOCKDESC_DTYPE)
    desc["lW"] = 1; desc["nW"] = 1; desc["blocktype"] = rng.integers(0, 2, nb)
    desc["ampmax"] = rng.uniform(-30, -3, nb).astype(np.float32)
    return pcm, desc


def _timelines(ctx, ns, secs, seed):
    ch = ctx.channels
    sig = [probe_signal(ch, 44100, secs * (1 + 0.25 * s), seed + s) for s in range(ns)]
    stride = (max(x.shape[1] for x in sig) + ctx.bs[1] + 3) & ~3
    tl = np.zeros((ns, ch, stride), np.float32)
    for s, x in enumerate(sig):
        tl[s, :, ctx.bs[1] // 2:ctx.bs[1] // 2 + x.shape[1]] = x
    return tl, np.full(ns, stride, np.int64)


def _planned(plan, nb):
    """the plan rows the call writes: those past a stream's block count hold whatever the buffer held"""
    plan = plan.copy()
    for s, k in enumerate(nb):
        plan[s, k:] = np.zeros(1, plan.dtype)
    return plan


def _streams(out):
    out["plan"] = _planned(out["plan"], out["nblocks"])
    return out


def _calls(ctx):
    """(name, size, fn(ctx)) of every encode family's host form, sizes large then small"""
    out = []
    for size, (nb, ns, secs) in (("large", (12, 3, 0.5)), ("small", (5, 2, 0.25))):
        pcm, desc = _blocks(ctx, nb, 7 + nb)
        tl, tlen = _timelines(ctx, ns, secs, 40 + ns)
        nsteps = (tl.shape[2] - 128) // 64 + 1
        ret, _ = ctx.envelope_search(tl, 0, nsteps)
        mark = np.zeros((ns, nsteps + 4), np.int32)
        for s in range(ns):
            mark[s, :nsteps + 2] = ctx.envelope_marks(ret[s])
        out += [
            ("encode_dsp", size, lambda c, p=pcm, d=desc: c.encode_dsp(1, p, d, classes=True)),
            ("encode_dsp_managed", size, lambda c, p=pcm, d=desc: c.encode_dsp_managed(1, p, d)),
            ("encode_packets", size, lambda c, p=pcm, d=desc: c.encode_packets(1, p, d)),
            ("encode_packets_managed", size, lambda c, p=pcm, d=desc: c.encode_packets_managed(1, p, d)),
            ("encode_streams", size, lambda c, t=tl, n=tlen: _streams(c.encode_streams(t, n))),
            ("encode_streams_managed", size, lambda c, t=tl, n=tlen: _streams(c.encode_streams_managed(t, n))),
            ("plan_blocks", size,
             lambda c, m=mark, k=nsteps, n=tlen: (lambda p, nb: (_planned(p, nb), nb))(*c.plan_blocks(m, k, n))),
            ("envelope_search", size, lambda c, t=tl, k=nsteps: c.envelope_search(t, 0, k)),
            ("phaseA_taps", size, lambda c, p=pcm, d=desc: c.phaseA(1, p, d, taps=True)),
        ]
    return out


def test_families_do_not_share_scratch(cuda_ok):
    """every family's host form, in two orders on one context, equals the same call on a fresh context"""
    d = _encode_driver()
    try:
        calls = _calls(d.ctx)
    finally:
        d.close()
    want = {}
    for name, size, f in calls:
        d = _encode_driver()
        try:
            want[name, size] = f(d.ctx)
        finally:
            d.close()
    # order 1: each family large then small (the arenas grow, then are reused); order 2: the reverse
    for order in (calls, calls[::-1]):
        d = _encode_driver()
        try:
            for name, size, f in order:
                _same(f(d.ctx), want[name, size], "%s (%s)" % (name, size))
        finally:
            d.close()


def test_host_decode_keeps_the_cycle_counters(cuda_ok):
    """vb200_decode_packets_resume with a count array stages 11 buffers; the cycle counters are not among them"""
    from oracle import decode
    from oracle import decode_packets as dp
    if not (decode.available() and dp.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    p = decode.encode(2, 44100, 0.5, probe_signal(2, 44100, 0.5, seed=300))
    drv = dp.Driver(p)
    try:
        ctx, ch, bs = drv.ctx, drv.channels, drv.bs
        pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.audio[:, :2]][:10]
        W = dp.ref_headers(p, pk)
        data = np.frombuffer(b"".join(pk) + b"\0", np.uint8).copy()
        lens = np.array([len(b) for b in pk], np.int32)
        # stream 0 decodes the packets; stream 1 has none this call and keeps its fresh carry (W = -1)
        count = np.array([len(pk), 0], np.int32)
        Wseq = np.zeros((2, len(pk)), np.int32)
        Wseq[0] = W
        pkt_off = np.zeros((2, len(pk)), np.int64)
        pkt_off[0] = np.concatenate([[0], np.cumsum(lens)[:-1]])
        pkt_bytes = np.zeros((2, len(pk)), np.int32)
        pkt_bytes[0] = lens
        carry = ctx.new_decode_carry(2)
        coef_off, pcm_off, coef_len, pcm_len = lib.synthesis_layout(Wseq, bs, ch, carry_W=carry[1], count=count)
        ctx.debug_phase_cycles(reset=True)
        ctx.decode_packets_resume(Wseq, coef_off, max(coef_len, 1), pkt_off, pkt_bytes, data, pcm_off,
                                  max(pcm_len, 1), carry, count=count)
        assert (carry[1][1] == -1).all()
        assert not np.asarray(ctx.debug_phase_cycles(reset=False)).any()
    finally:
        drv.close()


def test_dev_calls_on_two_streams(cuda_ok):
    """vb200_encode_dsp_dev and vb200_encode_streams_dev alternating on two streams, no host synchronise between
    them, equal the host forms run one after the other"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device in torch")
    d = _encode_driver()
    try:
        ctx = d.ctx
        ch, dev = ctx.channels, torch.device("cuda", 0)
        pcm, desc = _blocks(ctx, 12, 5)
        tl, tlen = _timelines(ctx, 3, 0.5, 60)
        want_dsp = ctx.encode_dsp(1, pcm, desc)
        want_str = ctx.encode_streams(tl, tlen)
        nb, n = len(desc), ctx.bs[1] // 2
        max_blocks = tl.shape[2] // (ctx.bs[0] // 2) + 8
        caps = [max(c, 1) for c in want_str["count"]]
        s = [torch.cuda.Stream(), torch.cuda.Stream()]
        runs, launch = [], []
        for k in range(4):
            st = s[k & 1]
            if k % 2 == 0:
                t = {"pcm": torch.from_numpy(pcm).to(dev), "desc": torch.from_numpy(desc.view(np.uint8).copy()).to(dev),
                     "posts": torch.zeros((nb, ch, abi.FLOOR1_STRIDE), dtype=torch.int32, device=dev),
                     "nonzero": torch.zeros((nb, ch), dtype=torch.int32, device=dev),
                     "iwork": torch.zeros((nb, ch, n), dtype=torch.int32, device=dev),
                     "ampmax_out": torch.zeros(nb, device=dev)}
                io = abi.EncodeIO()
                for key, v in t.items():
                    setattr(io, key, v.data_ptr())
                io.independent = 1
                launch.append(lambda io=io, st=st: ctx.encode_dsp_dev(1, nb, 1, io, stream=st.cuda_stream))
            else:
                t = {"pcm": torch.from_numpy(tl).to(dev), "pcm_len": torch.from_numpy(tlen).to(dev),
                     "plan": torch.zeros(3 * max_blocks * abi.STREAM_BLOCK_DTYPE.itemsize, dtype=torch.uint8, device=dev),
                     "nblocks": torch.zeros(3, dtype=torch.int32, device=dev)}
                for w in range(2):
                    t[w] = {"posts": torch.zeros((caps[w], ch, abi.FLOOR1_STRIDE), dtype=torch.int32, device=dev),
                            "nonzero": torch.zeros((caps[w], ch), dtype=torch.int32, device=dev),
                            "iwork": torch.zeros((caps[w], ch, ctx.bs[w] // 2), dtype=torch.int32, device=dev),
                            "ampmax_out": torch.zeros(caps[w], device=dev)}
                io = abi.StreamsIO()
                io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = (t["pcm"].data_ptr(), lib.PCM_F32_PLANAR,
                                                                       max_blocks, tl.shape[2])
                io.pcm_len, io.plan, io.nblocks = t["pcm_len"].data_ptr(), t["plan"].data_ptr(), t["nblocks"].data_ptr()
                for w in range(2):
                    io.cap[w] = caps[w]
                    io.posts[w], io.nonzero[w] = t[w]["posts"].data_ptr(), t[w]["nonzero"].data_ptr()
                    io.iwork[w], io.ampmax_out[w] = t[w]["iwork"].data_ptr(), t[w]["ampmax_out"].data_ptr()

                def go(io=io, st=st):
                    ctx._chk(ctx.L.vb200_encode_streams_dev(ctx.h, 3, 7, C.byref(io), st.cuda_stream))
                    assert [io.count[0], io.count[1]] == want_str["count"]
                launch.append(go)
            runs.append((t, io))
        torch.cuda.synchronize()                              # the inputs are on the device
        for f in launch:
            f()
        torch.cuda.synchronize()
        for k, (t, _) in enumerate(runs):
            if k % 2 == 0:
                for key in ("posts", "nonzero", "iwork", "ampmax_out"):
                    _same(t[key].cpu().numpy(), want_dsp[key], "encode_dsp_dev run %d %s" % (k, key))
            else:
                _same(t["nblocks"].cpu().numpy(), want_str["nblocks"], "encode_streams_dev run %d nblocks" % k)
                for w in range(2):
                    cnt = want_str["count"][w]
                    for key in ("posts", "nonzero", "iwork", "ampmax_out"):
                        _same(t[w][key].cpu().numpy()[:cnt], want_str[w][key], "encode_streams_dev run %d %s[%d]" % (k, key, w))
    finally:
        d.close()
