"""Raw PCM to packets from device memory (vb200_encode_pcm_packets[_managed]_dev): after every call the packets,
info, plan, nblocks, counts and carry bytes equal the host form's bit for bit, with the carries moving between the
forms; a whole clip passed with first = 0 on every call gives the host form's output; refusals that depend on device
values are reported in status / result and leave the data and every carry as they were."""
import numpy as np
import pytest

from oracle import bitrate as B
from test_gpu_encode_packets import SETUPS, _driver
from test_gpu_pcm_packets import LONG_SETUP, Feed, _sched, _to_s16, _vs
from test_gpu_stream_packets import MANAGED, _streams
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

VB200_EINVAL = -131


def _torch():
    return pytest.importorskip("torch")


def _dev(a):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def dev_call(ctx, pcm, lens, carry, end=None, managed=False, max_blocks=None, cap=None, data_cap=None, first=None,
             sentinel=0, mark_steps=0, keep=False):
    """the _dev form on device copies of the host form's arguments (defaults as Context.encode_pcm_packets); returns
    that call's dict, with "status", "result", "carry" (the device carries read back) and the data buffer"""
    torch = _torch()
    ch, bs0, bs1 = ctx.channels, ctx.bs[0], ctx.bs[1]
    if pcm.dtype == np.int16:
        fmt, ns, stride = lib.PCM_S16_INTERLEAVED, pcm.shape[0], pcm.shape[1]
    else:
        fmt, ns, stride = lib.PCM_F32_PLANAR, pcm.shape[0], pcm.shape[2]
    span = stride + 4 * bs1
    if max_blocks is None:
        max_blocks = span // (bs0 // 2) + 8
    if cap is None:
        cap = [ns * max_blocks, ns * (span // (bs1 // 2) + 8)]
    if data_cap is None:
        data_cap = ns * max_blocks * max(ctx.packet_bound(0), ctx.packet_bound(1))
    d = {"pcm": _dev(pcm), "len": _dev(np.asarray(lens, np.int64)), "carry": _dev(carry),
         "end": None if end is None else _dev(np.asarray(end, np.int32)),
         "first": None if first is None else _dev(np.asarray(first, np.int64)),
         "plan": torch.zeros(ns * max_blocks * abi.STREAM_BLOCK_DTYPE.itemsize, dtype=torch.uint8, device="cuda"),
         "nb": torch.zeros(ns, dtype=torch.int32, device="cuda"),
         "info": torch.zeros(ns * max_blocks * abi.PACKET_INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda"),
         "data": torch.full((max(data_cap, 1),), sentinel, dtype=torch.uint8, device="cuda"),
         "status": torch.full((ns,), 7, dtype=torch.int32, device="cuda"),
         "res": torch.zeros(abi.ENCODE_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")}
    p = lambda k: None if d[k] is None else d[k].data_ptr()  # noqa: E731
    rc = ctx.encode_pcm_packets_dev(ns, p("pcm"), fmt, stride, p("len"), p("carry"), p("plan"), p("nb"), max_blocks,
                                    cap, p("info"), p("data"), data_cap, p("status"), p("res"), d_end=p("end"),
                                    d_first=p("first"), mark_steps=mark_steps, managed=managed, check=False)
    torch.cuda.synchronize()
    info = d["info"].cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(ns, max_blocks)
    data = d["data"].cpu().numpy()
    nb = d["nb"].cpu().numpy()
    res = d["res"].cpu().numpy().view(abi.ENCODE_RESULT_DTYPE)[0]
    out = {"rc": rc, "plan": d["plan"].cpu().numpy().view(abi.STREAM_BLOCK_DTYPE).reshape(ns, max_blocks),
           "nblocks": nb, "info": info, "data": data, "status": d["status"].cpu().numpy(), "result": res,
           "count": [int(res["count"][0]), int(res["count"][1])],
           "carry": d["carry"].cpu().numpy().reshape(carry.shape)}
    if keep:
        out["dev"] = d
    if rc == 0 and res["rc"] == 0:
        out["packets"] = [[bytes(data[r["offset"]:r["offset"] + r["bytes"]]) for r in info[i, :nb[i]]]
                          for i in range(ns)]
    return out


class DevFeed(Feed):
    """Feed through the _dev form; alt: every other call through the host form instead, on the same carries"""

    def __init__(self, *a, alt=False, **kw):
        super().__init__(*a, **kw)
        self.alt, self.calls, self.mark_steps = alt, 0, kw.get("mark_steps", 0)

    def step(self, new=None, end=None, **kw):
        ctx = self.ctx
        real = ctx.encode_pcm_packets
        use_dev = not (self.alt and self.calls % 2)
        self.calls += 1

        def fake(pcm, lens, carry, end=None, managed=False, max_blocks=None, check=True, **_):
            got = dev_call(ctx, pcm, lens, carry, end, managed=managed, max_blocks=max_blocks,
                           mark_steps=self.mark_steps)
            assert got["rc"] == 0 and got["result"]["rc"] == 0 and not got["status"].any()
            carry[:] = got["carry"]
            return got
        if use_dev:
            ctx.encode_pcm_packets = fake
        try:
            got = super().step(new, end, **kw)
        finally:
            ctx.encode_pcm_packets = real
        return got


def _lockstep(ctx, pcms, scheds, s16=False, managed=False, max_blocks=None, alt=False, mark_steps=0):
    """the host form and the _dev form fed the same writes, compared after every call"""
    feeds = [p for p in pcms]
    if s16:
        feeds = [_to_s16(p)[0].T for p in pcms]
    h = Feed(ctx, feeds, scheds, managed=managed, s16=s16, max_blocks=max_blocks, mark_steps=mark_steps)
    g = DevFeed(ctx, feeds, scheds, managed=managed, s16=s16, max_blocks=max_blocks, mark_steps=mark_steps, alt=alt)
    for k in range(100000):
        if ctx.encode_pcm_carry_head(h.carry)["enc"]["done"].all():
            break
        a = h.step()
        b = g.step()
        what = "call %d" % k
        assert np.array_equal(a["nblocks"], b["nblocks"]), what
        assert list(a["count"]) == list(b["count"]), what
        for s in range(len(pcms)):
            n = int(a["nblocks"][s])
            assert a["plan"][s, :n].tobytes() == b["plan"][s, :n].tobytes(), what
        assert a["info"].tobytes() == b["info"].tobytes(), what
        assert a["packets"] == b["packets"], what
        assert np.array_equal(h.carry, g.carry), what + ": carries"
    assert ctx.encode_pcm_carry_head(g.carry)["enc"]["done"].all()
    return h, g


@pytest.mark.parametrize("ch,rate,q", SETUPS + [LONG_SETUP])
def test_dev_equals_host(cuda_ok, ch, rate, q):
    """float and int16, writes of 64, 1000, 1024, 4410 samples and whole files, then the end: the _dev form equals the
    host form after every call, and through it the stock encoder where the reference is built"""
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        sig = _streams(ch, rate, 0.6)
        ws = (64, 1000, 1024, 4410, None)
        pcms = [p for w in ws for p in sig]
        scheds = [_sched(p.shape[1], w) for w in ws for p in sig]
        for s16 in (False, True):
            _, g = _lockstep(ctx, pcms, scheds, s16=s16)
            if B.ref_available():
                caps = [B.ref_stream_capture(B.vbr(ch, rate, q), _to_s16(p)[1] if s16 else p,
                                             chunk=w or max(p.shape[1], 1)) for w in ws for p in sig]
                _vs(g, caps, "q=%g %s" % (q, "s16" if s16 else "f32"))
    finally:
        d.close()


def test_dev_drain_and_alternation(cuda_ok):
    """max_blocks cuts a call short (drain calls), and carries that alternate between the forms call by call give
    the output of either form alone"""
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        sig = _streams(ch, rate, 0.6)
        n = [p.shape[1] for p in sig]
        steps = max(n) // 64 + ctx.bs[1] // 16 + 64
        _lockstep(ctx, sig, [[k] for k in n], max_blocks=2, mark_steps=steps)
        _lockstep(ctx, sig, [_sched(k, 1000) for k in n], max_blocks=1, mark_steps=steps)
        _lockstep(ctx, sig, [_sched(k, 4410) for k in n], alt=True)
    finally:
        d.close()


@pytest.mark.parametrize("name,ch,rate,max_br,nominal,min_br,rm2", MANAGED)
def test_managed_dev_equals_host(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2):
    if not B.ref_available(True):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    cf = B.managed(ch, rate, max_br, nominal, min_br, *(rm2 or ()))
    info, _ = B.ref_bitrate_info(cf)
    d = B.ManagedDriver(ch, rate, max_br, nominal, min_br)
    ctx = d.ctx
    try:
        ctx.bitrate_setup(info)
        sig = _streams(ch, rate, 0.8)
        ws = (1000, 4410)
        _lockstep(ctx, [p for w in ws for p in sig], [_sched(p.shape[1], w) for w in ws for p in sig], managed=True,
                  alt=True)
    finally:
        d.close()


def test_whole_clip_with_first_zero(cuda_ok):
    """every call passes the whole clip with first = 0: the same packets and carries as the host form's sliding
    buffers"""
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        sig = _streams(ch, rate, 0.6)
        ns, L = len(sig), max(p.shape[1] for p in sig)
        clip = np.zeros((ns, ch, L), np.float32)
        for s, p in enumerate(sig):
            clip[s, :, :p.shape[1]] = p
        h = Feed(ctx, sig, [_sched(p.shape[1], 4410) for p in sig])
        carry = ctx.encode_pcm_carry_init(ns)
        for k in range(10000):
            if ctx.encode_pcm_carry_head(h.carry)["enc"]["done"].all():
                break
            head = ctx.encode_pcm_carry_head(h.carry)
            a = h.step()
            # the same write, expressed against the whole clip
            new_head = ctx.encode_pcm_carry_head(h.carry)
            end = (new_head["ended"] & ~head["ended"]).astype(np.int32)
            lens = new_head["written"].astype(np.int64)
            b = dev_call(ctx, clip, lens, carry, end, first=np.zeros(ns, np.int64))
            assert b["rc"] == 0 and b["result"]["rc"] == 0, (k, b["status"])
            carry[:] = b["carry"]
            assert np.array_equal(a["nblocks"], b["nblocks"]) and a["packets"] == b["packets"], k
            for s in range(ns):
                n = int(a["nblocks"][s])
                assert a["info"][s, :n].tobytes() == b["info"][s, :n].tobytes(), k
            assert np.array_equal(h.carry, carry), k
    finally:
        d.close()


def test_device_refusals(cuda_ok):
    """each per-stream refusal sets its status and the call's rc; count > cap, bytes > data_cap and a mark window
    overflow set rc with the need in count / bytes; none writes a packet byte or changes a carry"""
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    other = lib.Context(__import__("conftest").load_setup("44k_mono_q4"))
    try:
        p = _streams(ch, rate, 0.6)[0]
        f = Feed(ctx, [p, p], [[20000, 3000], [20000, 3000]])
        f.step()
        head = ctx.encode_pcm_carry_head(f.carry)
        raw, kept = int(head["raw_base"][0]), int(head["written"][0] - head["raw_base"][0])
        buf = np.ascontiguousarray(np.stack([p[:, raw:raw + kept + 3000]] * 2))

        def refused(lens, end=None, carry=None, stream=0, **kw):
            c = f.carry.copy() if carry is None else carry
            before = c.copy()
            got = dev_call(ctx, buf, np.asarray(lens, np.int64), c, end, sentinel=0xA5, **kw)
            assert got["rc"] == 0
            assert got["result"]["rc"] == VB200_EINVAL
            assert (got["data"] == 0xA5).all(), "packet bytes written"
            assert np.array_equal(got["carry"], before), "carry changed"
            return got

        ok = [kept + 3000, kept + 3000]
        g = refused([kept - 1, kept + 3000])                           # pcm_len below the kept samples
        assert list(g["status"]) == [VB200_EINVAL, 0]
        g = refused([kept + 3000, buf.shape[2] + 1])                   # pcm_len above the stride
        assert list(g["status"]) == [0, VB200_EINVAL]
        g = refused(ok, end=[1, 0])                                    # an end with new samples
        assert list(g["status"]) == [VB200_EINVAL, 0]
        g = refused(ok, first=[raw + 1, raw])                          # first past raw_base
        assert list(g["status"]) == [VB200_EINVAL, 0]
        mixed = f.carry.copy()
        mixed[1, :] = 0
        g = refused(ok, carry=mixed)                                   # a carry of no setup
        assert list(g["status"]) == [0, VB200_EINVAL]
        assert int(g["result"]["bytes"]) > 0 and g["result"]["count"][1] > 0   # the other stream's need is reported
        m = next(m for m in range(1, 4096) if ctx.L.vb200_encode_pcm_carry_bytes(ctx.h, m) == f.carry.shape[1]
                 and not np.array_equal(ctx.encode_pcm_carry_init(1, m), ctx.encode_pcm_carry_init(1)))
        g = refused(ok, carry=ctx.encode_pcm_carry_init(2, m))              # a carry of another mark capacity
        assert list(g["status"]) == [VB200_EINVAL, VB200_EINVAL]
        g = refused(ok, cap=[0, 1])                                    # count > cap
        assert not g["status"].any() and g["result"]["count"][1] > 1
        full = dev_call(ctx, buf, np.asarray(ok, np.int64), f.carry.copy(), None)
        need = int(full["result"]["bytes"])
        assert full["result"]["rc"] == 0 and need > 0
        g = refused(ok, data_cap=need - 1)                             # bytes > data_cap
        assert int(g["result"]["bytes"]) == need and not g["status"].any()
        assert g["info"].tobytes() == full["info"].tobytes()
        # the end-of-stream refusals: an end on an undrained carry, then a second end and samples after the end
        steps = p.shape[1] // 64 + ctx.bs[1] // 16 + 64
        u = Feed(ctx, [p, p], [[p.shape[1]], [p.shape[1]]], max_blocks=2, mark_steps=steps)
        u.step()
        uh = ctx.encode_pcm_carry_head(u.carry)
        assert not uh["drained"].any()
        ulen = (uh["written"] - uh["raw_base"]).astype(np.int64)
        ubuf = np.ascontiguousarray(np.stack([p[:, int(uh["raw_base"][s]):] for s in range(2)]))
        c0 = u.carry.copy()
        g = dev_call(ctx, ubuf, ulen, c0, [1, 0], sentinel=0xA5, max_blocks=2, mark_steps=steps)
        assert g["result"]["rc"] == VB200_EINVAL and list(g["status"]) == [VB200_EINVAL, 0]
        assert (g["data"] == 0xA5).all() and np.array_equal(g["carry"], u.carry)
        u.run()
        uh = ctx.encode_pcm_carry_head(u.carry)
        assert uh["ended"].all()
        ulen = (uh["written"] - uh["raw_base"]).astype(np.int64)
        ubuf = np.zeros((2, ch, int(ulen.max()) + 1), np.float32)
        for end, extra in (([1, 0], 0), ([0, 0], 1)):           # a second end; samples after the end
            g = dev_call(ctx, ubuf, ulen + np.array([extra, 0]), u.carry.copy(), end, sentinel=0xA5, mark_steps=steps)
            assert g["result"]["rc"] == VB200_EINVAL and list(g["status"]) == [VB200_EINVAL, 0], (end, extra)
            assert (g["data"] == 0xA5).all() and np.array_equal(g["carry"], u.carry)
        # a mark window overflow: a carry with room for few marks fed a long write
        small = ctx.encode_pcm_carry_init(2, 8)
        lens = np.array([p.shape[1]] * 2, np.int64)
        whole = np.ascontiguousarray(np.stack([p, p]))
        before = small.copy()
        g = dev_call(ctx, whole, lens, small, None, sentinel=0xA5, mark_steps=8)
        assert g["rc"] == 0 and g["result"]["rc"] == VB200_EINVAL and not g["status"].any()
        assert (g["data"] == 0xA5).all() and np.array_equal(g["carry"], before)
        # the synchronous refusals
        assert ctx.encode_pcm_packets_dev(2, 0, 7, 10, 0, 0, 0, 0, 4, [4, 4], 0, 0, 0, 0, 0, check=False) == VB200_EINVAL
        assert other.encode_pcm_packets_dev(1, 1, lib.PCM_F32_PLANAR, 10, 1, 1, 1, 1, 4, [4, 4], 1, 1, 1, 1, 1,
                                            check=False) == VB200_EINVAL
        assert b"entropy" in other.L.vb200_last_error()
    finally:
        other.close()
        d.close()


def test_managed_carry_before_bitrate_setup(cuda_ok):
    """a managed _dev call on a carry made before the managed bitrate setup: status and rc, carry unchanged"""
    name, ch, rate, max_br, nominal, min_br, rm2 = MANAGED[0]
    if not B.ref_available(True):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    info, _ = B.ref_bitrate_info(B.managed(ch, rate, max_br, nominal, min_br))
    d = B.ManagedDriver(ch, rate, max_br, nominal, min_br)
    ctx = d.ctx
    try:
        early = ctx.encode_pcm_carry_init(1)
        ctx.bitrate_setup(info)
        pcm = np.zeros((1, ch, 5000), np.float32)
        g = dev_call(ctx, pcm, [5000], early, managed=True, sentinel=0xA5)
        assert g["rc"] == 0 and g["result"]["rc"] == VB200_EINVAL and list(g["status"]) == [VB200_EINVAL]
        assert np.array_equal(g["carry"], early) and (g["data"] == 0xA5).all()
    finally:
        d.close()


def test_no_host_wait(cuda_ok):
    """the call returns while the stream is still busy with work queued before it; then its outputs are the host
    form's"""
    torch = _torch()
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        sig = _streams(ch, rate, 0.6)
        ns, n = len(sig), max(p.shape[1] for p in sig)
        clip = np.zeros((ns, ch, n), np.float32)
        for s, p in enumerate(sig):
            clip[s, :, :p.shape[1]] = p
        lens = np.array([p.shape[1] for p in sig], np.int64)
        want = ctx.encode_pcm_packets(clip, lens, ctx.encode_pcm_carry_init(ns))
        max_blocks = (n + 4 * ctx.bs[1]) // (ctx.bs[0] // 2) + 8
        cap = [ns * max_blocks, ns * ((n + 4 * ctx.bs[1]) // (ctx.bs[1] // 2) + 8)]
        data_cap = ns * max_blocks * max(ctx.packet_bound(0), ctx.packet_bound(1))
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()  # noqa: E731
        pcm, dl = t(clip), t(lens)
        z = lambda k: torch.zeros(k, dtype=torch.uint8, device="cuda")  # noqa: E731
        st = torch.cuda.Stream()
        for rep in range(2):                             # a warm-up call at the same sizes, then the timed one
            carry = t(ctx.encode_pcm_carry_init(ns))
            plan, nb = z(ns * max_blocks * abi.STREAM_BLOCK_DTYPE.itemsize), z(4 * ns)
            info, data = z(ns * max_blocks * abi.PACKET_INFO_DTYPE.itemsize), z(data_cap)
            status, res = z(4 * ns), z(abi.ENCODE_RESULT_DTYPE.itemsize)
            torch.cuda.synchronize()
            with torch.cuda.stream(st):
                if rep:
                    torch.cuda._sleep(200_000_000)       # about 100 ms of GPU clock
                ctx.encode_pcm_packets_dev(ns, pcm.data_ptr(), lib.PCM_F32_PLANAR, n, dl.data_ptr(), carry.data_ptr(),
                                           plan.data_ptr(), nb.data_ptr(), max_blocks, cap, info.data_ptr(),
                                           data.data_ptr(), data_cap, status.data_ptr(), res.data_ptr(),
                                           stream=st.cuda_stream)
                busy = not st.query()
            st.synchronize()
            if rep:
                assert busy, "the call waited for the stream"
        r = res.cpu().numpy().view(abi.ENCODE_RESULT_DTYPE)[0]
        assert r["rc"] == 0 and list(r["count"]) == list(want["count"])
        got_info = info.cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(ns, max_blocks)
        got_nb = nb.cpu().numpy().view(np.int32)
        got_data = data.cpu().numpy()
        assert np.array_equal(got_nb, want["nblocks"])
        for s in range(ns):
            pk = [bytes(got_data[i["offset"]:i["offset"] + i["bytes"]]) for i in got_info[s, :got_nb[s]]]
            assert pk == want["packets"][s], s
    finally:
        d.close()


def test_dev_round_trip_decode(cuda_ok):
    """_dev encode, then vb200_decode_streams_packets_dev on the same device buffers: the stock decoder's output of
    the same packets (which are the stock encoder's for these writes, test_dev_equals_host)"""
    from oracle import decode
    from oracle import decode_packets as dp
    from oracle import decode_streams as ds
    torch = _torch()
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    sig = _streams(ch, rate, 0.6)[:2]
    stock = decode.encode(ch, rate, q, sig[0])              # its header packets set the decoder up
    dec = dp.Driver(decode.Packets(stock.buf, stock.meta))
    try:
        ctx, dctx = d.ctx, dec.ctx
        ns = len(sig)
        lens = np.array([p.shape[1] for p in sig], np.int64)
        clip = np.zeros((ns, ch, int(lens.max())), np.float32)
        for s, p in enumerate(sig):
            clip[s, :, :p.shape[1]] = p
        carry = ctx.encode_pcm_carry_init(ns)
        dcarry = dctx.decode_streams_carry(ns)
        pcm, pk, inf = [[] for _ in range(ns)], [[] for _ in range(ns)], [[] for _ in range(ns)]
        for end in (None, [1] * ns):
            g = dev_call(ctx, clip, lens, carry, end, first=np.zeros(ns, np.int64), keep=True)
            assert g["rc"] == 0 and g["result"]["rc"] == 0
            carry[:] = g["carry"]
            dv, mb = g["dev"], g["info"].shape[1]
            pcm_cap = int(g["nblocks"].sum()) * (ctx.bs[1] // 2) * ch
            d_pcm = torch.zeros(max(pcm_cap, 1), dtype=torch.float32, device="cuda")
            d_base = torch.zeros(ns + 1, dtype=torch.int64, device="cuda")
            d_out = torch.zeros(ns * mb * abi.DECODED_PACKET_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            dctx.decode_streams_packets_dev(ns, mb, dv["nb"].data_ptr(), dv["info"].data_ptr(), dv["data"].data_ptr(),
                                            dcarry.ptr, 0, d_pcm.data_ptr(), pcm_cap, d_base.data_ptr(),
                                            d_out.data_ptr())
            torch.cuda.synchronize()
            base, out = d_base.cpu().numpy(), d_pcm.cpu().numpy()
            for s in range(ns):
                pcm[s].append(out[base[s] * ch:base[s + 1] * ch].reshape(ch, -1))
                pk[s] += g["packets"][s]
                inf[s] += list(g["info"][s, :g["nblocks"][s]])
        hdr = np.ascontiguousarray(stock.meta[:3])
        hbuf = bytes(stock.buf[:int(hdr[2, 0] + hdr[2, 1])])
        for s in range(ns):
            got = np.concatenate(pcm[s], axis=1)
            buf, rows, off = bytearray(hbuf), [], len(hbuf)
            for b, r in zip(pk[s], inf[s]):
                rows.append([off, len(b), r["granulepos"], r["e_o_s"], r["packetno"]])
                buf += b
                off += len(b)
            want, _, _ = ds.ref_decode(np.frombuffer(bytes(buf), np.uint8), hdr, np.array(rows, np.int64), ch)
            assert got.shape == want.shape, (s, got.shape, want.shape)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), s
    finally:
        dec.close()
        d.close()
