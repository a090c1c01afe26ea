"""Raw PCM to packets (vb200_encode_pcm_packets[_managed], vb200_lpc_extrapolate): the LPC kernels equal the
reference's vorbis_lpc_from_data / vorbis_lpc_predict bit for bit, and raw float or int16 PCM fed with one call per
stock write gives the stock encoder's packets, granulepos, e_o_s and packetno.  The stock-encoder comparisons need
oracle/_ref (built where the reference sources exist; the libraries travel)."""
import ctypes as C

import numpy as np
import pytest

from oracle import bitrate as B
from oracle import lpc
from test_gpu_encode_packets import SETUPS, _driver
from test_gpu_stream_packets import MANAGED, _need_ref, _noise_and_silence, _streams
from test_pcm_timeline_oracle import KINDS, LENGTHS, lpc_signal
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

VB200_EINVAL = -131
LONG_SETUP = (2, 44100, -0.1)          # 512/4096


def _to_s16(pcm):
    """int16 [n][ch] of pcm [ch][n], and the float input encoder_example makes of it (x / 32768.f)"""
    q = np.clip(np.round(pcm * 32767.0), -32768, 32767).astype(np.int16)
    return np.ascontiguousarray(q.T), (q.astype(np.float32) / np.float32(32768.0)).astype(np.float32)


def _sched(n, w):
    """the stock writes of ref_stream_capture(chunk=w) for n samples (w None: all at once)"""
    w = w or max(n, 1)
    return [w] * (n // w) + ([n % w] if n % w else [])


class Feed:
    """streams fed through encode_pcm_packets: stream s writes sched[s] one piece per call, then ends; a carry that
    max_blocks left undrained gets drain calls (no new samples) first.  Collects packets and infos per stream."""

    def __init__(self, ctx, pcms, scheds, managed=False, s16=False, max_blocks=None, mark_steps=0):
        self.ctx, self.pcms, self.scheds, self.managed, self.s16 = ctx, pcms, scheds, managed, s16
        self.max_blocks = max_blocks
        self.ns, self.ch = len(pcms), pcms[0].shape[0]
        self.carry = ctx.encode_pcm_carry_init(self.ns, mark_steps)
        self.idx = [0] * self.ns
        self.pk, self.inf = [[] for _ in range(self.ns)], [[] for _ in range(self.ns)]

    def step(self, new=None, end=None, **kw):
        """one call: new[s] samples for stream s and end[s] (default: the next write, drain or end)"""
        head = self.ctx.encode_pcm_carry_head(self.carry)
        if new is None:
            new, end = np.zeros(self.ns, np.int64), np.zeros(self.ns, np.int32)
            for s in range(self.ns):
                if not head["drained"][s]:
                    continue
                if self.idx[s] < len(self.scheds[s]):
                    new[s] = self.scheds[s][self.idx[s]]
                    self.idx[s] += 1
                elif not head["ended"][s]:
                    end[s] = 1
        raw, wr = head["raw_base"], head["written"]
        lens = wr + np.asarray(new, np.int64) - raw
        stride = max(int(lens.max()), 1)
        if self.s16:
            buf = np.zeros((self.ns, stride, self.ch), np.int16)
            for s in range(self.ns):
                buf[s, :lens[s]] = self.pcms[s][:, raw[s]:raw[s] + lens[s]].T
        else:
            buf = np.zeros((self.ns, self.ch, stride), np.float32)
            for s in range(self.ns):
                buf[s, :, :lens[s]] = self.pcms[s][:, raw[s]:raw[s] + lens[s]]
        got = self.ctx.encode_pcm_packets(buf, lens, self.carry, end, managed=self.managed,
                                          max_blocks=kw.pop("max_blocks", self.max_blocks), **kw)
        if "rc" in got and got["rc"]:
            return got
        for s in range(self.ns):
            n = int(got["nblocks"][s])
            self.pk[s] += got["packets"][s] if "packets" in got else []
            self.inf[s] += list(got["info"][s, :n])
        return got

    def run(self, rounds=100000):
        for _ in range(rounds):
            if self.ctx.encode_pcm_carry_head(self.carry)["enc"]["done"].all():
                return self
            self.step()
        raise AssertionError("streams not done")


def _vs(feed, caps, what):
    for s, c in enumerate(caps):
        assert feed.pk[s] == c["packets"], "%s stream %d: packets (%d vs %d)" % (what, s, len(feed.pk[s]), len(c["packets"]))
        for f in ("granulepos", "e_o_s", "packetno"):
            assert np.array_equal(np.array([r[f] for r in feed.inf[s]], np.int64), c[f]), "%s stream %d: %s" % (what, s, f)


def test_lpc_extrapolate_equals_reference(cuda_ok):
    """vb200_lpc_extrapolate on the rows of the CPU test: coefficients and 3*2048 predicted samples bit for bit"""
    if not lpc.ref_available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ctx = lib.Context(__import__("conftest").load_setup("44k_stereo_q5"))
    try:
        for m in (16, 32):
            for n in LENGTHS:
                rows = np.stack([lpc_signal(k, n) for k in KINDS])
                coef, out = ctx.lpc_extrapolate(rows, np.full(len(KINDS), n, np.int32), m, 3 * 2048)
                for i, k in enumerate(KINDS):
                    c0, y0 = lpc.ref_extrapolate(rows[i], m, 3 * 2048)
                    assert np.array_equal(coef[i].view(np.uint32), c0.view(np.uint32)), "%s m=%d n=%d" % (k, m, n)
                    assert np.array_equal(out[i].view(np.uint32), y0.view(np.uint32)), "%s m=%d n=%d" % (k, m, n)
        assert ctx.lpc_extrapolate(rows, np.full(len(KINDS), 8, np.int32), 32, 4, check=False) == VB200_EINVAL
        assert ctx.lpc_extrapolate(rows, np.full(len(KINDS), 64, np.int32), 24, 4, check=False) == VB200_EINVAL
    finally:
        ctx.close()


@pytest.mark.parametrize("ch,rate,q", SETUPS + [LONG_SETUP])
def test_one_call_per_stock_write(cuda_ok, ch, rate, q):
    """float planar and int16 interleaved PCM, one call per write of 64, 1000, 1024, 4410 samples or all at once:
    the stock encoder's packets, granulepos, e_o_s and packetno, streams at different phases in every call"""
    _need_ref()
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        if (ch, rate, q) == LONG_SETUP:
            assert list(ctx.bs) == [512, 4096]
        sig = _streams(ch, rate, 0.6)
        ws = (64, 1000, 1024, 4410, None)
        for s16 in (False, True):
            pcms, feeds, caps = [], [], []
            for w in ws:
                for p in sig:
                    if s16:
                        q16, p = _to_s16(p)
                        feeds.append(q16.T)
                    else:
                        feeds.append(p)
                    pcms.append(p)
                    caps.append(B.ref_stream_capture(B.vbr(ch, rate, q), p, chunk=w or max(p.shape[1], 1)))
            scheds = [_sched(p.shape[1], w) for w in ws for p in sig]
            f = Feed(ctx, feeds, scheds, s16=s16).run()
            _vs(f, caps, "q=%g %s" % (q, "s16" if s16 else "f32"))
    finally:
        d.close()


@pytest.mark.parametrize("name,ch,rate,max_br,nominal,min_br,rm2", MANAGED)
def test_managed_one_call_per_stock_write(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2):
    """bitrate-managed, including the small-reservoir CBR case with cut and padded packets; a carry made before the
    managed bitrate setup is refused"""
    _need_ref()
    if not B.ref_available(True):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    cf = B.managed(ch, rate, max_br, nominal, min_br, *(rm2 or ()))
    info, _ = B.ref_bitrate_info(cf)
    d = B.ManagedDriver(ch, rate, max_br, nominal, min_br)
    ctx = d.ctx
    try:
        early = Feed(ctx, [np.zeros((ch, 5000), np.float32)], [[5000]], managed=True)
        ctx.bitrate_setup(info)
        before = early.carry.copy()
        assert early.step(check=False)["rc"] == VB200_EINVAL
        assert np.array_equal(early.carry, before)
        sig = _streams(ch, rate, 0.8)
        if rm2:
            sig = [_noise_and_silence(ch, rate, 1.5, 1), _noise_and_silence(ch, rate, 1.0, 2)] + sig
        ws = (1000, 4410)
        caps = [B.ref_stream_capture(cf, p, chunk=w) for w in ws for p in sig]
        f = Feed(ctx, [p for w in ws for p in sig], [_sched(p.shape[1], w) for w in ws for p in sig], managed=True).run()
        _vs(f, caps, name)
    finally:
        d.close()


def test_only_the_crossing_write_matters(cuda_ok):
    """calls that copy the stock writes until blocksizes[1] samples are crossed, then take arbitrary pieces (larger and
    smaller, some empty), give the stock encoder's packets; short and silent streams, and streams of 0 to
    blocksizes[1] + 1 samples, in the same calls"""
    _need_ref()
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    rng = np.random.default_rng(7)
    try:
        bs1 = ctx.bs[1]
        sig = _streams(ch, rate, 1.5)
        from conftest import probe_signal
        short = [probe_signal(ch, rate, 0.2, seed=n)[:, :n] for n in (0, 1, 32, 33, 64, 65, bs1, bs1 + 1)]
        pcms, scheds, caps = [], [], []
        for w in (1000, 4410):
            for p in sig + short:
                n = p.shape[1]
                stock = _sched(n, w)
                k = 0
                while k < len(stock) and sum(stock[:k]) <= bs1:
                    k += 1
                rest, pieces = n - sum(stock[:k]), []
                while rest > 0:
                    pieces.append(min(rest, int(rng.choice([0, 1, 63, 5000, 30000]))))
                    rest -= pieces[-1]
                pcms.append(p)
                scheds.append(stock[:k] + pieces)
                caps.append(B.ref_stream_capture(B.vbr(ch, rate, q), p, chunk=w))
        f = Feed(ctx, pcms, scheds).run()
        _vs(f, caps, "pieces")
        # the same streams written as the stock writes, for contrast, in one batch with the pieces
        f2 = Feed(ctx, pcms + pcms, scheds + [_sched(p.shape[1], w) for w in (1000, 4410) for p in sig + short]).run()
        _vs(f2, caps + caps, "mixed")
    finally:
        d.close()


def test_max_blocks_and_undrained_end(cuda_ok):
    """max_blocks cuts: an end on an undrained carry is refused and leaves the carry byte for byte; after drain calls
    the end is taken and the streams give the stock encoder's packets"""
    _need_ref()
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        sig = _streams(ch, rate, 0.6)[:2]
        n = [p.shape[1] for p in sig]
        steps = max(n) // 64 + ctx.bs[1] // 16 + 64
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p, chunk=p.shape[1]) for p in sig]
        f = Feed(ctx, sig, [[k] for k in n], max_blocks=2, mark_steps=steps)
        f.step()
        head = ctx.encode_pcm_carry_head(f.carry)
        assert not head["drained"].any() and not head["ended"].any()
        before = f.carry.copy()
        got = f.step(new=np.zeros(2, np.int64), end=np.ones(2, np.int32), check=False)
        assert got["rc"] == VB200_EINVAL and np.array_equal(f.carry, before)
        f.run()
        _vs(f, caps, "max_blocks=2")
        g = Feed(ctx, sig, [_sched(k, 1000) for k in n], max_blocks=1, mark_steps=steps).run()
        _vs(g, [B.ref_stream_capture(B.vbr(ch, rate, q), p, chunk=1000) for p in sig], "max_blocks=1")
    finally:
        d.close()


def test_errors_and_launches(cuda_ok):
    """VB200_EINVAL, each leaving every carry as it was: another pcm format, pcm_len below the kept samples or above
    the stride, an end with new samples, a second end, samples after the end, a carry of another setup; launches per
    call do not grow with the stream count"""
    _need_ref()
    ch, rate, q = 2, 44100, 0.5
    d = _driver(ch, rate, q)
    ctx = d.ctx
    other = lib.Context(__import__("conftest").load_setup("44k_mono_q4"))
    try:
        p = _streams(ch, rate, 0.6)[0]
        f = Feed(ctx, [p], [[20000, 3000]])
        f.step()
        head = ctx.encode_pcm_carry_head(f.carry)
        assert head["written"][0] == 20000 and head["enc"]["base"][0] > 0 and head["raw_base"][0] > 0
        kept = int(head["written"][0] - head["raw_base"][0])
        before = f.carry.copy()
        buf = np.ascontiguousarray(p[None, :, head["raw_base"][0]:head["raw_base"][0] + kept + 3000])

        def rc(lens, end=None, pcm=buf, carry=f.carry):
            return ctx.encode_pcm_packets(pcm, np.array([lens], np.int64), carry,
                                          None if end is None else np.array([end], np.int32), check=False)["rc"]
        assert rc(kept - 1) == VB200_EINVAL
        assert rc(buf.shape[2] + 1) == VB200_EINVAL
        assert rc(kept + 10, end=1) == VB200_EINVAL
        assert rc(kept, pcm=buf, carry=other.encode_pcm_carry_init(1)) == VB200_EINVAL
        io = abi.PcmIO()
        io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = buf.ctypes.data, 7, 64, buf.shape[2]
        lens = np.array([kept], np.int64)
        io.pcm_len = lens.ctypes.data
        plan, nbk = np.zeros((1, 64), abi.STREAM_BLOCK_DTYPE), np.zeros(1, np.int32)
        io.plan, io.nblocks = plan.ctypes.data, nbk.ctypes.data
        io.cap[0] = io.cap[1] = 64
        info, data = np.zeros(64, abi.PACKET_INFO_DTYPE), np.zeros(1 << 20, np.uint8)
        assert ctx.L.vb200_encode_pcm_packets(ctx.h, 1, 7, C.byref(io), f.carry.ctypes.data, info.ctypes.data,
                                              data.ctypes.data, data.size) == VB200_EINVAL
        assert np.array_equal(f.carry, before)
        assert rc(kept, end=1) == 0                      # the end
        head = ctx.encode_pcm_carry_head(f.carry)
        assert head["ended"][0] and head["enc"]["done"][0]
        kept = int(head["written"][0] - head["raw_base"][0])
        before = f.carry.copy()
        assert rc(kept, end=1) == VB200_EINVAL           # a second end
        assert rc(kept + 1) == VB200_EINVAL              # samples after the end
        assert np.array_equal(f.carry, before)
        # launches: the same count for 2 and 12 streams at the same phase
        counts = []
        for ns in (2, 12):
            g = Feed(ctx, [p] * ns, [[20000]] * ns)
            l0 = ctx.launch_count()
            g.step()
            counts.append(ctx.launch_count() - l0)
        assert counts[0] == counts[1] <= 44, counts
    finally:
        other.close()
        d.close()
