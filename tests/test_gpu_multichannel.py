"""Every device path on the uncoupled setups vorbisenc picks for channel counts other than 1, 2 and 6 (quad, 5.0, 7.1,
odd counts), and the channel-count limits of the device.  Bit-exact.

vorbisenc serves every count but 2 and 6 from its uncoupled templates (ve_setup_{44,32,22}_uncoupled): one submap
with every channel on it, no coupling steps, and type-1 residue over several channels.  There res1_class and
res1_forward drop the channels whose nonzero flag is 0 and keep the others in order, so the u-th residue vector is
the u-th *used* channel; with one channel per submap (mono, the LFE submap of 5.1) that compaction never shows.  The
s16 staging of the transform, the k_cqn fallback, interleaved int16 output at odd channel counts, bitrate management
(vorbisenc divides the requested rate by the channel count) and every buffer sized by the channel count run at
counts no other test reaches.

- The setup-family suite of tests/setup_families.py on the rows of FAMILY: the stages against the oracle, which
  tests/test_oracle_vs_ref.py pins to the reference at these setups (MULTI), fed the blocks the reference encoder cut
  from its chain stream (tests/golden/ref), and packets and PCM against the stock encoder and decoder.
- Content built so that the reference itself exercises the compaction: a silent channel between used ones, a channel
  that starts late, a copied channel, a full-scale int16 square wave, a 40 Hz sine and a stretch where every channel
  is silent.  The tests assert that the reference's capture holds those cases, then compare residue, classes, packets
  and PCM with the stock encoder and decoder.
- The classes layout of vb200_residue_classify: rows by channel, zero for unused channels, equal to what the
  reference's rows by used index map back to.
- Against the stock encoder and decoder (needs oracle/_ref) at every MULTI setup, for two managed rates, and at 24,
  79, 80 and 255 channels: 79 is the last count the coupling kernel takes, and 80 is refused with VB200_EIMPL."""
import numpy as np
import pytest

import refgold as G
import test_gpu_decode_packets as DP
import test_gpu_decode_ranges as DR
import test_gpu_decode_streams as DS
import test_gpu_encode_packets as EP
import test_gpu_pcm_packets as PC
import test_gpu_stream_packets as SP
import test_oracle_vs_ref as T
from conftest import assert_bits_equal, probe_signal
from oracle import bitrate as B
from oracle import decode, pyoracle, pyref
from oracle import decode_packets as dp
from oracle import decode_streams as ds
from setup_families import *  # noqa: F401,F403  (the suite's tests and fixtures, among them drivers)
from setup_families import Family
from test_decode_streams_oracle import make_streams
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu

MULTI = T.MULTI
# per setup: block sizes and (type, begin, end, grouping, partitions) of the residue for W = 0 and 1, read from the
# stored setups; every one has no coupling steps and one submap holding every channel
FEATURES = {
    (3, 44100, 0.4): ([256, 2048], [(1, 0, 112, 16, 8), (1, 0, 896, 32, 8)]),
    (4, 48000, 0.1): ([256, 2048], [(1, 0, 96, 16, 8), (1, 0, 672, 32, 8)]),
    (5, 44100, 0.9): ([256, 2048], [(1, 0, 128, 16, 10), (1, 0, 1024, 32, 10)]),
    (8, 48000, 0.3): ([256, 2048], [(1, 0, 96, 16, 8), (1, 0, 736, 32, 8)]),
    (8, 44100, -0.1): ([512, 4096], [(1, 0, 160, 32, 8), (1, 0, 1312, 32, 8)]),
    (4, 32000, 0.2): ([256, 2048], [(1, 0, 112, 16, 8), (1, 0, 896, 32, 8)]),
    (3, 22050, 0.3): ([512, 1024], [(1, 0, 256, 32, 10), (1, 0, 512, 32, 10)]),
}
EIMPL = -130


def _residue(setup, W):
    return setup.c.residue[W][0]


def check_features(setup, args):
    """the setup has the structure this family is about, so that a vorbisenc change cannot turn the tests into a
    repeat of the mono ones"""
    bs, res = FEATURES[args]
    ch = args[0]
    assert setup.channels == ch
    assert [setup.blocksize(0), setup.blocksize(1)] == bs
    assert list(setup.c.coupling_steps) == [0, 0] and list(setup.c.submaps) == [1, 1]
    for W in (0, 1):
        assert list(setup.c.chmux[W])[:ch] == [0] * ch, "W=%d chmux" % W
        r = _residue(setup, W)
        got = (r.type, r.begin, r.end, r.grouping, r.partitions)
        assert got == res[W], "W=%d residue %s" % (W, got)


# name, channels, rate, max, nominal and min bitrate, the small-reservoir settings, and the VBR quality whose template
# vorbisenc picks for the nominal rate per channel (64 and 96 kbit/s on rate_mapping_44_un)
MANAGED = [("abr512_71", 8, 48000, -1, 512000, -1, None, 0.14),
           ("cbr384_quad", 4, 44100, 384000, 384000, 384000, None, 0.5)]
FAMILY = Family(
    name="multi", setups=MULTI, capture={}, check=check_features, blocksizes=lambda args: FEATURES[args][0],
    nvec=[[133]], fmts=[["f32", "s16"]], envelope=[MULTI],
    rows={"test_stock_encoder_packets": MULTI, "test_stock_decoder": MULTI, "test_stock_halfrate_decoder": MULTI,
          "test_function_level_dropin": MULTI,
          "test_stock_managed_encoder": [pytest.param(*m[:7], id="-".join(map(str, m))) for m in MANAGED]},
    uncoupled_q={m[0]: m[7] for m in MANAGED})


# ---- the classes layout ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("args", [(3, 44100, 0.4), (8, 44100, -0.1)], ids=lambda a: G.case_id(*a))
def test_classes_rows_by_channel(cuda_ok, args):
    """type-1 residue classifies each used channel on its own, so row c of a call is the row c of a call where only c
    is used: the reference's rows by used index, mapped back, and the oracle's and the device's rows by channel.  The
    rows of unused channels are zero, including in a device buffer that held other values; so are entries past
    partvals"""
    import torch
    setup = G.load_setup(*args)
    ch = args[0]
    o = pyoracle.Oracle(setup)
    ctx = vlib.Context(setup)
    ref = pyref.Ref(*args) if pyref.available() else None
    try:
        rng = np.random.default_rng(ch)
        for W in (0, 1):
            n, nb = setup.blocksize(W) // 2, 12
            pv = ctx.residue_partvals(W)
            iwork = np.rint(rng.standard_normal((nb, ch, n)) * np.exp(rng.uniform(-1, 3, (nb, ch, 1)))).astype(np.int32)
            nz = (rng.random((nb, ch)) < 0.6).astype(np.int32)
            nz[0] = 0
            nz[1] = 1
            nz[2] = np.arange(ch) % 2 == 0              # silent channels between used ones
            nz[3] = np.arange(ch) % 2 == 1
            nz[4] = 0
            nz[4, ch - 1] = 1                           # the last channel alone: used index 0
            got = ctx.residue_classify(W, iwork, nz)
            want = o.residue_classify(W, iwork, nz)
            assert np.array_equal(got, want), "W=%d device vs oracle" % W
            if ref is not None:
                assert np.array_equal(ref.residue_classify(W, iwork, nz, pv), want), "W=%d reference vs oracle" % W
            assert not got[nz == 0].any(), "W=%d rows of unused channels" % W
            assert (got[nz == 1] > 0).any()
            for c in range(ch):
                solo = np.zeros_like(nz)
                solo[:, c] = nz[:, c]
                alone = ctx.residue_classify(W, iwork, solo)
                assert np.array_equal(alone[:, c], got[:, c]), "W=%d channel %d alone" % (W, c)
                if ref is not None:
                    assert np.array_equal(ref.residue_classify(W, iwork, solo, pv)[:, c], got[:, c]), \
                        "W=%d reference, channel %d alone" % (W, c)
            dev = torch.device("cuda")
            d_cls = torch.full((nb, ch, pv + 3), -7, dtype=torch.int32, device=dev)
            d_iw, d_nz = torch.from_numpy(iwork).to(dev), torch.from_numpy(nz).to(dev)
            torch.cuda.synchronize()
            ctx.residue_classify_dev(W, nb, d_iw.data_ptr(), d_nz.data_ptr(), d_cls.data_ptr(), pv + 3)
            torch.cuda.synchronize()
            wide = d_cls.cpu().numpy()
            assert np.array_equal(wide[:, :, :pv], got) and not wide[:, :, pv:].any(), "W=%d _dev form" % W
    finally:
        ctx.close()
        if ref is not None:
            ref.close()


# ---- multichannel content -------------------------------------------------------------------------------------------
def multi_signal(ch, rate, seed=0):
    """one second per channel: 0 the probe, 1 digital silence, 2 silent for the first half and then noise at +-0.9,
    3 a copy of channel 0, 4 a full-scale int16 square wave, 5 a 40 Hz sine, further channels probes of their own.
    With fewer than six channels, channel 0 carries the 40 Hz sine under the probe and the square wave after the
    middle.  Every channel is silent from 0.7 s to 0.9 s."""
    rng = np.random.default_rng(seed)
    n = rate
    t = np.arange(n)
    probe = probe_signal(ch, rate, 1.0, seed=seed)[:, :n]
    square = np.where((t // max(1, rate // 2000)) % 2 == 0, 32767, -32768) / 32768.0
    lfe = 0.8 * np.sin(2 * np.pi * 40 * t / rate)
    pcm = probe.astype(np.float64)
    if ch < 6:
        pcm[0] = 0.6 * probe[0] + 0.3 * lfe
        pcm[0, n // 2:] = square[n // 2:]
    pcm[1] = 0
    pcm[2] = 0
    pcm[2, n // 2:] = rng.uniform(-0.9, 0.9, n - n // 2)
    if ch > 3:
        pcm[3] = pcm[0]
    if ch > 4:
        pcm[4] = square
    if ch > 5:
        pcm[5] = lfe
    pcm[:, int(0.7 * rate):int(0.9 * rate)] = 0
    return pcm.astype(np.float32)


def _check_content(setup, nonzero, classes_by_W):
    """the reference's capture holds what the content is for"""
    ch = setup.channels
    gap = any(nz[c] == 0 and nz[:c].any() and nz[c + 1:].any() for nz in nonzero for c in range(1, ch - 1))
    assert gap, "no block with an unused channel between used ones"
    assert (nonzero.sum(axis=1) == 0).any(), "no block without a used channel"
    counts = np.zeros(_residue(setup, 0).partitions, np.int64)
    last = 0
    for W, (cls, nz) in classes_by_W.items():
        r = _residue(setup, W)
        p = (r.end - r.begin) // r.grouping
        rows = cls[nz == 1][:, :p]
        counts += np.bincount(rows.ravel(), minlength=r.partitions)[:r.partitions]
        last += int((rows[:, p - 1] > 0).sum())
    top = len(counts) - 1
    assert (counts[top - 2:] > 0).all(), "top classes not reached: %s" % counts
    assert last > 0, "the last partition is silent in every block"


@pytest.mark.parametrize("args", MULTI, ids=lambda a: G.case_id(*a))
def test_content_vs_stock_encoder(cuda_ok, args):
    """the stock encoder's blocks of the multichannel content: the device chain gives its residue, nonzero flags and
    partition classes (zero rows for unused channels), and through encode_dsp + encode_entropy and encode_packets its
    audio packets; whole streams in float and int16 give its packets"""
    ch, rate, q = args
    d = EP._driver(ch, rate, q)
    ctx = d.ctx
    try:
        setup = G.load_setup(*args)                   # the driver's setup: tests/test_oracle_vs_ref.py pins it
        check_features(setup, args)
        pcm = multi_signal(ch, rate)
        ref = pyref.Ref(ch, rate, q)
        cap = ref.encode_capture(pcm, fields=("pcm", "iwork_out"))
        pk = ref.packets()
        want = pk[len(pk) - cap["nblocks"]:]
        o = pyoracle.Oracle(setup)
        seen = {}
        for W in (0, 1):
            sel = cap["W"] == W
            n, stride = ctx.bs[W] // 2, o.residue_partvals(W)
            blocks = np.ascontiguousarray(cap["pcm"][sel][:, :, :ctx.bs[W]])
            desc = EP._desc(cap, sel)
            wnz = cap["nonzero_out"][sel]
            wcls = ref.residue_classify(W, cap["iwork_out"][sel][:, :, :n], wnz, stride)
            seen[W] = (wcls, wnz)
            got = ctx.encode_dsp(W, blocks, desc, classes=True)
            assert np.array_equal(got["iwork"], cap["iwork_out"][sel][:, :, :n]), "W=%d residue" % W
            assert np.array_equal(got["nonzero"], wnz), "W=%d nonzero" % W
            assert np.array_equal(got["classes"], wcls), "W=%d classes" % W
            assert not got["classes"][wnz == 0].any(), "W=%d rows of unused channels" % W
            wp = [p for p, s in zip(want, sel) if s]
            ent = ctx.encode_entropy(W, desc, got["posts"], got["nonzero"], got["iwork"])
            assert ent["packets"] == wp, "W=%d packets (encode_entropy)" % W
            assert ctx.encode_packets(W, blocks, desc)["packets"] == wp, "W=%d packets (encode_packets)" % W
        ref.close()
        _check_content(setup, cap["nonzero_out"][:cap["nblocks"]], seen)
        q16, pf = PC._to_s16(pcm)
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p) for p in (pcm, pf)]
        tl, pcm_len, eof = SP._timelines(caps, ch)
        SP._compare(ctx.encode_streams_packets(tl, pcm_len, eof), caps, "content timelines")
        # the int16 samples themselves, as raw interleaved PCM in one call (the stock encoder in one write)
        feed = PC.Feed(ctx, [q16.T], [PC._sched(pcm.shape[1], None)], s16=True).run()
        PC._vs(feed, [B.ref_stream_capture(B.vbr(ch, rate, q), pf, chunk=pcm.shape[1])], "content int16 PCM")
    finally:
        d.close()


@pytest.mark.parametrize("args", MULTI, ids=lambda a: G.case_id(*a))
def test_content_vs_stock_decoder(cuda_ok, drivers, args):  # noqa: F811
    """the stock encoder's packets of the multichannel content: the device's entropy decode stages the reference's
    residue, posts and floor flags, and the whole-stream decode gives the stock decoder's PCM in float and int16"""
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ch, rate, q = args
    p = decode.encode(ch, rate, q, multi_signal(ch, rate, seed=1))
    drv = dp.Driver(p)
    try:
        assert drv.on_device
        DP._check(p, drv, DP._pkts(p), "content")
    finally:
        drv.close()
    ctx = DS._ctx(drivers, p.buf, p.hdr)
    audios = [p.audio]
    want = DS._stock(p.buf, p.hdr, audios, ch)
    npkt, info = DS._table(audios)
    for s16 in (False, True):
        got = ctx.decode_streams_packets(npkt, info, p.buf, ctx.decode_streams_carry(1), s16=s16)
        DS._check(got, want, ch, s16, "content s16=%s" % s16)


# ---- odd channel counts ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_stride", [4097, 11025])
@pytest.mark.parametrize("args", [(3, 44100, 0.4), (5, 44100, 0.9), (3, 22050, 0.3)], ids=lambda a: G.case_id(*a))
def test_odd_channels_and_odd_out_stride(cuda_ok, drivers, args, out_stride):  # noqa: F811
    """int16 frames of an odd channel count at an odd out_stride, and float rows: every request equals the slice of
    the stock decoder's PCM"""
    DS._need()
    ch, rate, q = args
    buf, hdr, audios = make_streams(ch, rate, q)
    ctx = DS._ctx(drivers, buf, hdr)
    whole = DR._stock(buf, hdr, audios, ch)
    idx = ctx.decode_streams_index(*DS._table(audios), buf)
    req = DR._requests(audios, whole, idx, out_stride, np.random.default_rng(out_stride + ch))
    npkt, info = DS._table(audios)
    for s16 in (False, True):
        DR._check_ranges(ctx.decode_ranges(npkt, info, buf, req, out_stride, s16=s16), req, whole, s16,
                         "%d channels, out_stride %d s16=%s" % (ch, out_stride, s16))


# ---- many channels --------------------------------------------------------------------------------------------------
MANY_RATE, MANY_Q = 44100, 0.4


def _many_signal(ch, seed=0):
    """a quarter second: probes, every third channel silent"""
    pcm = probe_signal(ch, MANY_RATE, 0.25, seed=seed)
    pcm[1::3] = 0
    return pcm


def test_24_channels(cuda_ok, drivers):  # noqa: F811
    """24 channels: the stock encoder's captured blocks give its packets, whole streams its packets, and the decode
    of its packets its PCM in float and int16"""
    ch = 24
    pcm = _many_signal(ch)
    d = EP._driver(ch, MANY_RATE, MANY_Q)
    ctx = d.ctx
    try:
        cap, want = EP._capture(ch, MANY_RATE, MANY_Q, pcm)
        for W in (0, 1):
            sel = cap["W"] == W
            assert sel.any()
            blocks = np.ascontiguousarray(cap["pcm"][sel][:, :, :ctx.bs[W]])
            wp = [p for p, s in zip(want, sel) if s]
            assert ctx.encode_packets(W, blocks, EP._desc(cap, sel))["packets"] == wp, "W=%d packets" % W
        caps = [B.ref_stream_capture(B.vbr(ch, MANY_RATE, MANY_Q), pcm)]
        SP._compare(ctx.encode_streams_packets(*SP._timelines(caps, ch)), caps, "24 channels")
    finally:
        d.close()
    DS._need()
    p = decode.encode(ch, MANY_RATE, MANY_Q, _many_signal(ch, seed=1))
    dctx = DS._ctx(drivers, p.buf, p.hdr)
    want = [ds.ref_decode(p.buf, p.hdr, p.audio, ch, cap=1 << 15)]
    npkt, info = DS._table([p.audio])
    for s16 in (False, True):
        DS._check(dctx.decode_streams_packets(npkt, info, p.buf, dctx.decode_streams_carry(1), s16=s16), want, ch, s16,
                  "24 channels s16=%s" % s16)


def test_79_channels_stream_encoder(cuda_ok):
    """79 channels, the most the coupling kernel's shared memory takes: the unmanaged stream encoder gives the stock
    encoder's packets"""
    ch = 79
    SP._need_ref()
    d = EP._driver(ch, MANY_RATE, MANY_Q)
    try:
        caps = [B.ref_stream_capture(B.vbr(ch, MANY_RATE, MANY_Q), _many_signal(ch))]
        SP._compare(d.ctx.encode_streams_packets(*SP._timelines(caps, ch)), caps, "79 channels")
    finally:
        d.close()


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


def test_80_channels_refused(cuda_ok, monkeypatch):
    """80 channels: every encode entry point returns VB200_EIMPL with the coupling kernel's "too many channels", writes
    none of its outputs and leaves its carries as they were, and the context then synthesises PCM as the oracle does"""
    import torch
    ch, rate, q = 80, MANY_RATE, MANY_Q
    SP._need_ref()
    cap = B.ref_stream_capture(B.vbr(ch, rate, q), _many_signal(ch))
    tl, pcm_len, eof = SP._timelines([cap], ch)
    r = pyref.Ref(ch, rate, q)
    setup = r.setup()
    blk = r.encode_capture(_many_signal(ch)[:, :8192], fields=("pcm",))
    r.close()
    d = EP._driver(ch, rate, q)
    ctx = d.ctx
    try:
        W = 1
        sel = blk["W"] == W
        blocks = np.ascontiguousarray(blk["pcm"][sel][:, :, :ctx.bs[W]])
        desc = EP._desc(blk, sel)
        nb, n = len(desc), ctx.bs[W] // 2
        carry = ctx.encode_carry_init(1)
        pcarry = ctx.encode_pcm_carry_init(1)
        kept = carry.copy(), pcarry.copy()
        mdct = np.random.default_rng(0).standard_normal((nb, ch, n)).astype(np.float32)
        s16 = np.ascontiguousarray(np.clip(np.rint(tl * 32768.0), -32768, 32767).astype(np.int16).transpose(0, 2, 1))
        def cqn():                                    # iwork and nonzero are in/out: the wrapper copies them
            iw, nz = vlib.np.zeros((nb, ch, n), np.int32), vlib.np.zeros((nb, ch), np.int32)
            ctx._chk(ctx.L.vb200_couple_quantize_normalize(ctx.h, W, 0, 7, nb, vlib._ptr(mdct), vlib._ptr(iw),
                                                           vlib._ptr(nz)))
        calls = {
            "couple_quantize_normalize": cqn,
            "encode_dsp":lambda: ctx.encode_dsp(W, blocks, desc, classes=True),
            "encode_dsp_managed": lambda: ctx.encode_dsp_managed(W, blocks, desc),
            "encode_packets": lambda: ctx.encode_packets(W, blocks, desc),
            "encode_packets_managed": lambda: ctx.encode_packets_managed(W, blocks, desc),
            "encode_streams": lambda: ctx.encode_streams(tl, pcm_len, eof),
            "encode_streams_s16": lambda: ctx.encode_streams(s16, pcm_len, eof, fmt=vlib.PCM_S16_INTERLEAVED),
            "encode_streams_managed": lambda: ctx.encode_streams_managed(tl, pcm_len, eof),
            "encode_streams_packets": lambda: ctx.encode_streams_packets(tl, pcm_len, eof),
            "encode_streams_packets_resume": lambda: ctx.encode_streams_packets_resume(tl, pcm_len, carry, eof),
            "encode_pcm_packets": lambda: ctx.encode_pcm_packets(_many_signal(ch)[None], [rate // 4], pcarry),
        }
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
        assert np.array_equal(carry, kept[0]) and np.array_equal(pcarry, kept[1]), "a carry changed"
        # the device forms
        dev = torch.device("cuda")
        d_mdct = torch.from_numpy(mdct).to(dev)
        d_iw = torch.full((nb, ch, n), 0x5A5A5A5A, dtype=torch.int32, device=dev)
        d_nz = torch.full((nb, ch), 0x5A5A5A5A, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        with pytest.raises(vlib.VB200Error, match="too many channels"):
            ctx.couple_quantize_normalize_dev(W, 0, 7, nb, d_mdct.data_ptr(), d_iw.data_ptr(), d_nz.data_ptr())
        t = {"pcm": torch.from_numpy(blocks).to(dev),
             "desc": torch.from_numpy(desc.view(np.uint8).reshape(nb, -1).copy()).to(dev),
             "posts": torch.full((nb, ch, abi.FLOOR1_STRIDE), 0x5A5A5A5A, dtype=torch.int32, device=dev),
             "nonzero": d_nz, "iwork": d_iw,
             "ampmax_out": torch.full((nb,), 7.0, device=dev)}
        io = abi.EncodeIO()
        for k, v in t.items():
            setattr(io, k, v.data_ptr())
        io.independent = 1
        with pytest.raises(vlib.VB200Error, match="too many channels"):
            ctx.encode_dsp_dev(W, nb, 1, io)
        torch.cuda.synchronize()
        for k in ("posts", "nonzero", "iwork"):
            assert (t[k] == 0x5A5A5A5A).all().item(), "encode_dsp_dev wrote %s" % k
        # still a working context: synthesis of random blocks equals the oracle's
        rng = np.random.default_rng(80)
        Wseq = rng.integers(0, 2, (2, 6)).astype(np.int32)
        coef_off, pcm_off, coef_len, pcm_stride = vlib.synthesis_layout(Wseq, ctx.bs, ch)
        coef = (rng.uniform(-1, 1, coef_len) * 0.05).astype(np.float32)
        o = pyoracle.Oracle(setup)
        assert_bits_equal(ctx.synthesis(Wseq, coef_off, coef, pcm_off, pcm_stride),
                          o.synthesis(Wseq, coef_off, coef, pcm_off, pcm_stride), "synthesis after the refusals")
    finally:
        d.close()


def test_255_channels_stream_decoder(cuda_ok, drivers):  # noqa: F811
    """255 channels, the most a Vorbis stream holds: decode_streams_packets gives the stock decoder's PCM in float
    and int16"""
    ch = 255
    DS._need()
    p = decode.encode(ch, MANY_RATE, MANY_Q, _many_signal(ch, seed=2))
    ctx = DS._ctx(drivers, p.buf, p.hdr)
    want = [ds.ref_decode(p.buf, p.hdr, p.audio, ch, cap=1 << 15)]
    assert want[0][0].shape[1] > MANY_RATE // 5
    npkt, info = DS._table([p.audio])
    for s16 in (False, True):
        DS._check(ctx.decode_streams_packets(npkt, info, p.buf, ctx.decode_streams_carry(1), s16=s16), want, ch, s16,
                  "255 channels s16=%s" % s16)
