"""Every device path on the setups vorbisenc picks above q = 0.5, and at the high nominal rates of managed encodes that
pick the same templates.  Bit-exact.

There the setups have a structure the q <= 0.5 setups never show the device:
- stereo 44.1/48 kHz q >= 0.6, 96 kHz and 22.05 kHz q 0.9: the _residue_44_high books, whose classes reach the
  thresholds 71 and 157 and whose top classes have two and three cascade stages; the residue covers the whole
  interleaved vector (end = 2 * n), so the last partition ends on the last coefficient of channel 1;
- mono q >= 0.8: the _residue_44_hi_un books, type-1 residue up to end = n;
- 5.1 q >= 0.5: no coupling steps on six channels, two submaps, and the _residue_44p_hi books over the five
  interleaved channels (end 4290 or 5100 of 5120, partitions of 30);
- 96 kHz (256/2048 with 586/776 total octave lines) and coupled 22.05 kHz stereo (512/1024).

- The setup-family suite of tests/setup_families.py on the rows of FAMILY: the stages against the oracle, which
  tests/test_oracle_vs_ref.py pins to the reference at these setups, fed the blocks the reference encoder cut from its
  chain stream (tests/golden/ref).
- Packets and PCM against the stock encoder and decoder (needs oracle/_ref), on the usual probe streams and on loud
  full-band content (white noise at +-0.9, a tone 3 bins below Nyquist, full-scale clicks, an int16 full-scale square
  wave, and for stereo L = R and L = -R).  On that content the reference's own residue reaches the three top classes of
  each setup's books and a non-zero last partition before `end`, which the tests assert, so that a device that
  mishandled the top classes or the last partition could not pass."""
import numpy as np
import pytest

import refgold as G
import test_gpu_decode_packets as DP
import test_gpu_decode_streams as DS
import test_gpu_encode_packets as EP
import test_gpu_stream_packets as SP
import test_oracle_vs_ref as T
from oracle import bitrate as B
from oracle import decode, pyoracle, pyref
from oracle import decode_packets as dp
from oracle import decode_streams as ds
from setup_families import *  # noqa: F401,F403  (the suite's tests and fixtures, among them drivers)
from setup_families import (Family, test_entropy_coder_fuzz, test_stock_decoder_streams_and_ranges,  # noqa: F401
                            test_stock_encoder_streams_in_pieces_and_raw_pcm)

pytestmark = pytest.mark.gpu

HIGH = T.HIGH
HIGH3 = [(2, 44100, 1.0), (6, 48000, 0.9), (2, 22050, 0.9)]
# per setup: block sizes, coupling steps, submaps, and (type, end, grouping) of each submap's residue for W = 0 and 1
FEATURES = {
    (2, 44100, 0.6): ([256, 2048], 1, 1, [[(2, 256, 16)], [(2, 2048, 32)]]),
    (2, 44100, 1.0): ([256, 2048], 1, 1, [[(2, 256, 16)], [(2, 2048, 32)]]),
    (1, 44100, 0.9): ([256, 2048], 0, 1, [[(1, 128, 16)], [(1, 1024, 32)]]),
    (6, 48000, 0.5): ([256, 2048], 0, 2, [[(2, 540, 15), (1, 12, 6)], [(2, 4290, 30), (1, 12, 6)]]),
    (6, 48000, 0.9): ([256, 2048], 0, 2, [[(2, 630, 15), (1, 12, 6)], [(2, 5100, 30), (1, 12, 6)]]),
    (2, 96000, 0.7): ([256, 2048], 1, 1, [[(2, 256, 16)], [(2, 2048, 32)]]),
    (2, 22050, 0.9): ([512, 1024], 1, 1, [[(2, 512, 32)], [(2, 1024, 32)]]),
}


def _residue(setup, W, sm):
    return setup.c.residue[W][sm]


def check_features(setup, args):
    """the setup has the structure this family is about, so that a vorbisenc change cannot turn the tests into a
    repeat of the q <= 0.5 ones"""
    bs, steps, submaps, res = FEATURES[args]
    assert [setup.blocksize(0), setup.blocksize(1)] == bs
    assert list(setup.c.coupling_steps) == [steps, steps] and list(setup.c.submaps) == [submaps, submaps]
    for W in (0, 1):
        got = [(r.type, r.end, r.grouping) for r in (_residue(setup, W, sm) for sm in range(submaps))]
        assert got == res[W], "W=%d residues %s" % (W, got)
        r = _residue(setup, W, 0)
        assert r.begin == 0
        metric = list(r.classmetric1)[:r.partitions]
        if args[0] == 6:                              # _residue_44p_hi
            assert r.partitions == 8 and metric[4:7] == [7, 17, 31]
        else:                                         # _residue_44_high / _residue_44_hi_un
            assert r.partitions == 10 and metric[6:9] == [32, 71, 157]
    if args[0] == 2:
        assert res[1][0][1] == setup.blocksize(1)      # type 2 over the whole interleaved vector
    if args[0] == 1:
        assert res[1][0][1] == setup.blocksize(1) // 2


# name, channels, rate, max, nominal and min bitrate, and the small-reservoir settings; vorbisenc picks the q > 0.5
# templates for these nominal rates: full-band residue in stereo, no coupling steps at 5.1
MANAGED = [("abr256", 2, 44100, -1, 256000, -1, None),
           ("cbr320", 2, 44100, 320000, 320000, 320000, None),
           ("cbr320_small", 2, 44100, 320000, 320000, 320000, (4000, 0.3, 0.5)),
           ("abr512_51", 6, 48000, -1, 512000, -1, None)]
FAMILY = Family(
    name="high", setups=HIGH, capture={}, check=check_features, blocksizes=lambda args: FEATURES[args][0],
    nvec=[[133]], fmts=[["f32", "s16"]], envelope=[HIGH],
    rows={"test_stock_encoder_packets": HIGH, "test_stock_encoder_streams_in_pieces_and_raw_pcm": HIGH3,
          "test_stock_managed_encoder": MANAGED, "test_stock_decoder": HIGH,
          "test_stock_decoder_streams_and_ranges": HIGH, "test_stock_halfrate_decoder": HIGH3,
          "test_function_level_dropin": [(2, 44100, 1.0), (1, 44100, 0.9), (6, 48000, 0.9)]},
    fuzz=[(2, 44100, 1.0), (6, 48000, 0.9)])


# ---- loud full-band content -----------------------------------------------------------------------------------------
def loud_signal(ch, rate, seed=0):
    """a quarter second each of white noise at +-0.9, a tone 3 long-block bins below Nyquist, full-scale clicks, an
    int16 full-scale square wave, and for stereo L = R and L = -R noise"""
    rng = np.random.default_rng(seed)
    seg = rate // 4
    t = np.arange(seg)
    f = rate / 2 - 3 * rate / 2048.0
    clicks = np.zeros((ch, seg))
    clicks[:, ::997], clicks[:, 498::997] = 1.0, -1.0
    square = np.where((t // max(1, rate // 2000)) % 2 == 0, 32767, -32768) / 32768.0
    parts = [rng.uniform(-0.9, 0.9, (ch, seg)), np.tile(0.9 * np.sin(2 * np.pi * f * t / rate + 0.3), (ch, 1)),
             clicks, np.tile(square, (ch, 1))]
    if ch == 2:
        n = rng.uniform(-0.9, 0.9, seg)
        parts += [np.stack([n, n]), np.stack([n, -n])]
    return np.concatenate(parts, axis=1).astype(np.float32)


def _coverage(setup, W, classes, seen):
    """the classes of the main submap's residue: counts per class and how often its last partition is not class 0"""
    r = _residue(setup, W, 0)
    p = (r.end - r.begin) // r.grouping
    rows = [c for c in range(setup.channels) if setup.floor_of(W, c) == 0]
    c0 = classes[:, rows, :p]
    seen["classes"] += np.bincount(c0.ravel(), minlength=r.partitions)[:r.partitions]
    seen["last"] += int((c0[..., p - 1] > 0).sum())


@pytest.mark.parametrize("args", HIGH, ids=lambda a: G.case_id(*a))
def test_loud_content_vs_stock_encoder(cuda_ok, args):
    """the stock encoder's blocks of the loud signal: the device chain gives its residue and nonzero flags, the
    reference's partition classes (which reach the three top classes and the last partition before `end`), and
    through encode_dsp + encode_entropy and encode_packets its audio packets; whole streams give its packets"""
    ch, rate, q = args
    d = EP._driver(ch, rate, q)
    ctx = d.ctx
    try:
        setup = G.load_setup(*args)                   # the driver's setup: tests/test_oracle_vs_ref.py pins it
        check_features(setup, args)
        pcm = loud_signal(ch, rate)
        ref = pyref.Ref(ch, rate, q)
        cap = ref.encode_capture(pcm, fields=("pcm", "iwork_out"))
        pk = ref.packets()
        want = pk[len(pk) - cap["nblocks"]:]
        o = pyoracle.Oracle(setup)
        seen = {"classes": np.zeros(_residue(setup, 0, 0).partitions, np.int64), "last": 0}
        for W in (0, 1):
            sel = cap["W"] == W
            n, stride = ctx.bs[W] // 2, o.residue_partvals(W)
            blocks = np.ascontiguousarray(cap["pcm"][sel][:, :, :ctx.bs[W]])
            desc = EP._desc(cap, sel)
            wcls = ref.residue_classify(W, cap["iwork_out"][sel][:, :, :n], cap["nonzero_out"][sel], stride)
            _coverage(setup, W, wcls, seen)
            got = ctx.encode_dsp(W, blocks, desc, classes=True)
            assert np.array_equal(got["iwork"], cap["iwork_out"][sel][:, :, :n]), "W=%d residue" % W
            assert np.array_equal(got["nonzero"], cap["nonzero_out"][sel]), "W=%d nonzero" % W
            assert np.array_equal(got["classes"], wcls), "W=%d classes" % W
            wp = [p for p, s in zip(want, sel) if s]
            ent = ctx.encode_entropy(W, desc, got["posts"], got["nonzero"], got["iwork"])
            assert ent["packets"] == wp, "W=%d packets (encode_entropy)" % W
            assert ctx.encode_packets(W, blocks, desc)["packets"] == wp, "W=%d packets (encode_packets)" % W
            assert max(len(p) for p in wp) <= ctx.packet_bound(W)
        top = len(seen["classes"]) - 1
        assert (seen["classes"][top - 2:] > 0).all(), "top classes not reached: %s" % seen["classes"]
        assert seen["last"] > 0, "the last partition is silent in every block"
        sig = [pcm, np.clip(np.rint(pcm * 32768.0), -32768, 32767).astype(np.float32) / np.float32(32768.0)]
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p) for p in sig]
        tl, pcm_len, eof = SP._timelines(caps, ch)
        SP._compare(ctx.encode_streams_packets(tl, pcm_len, eof), caps, "loud q=%g" % q)
    finally:
        d.close()


@pytest.mark.parametrize("args", HIGH, ids=lambda a: G.case_id(*a))
def test_loud_content_vs_stock_decoder(cuda_ok, drivers, args):  # noqa: F811
    """the stock encoder's packets of the loud signal: the device's entropy decode stages the reference's residue,
    posts and floor flags, and the whole-stream decode gives the stock decoder's PCM in float and int16"""
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ch, rate, q = args
    p = decode.encode(ch, rate, q, loud_signal(ch, rate, seed=1))
    drv = dp.Driver(p)
    try:
        assert drv.on_device
        DP._check(p, drv, DP._pkts(p), "loud")
    finally:
        drv.close()
    ctx = DS._ctx(drivers, p.buf, p.hdr)
    audios = [p.audio]
    want = DS._stock(p.buf, p.hdr, audios, ch)
    npkt, info = DS._table(audios)
    for s16 in (False, True):
        got = ctx.decode_streams_packets(npkt, info, p.buf, ctx.decode_streams_carry(1), s16=s16)
        DS._check(got, want, ch, s16, "loud s16=%s" % s16)
