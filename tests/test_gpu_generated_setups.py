"""The device decode paths on generated Vorbis setups (tests/vorbis_gen.py), bit for bit against the stock decoder.

On the "inside" corpus (block sizes 64 to 8192, 1 to 64 channels, up to 4 submaps, 32-bit codewords, books without
codewords, 0-partition and 65-post floors, 64 residue classes, cascades with gaps):
- the multi-stream driver takes the device path, and the staging of vb200_decode_entropy (residue as uint32, posts,
  presence) equals the reference's for the structured packets and for truncated, bit-flipped and empty ones;
- vb200_decode_packets_resume in float and int16 equals the stock decoder's PCM at full rate, and the stock half-rate
  decoder's at half rate (refused where blocksizes[0] == 64, as the reference refuses it);
- vb200_decode_streams_packets and vb200_decode_ranges equal the stock pcmout loop, with granulepos on every packet
  and on page-final packets only;
- the driver's device and forced-host paths give the stock PCM.
On the "outside" corpus: the driver refuses the setups whose modes or floors the device context cannot take, keeps
the host path where the entropy setup is refused and still decodes like the stock decoder; a context that refused an
entropy setup (VB200_EIMPL for residue type 0, VB200_EINVAL for a residue past the block) keeps decoding with the one
it had."""
import ctypes as C

import numpy as np
import pytest

import vorbis_gen as G
from oracle import decode, halfrate
from oracle import decode_packets as dp
from oracle import decode_streams as ds
from test_generated_setups_oracle import ALL, corpus
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
OV_EFAULT, OV_EIMPL = -129, -130


def _need():
    if not (decode.available() and dp.available() and ds.ref_available() and halfrate.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


@pytest.fixture(scope="module", params=G.INSIDE)
def case(request, cuda_ok):
    _need()
    d, pk, p = corpus(request.param)
    drv = dp.Driver(p)
    yield request.param, d, pk, p, drv
    drv.close()


def _table(audios):
    """every audio row of each stream -> (npkt, info) of vb200_decode_streams_packets / vb200_decode_ranges"""
    npkt = np.array([len(a) for a in audios], np.int32)
    info = np.zeros((len(audios), int(npkt.max())), abi.PACKET_INFO_DTYPE)
    for s, m in enumerate(audios):
        k = len(m)
        info["offset"][s, :k], info["bytes"][s, :k], info["granulepos"][s, :k] = m[:, 0], m[:, 1], m[:, 2]
        info["e_o_s"][s, :k], info["packetno"][s, :k] = m[:, 3], m[:, 4]
    return npkt, info


def _check_streams(got, want, s16, what):
    """decode_streams_packets' output against the stock pcmout loop (ds.ref_decode) of each stream"""
    for s, (pcm, rec, _) in enumerate(want):
        o = got["out"][s, :len(rec)]
        assert (o["status"] == rec[:, 0]).all(), "%s stream %d: status" % (what, s)
        assert (o["samples"] == rec[:, 2]).all(), "%s stream %d: samples" % (what, s)
        assert (o["granulepos"] == rec[:, 3]).all(), "%s stream %d: granulepos" % (what, s)
        g = got["pcm"][s]
        if s16:
            assert np.array_equal(g, ds.s16_of(pcm)), "%s stream %d: int16 PCM" % (what, s)
        else:
            assert g.shape == pcm.shape and np.array_equal(g.view(np.uint32), pcm.view(np.uint32)), \
                "%s stream %d: PCM" % (what, s)


def _staging(p, drv, pkts, what):
    W = dp.ref_headers(p, pkts)
    ref = dp.ref_staging(p, pkts, W, drv.bs, drv.channels)
    got = dp.dev_staging(drv.ctx, pkts, W, drv.bs, drv.channels)
    assert np.array_equal(ref[0].view(np.uint32), got[0].view(np.uint32)), what + ": residue"
    assert np.array_equal(ref[1], got[1]), what + ": posts"
    assert np.array_equal(ref[2], got[2]), what + ": present"
    return W, ref


def test_device_path_and_staging(case):
    name, d, pk, p, drv = case
    assert drv.on_device, name
    assert drv.bs == list(d["bs"]) and drv.channels == d["channels"]
    W, ref = _staging(p, drv, pk, name)
    assert (W >= 0).all() and ref[2].any()
    bad = G.damaged(pk, 2000 + ALL.index(name), G.header_bits(d))
    W, ref = _staging(p, drv, bad, name + " damaged")
    assert (W < 0).any() and (W >= 0).any()


def _resume(ctx, p, s16):
    """every audio packet of p in one vb200_decode_packets_resume call"""
    pkts = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.audio[:, :2]]
    W = dp.ref_headers(p, pkts)
    Wseq = W[None].astype(np.int32)
    co, po, clen, plen = lib.synthesis_layout(Wseq, ctx.bs, ctx.channels, halfrate=ctx.halfrate)
    out = ctx.decode_packets_resume(Wseq, co, max(clen, 1), p.audio[None, :, 0].copy(),
                                    p.audio[None, :, 1].astype(np.int32), p.buf, po, max(plen, 1),
                                    ctx.new_decode_carry(1), s16=s16)
    return out[0][:plen] if s16 else out[0][:, :plen]


def test_packets_resume_equals_stock(case):
    name, d, pk, _, drv = case
    ctx, ch = drv.ctx, d["channels"]
    _, _, p = corpus(name, granule=False)          # no trims: the stock PCM is every finished sample
    want = decode.stock_decode(p, channels=ch)
    got = _resume(ctx, p, False)
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), name + " float"
    assert np.array_equal(_resume(ctx, p, True), ds.s16_of(want)), name + " int16"
    if d["bs"][0] == 64:
        with pytest.raises(lib.VB200Error, match="-131"):
            ctx.synthesis_halfrate(True)
        return
    lens = p.meta[:, 1].copy()
    win = halfrate.ref_decode((p.buf, lens), list(d["bs"]), ch, 1 << 18, halfrate=True)
    want, _, _ = ds.ref_decode(p.buf, p.hdr, p.audio, ch, halfrate=True)
    ctx.synthesis_halfrate(True, [win["window0"], win["window1"]])
    try:
        got = _resume(ctx, p, False)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), name + " half rate"
        assert np.array_equal(_resume(ctx, p, True), ds.s16_of(want)), name + " half rate int16"
    finally:
        ctx.synthesis_halfrate(False)


def test_streams_and_ranges_equal_stock(case):
    name, d, pk, p, drv = case
    ctx, ch = drv.ctx, d["channels"]
    _, _, pf = corpus(name, page_final=True)
    audios = [p.audio, pf.audio]
    want = [ds.ref_decode(p.buf, p.hdr, a, ch) for a in audios]
    npkt, info = _table(audios)
    for s16 in (False, True):
        got = ctx.decode_streams_packets(npkt, info, p.buf, ctx.decode_streams_carry(2), s16=s16)
        _check_streams(got, want, s16, name + " s16=%s" % s16)
    rng = np.random.default_rng(3000 + ALL.index(name))
    stride = 3 * d["bs"][1]
    req = []
    for s, (pcm, _, _) in enumerate(want):
        n = pcm.shape[1]
        for _ in range(6):
            start = int(rng.integers(0, n + 1))
            req.append((start, s, int(rng.integers(0, stride + 1))))
    req.append((0, 0, stride))
    r = ctx.decode_ranges(npkt, info, p.buf, req, stride)
    for i, (start, s, length) in enumerate(req):
        w = want[s][0][:, start:start + length]
        assert r["got"][i] == w.shape[1], "%s range %d" % (name, i)
        g = r["pcm"][i][:, :w.shape[1]]
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), "%s range %d" % (name, i)
        assert not r["pcm"][i][:, w.shape[1]:].any()


@pytest.mark.parametrize("s16", [False, True])
def test_driver_paths_equal_stock(case, s16):
    name, d, pk, p, drv = case
    ch = d["channels"]
    want = decode.stock_decode(p, channels=ch, s16=s16)
    joined = decode.join([(p.buf, p.audio, p.meta[:3])] * 2)
    sched = np.random.default_rng(ALL.index(name)).integers(0, 5, (40, 2))
    for host in (False, True):
        got, st = dp.md_run(joined, sched, ch, s16=s16, host_entropy=host)
        assert st["entropy_on_device"] == (not host)
        for s in range(2):
            assert got[s].shape == want.shape
            assert np.array_equal(got[s].view(np.uint8), want.view(np.uint8)), "%s stream %d host=%s" % (name, s, host)


# ---- outside the limits --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(G.OUTSIDE))
def test_outside_refused_or_host_path(cuda_ok, name):
    _need()
    d, pk, p = corpus(name)
    ch = d["channels"]
    want = decode.stock_decode(p, channels=ch)
    assert want.shape[1] > 0
    if G.OUTSIDE[name] == "context":
        if name == "floor_wider_than_block":          # vb200_ctx_create refuses the floor; the driver cannot open
            from test_generated_setups_oracle import decode_setup
            with pytest.raises(lib.VB200Error, match="-131"):
                lib.Context(decode_setup(d))
            assert dp.open_error(p) == OV_EFAULT
        else:                                         # the driver takes two modes with block flags 0 and 1 only
            assert dp.open_error(p) == OV_EIMPL
        return
    drv = dp.Driver(p)
    try:
        assert not drv.on_device
    finally:
        drv.close()
    got, st = dp.md_run(decode.join([(p.buf, p.audio, p.meta[:3])]), np.full((8, 1), 3), ch)
    assert not st["entropy_on_device"]
    assert np.array_equal(got[0].view(np.uint32), want.view(np.uint32)), name


def _entropy_setup(d):
    """the abi.EntropySetup of a description as vb200md derives it from the decoder, with all-zero value rows:
    (keep-alive, struct)"""
    keep, books = [], (abi.Codebook * len(d["books"]))()
    for i, b in enumerate(d["books"]):
        cw = G.Coder(b)
        used = cw.used
        length = np.array([cw.words[e][1] for e in used], np.uint8)
        bits = np.array([cw.words[e][0] for e in used], np.uint32)
        entry = np.array(used, np.int32)
        value = np.zeros(max(len(used) * b["dim"], 1), np.float32)      # value rows are not restated here
        keep += [length, bits, entry, value]
        books[i].dim, books[i].used = b["dim"], len(used)
        books[i].length, books[i].bits, books[i].entry = length.ctypes.data, bits.ctypes.data, entry.ctypes.data
        books[i].value = value.ctypes.data if b["maptype"] else None
    es = abi.EntropySetup()
    es.nbooks, es.books, es.modebits = len(d["books"]), C.cast(books, C.POINTER(abi.Codebook)), 1
    for w, (_, mi) in enumerate(d["modes"]):
        m = d["mappings"][mi]
        for s in range(m["submaps"]):
            f, r = d["floors"][m["floor"][s]], d["residues"][m["residue"][s]]
            F = es.floor[w][s]
            F.type, F.partitions = 1, len(f["pclass"])
            for k, c in enumerate(f["pclass"]):
                F.partitionclass[k] = c
            for c in f["cdim"]:
                F.class_dim[c], F.class_subs[c], F.class_book[c] = f["cdim"][c], f["csubs"][c], max(f["cbook"][c], 0)
                for k, sb in enumerate(f["subbook"][c]):
                    F.class_subbook[c][k] = sb
            R = es.residue[w][s]
            R.type, R.begin, R.end, R.grouping = r["type"], r["begin"], r["end"], r["grouping"]
            R.partitions, R.groupbook = len(r["cascade"]), r["groupbook"]
            R.partvals = len(r["cascade"]) ** d["books"][r["groupbook"]]["dim"]
            for c in range(64):
                for k in range(8):
                    R.stagebook[c][k] = r["books"][c][k] if c < len(r["cascade"]) else -1
    return (keep, books), es


def test_refused_entropy_setup_keeps_the_registered_one(cuda_ok):
    """an inside driver's context refuses a residue of type 0 (VB200_EIMPL) and one past the block (VB200_EINVAL) and
    keeps decoding with the setup it had; the description's own codewords, floors and residues (zero value rows) are
    taken and give the reference's posts and presence"""
    _need()
    name = "s256_512_3ch"
    d, pk, p = corpus(name)
    drv = dp.Driver(p)
    try:
        assert drv.on_device
        for mutate, code in (("type0", "-130"), ("past", "-131")):
            bad = G.setup(name)
            r = bad["residues"][bad["mappings"][bad["modes"][0][1]]["residue"][0]]
            if mutate == "type0":
                r["type"] = 0
            else:
                r["begin"], r["end"] = 10 ** 6, 10 ** 6 + 64
            keep, es = _entropy_setup(bad)
            with pytest.raises(lib.VB200Error, match=code):
                drv.ctx.decode_entropy_setup(es)
            _staging(p, drv, pk, name + " after a refused " + mutate)
        keep, es = _entropy_setup(d)
        drv.ctx.decode_entropy_setup(es)
        W = dp.ref_headers(p, pk)
        ref = dp.ref_staging(p, pk, W, drv.bs, drv.channels)
        got = dp.dev_staging(drv.ctx, pk, W, drv.bs, drv.channels)
        assert np.array_equal(ref[1], got[1]) and np.array_equal(ref[2], got[2])
    finally:
        drv.close()
