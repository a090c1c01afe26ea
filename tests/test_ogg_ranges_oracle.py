"""oracle/ogg_ranges.py, the restatement of vb200_ogg_ranges' seek, without a GPU:
- on clean rows (seeded pages of 1-255 segments from oracle.ogg.write; granulepos from 0, far above zero, and with a
  beginning trim; e_o_s trims; both block sizes) it keeps the blocks, windows and positions that
  oracle.decode_ranges.plan keeps on oracle.ogg.demux's packet table of the same row, at full and half rate, for
  starts at 0, at page granulepos +- blocksizes[1]/2, near and past the end, and lengths 0..out_stride; rows with
  another serial's pages interleaved and the links of a chained file included;
- on rows with a removed page or a CRC-damaged page, a request that seeks past the damage keeps the blocks and
  positions of the clean row: positions follow the granulepos, where the packet-table count drifts by the lost
  packets."""
import numpy as np
import pytest

from oracle import decode_ranges as dr
from oracle import ogg
from oracle import ogg_links
from oracle import ogg_ranges as orr

BS = (256, 2048)
MODEBITS = 1


def _audio_packet(rng, W):
    """a packet whose header bits read as block flag W (type 0, mode W, and for a long block lW and nW)"""
    n = int(rng.integers(2, 700))
    body = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    body[0] = (body[0] & ~0x3) | (W << 1)            # bit 0: audio; bit 1: the mode
    return bytes(body)


def _stream(rng, n, g0=0, trim=0, eos_trim=100):
    """three header packets and n audio packets with the granulepos a stock encoder gives them: the first audio
    packet's is g0, then the running count, all less trim (a beginning trim); the last is cut by eos_trim"""
    Ws = [int(w) for w in rng.integers(0, 2, n)]
    pk = [b"\x01vorbis" + bytes(23), b"\x03vorbis" + bytes(10), b"\x05vorbis" + bytes(40)]
    pk += [_audio_packet(rng, W) for W in Ws]
    g, gr = g0, [0, 0, 0]
    for k, W in enumerate(Ws):
        if k:
            g += BS[Ws[k - 1]] // 4 + BS[W] // 4
        gr.append(g - trim)
    gr[-1] -= eos_trim
    return pk, gr


def _row(rng, pk, gr, serial=7, **kw):
    return b"".join(ogg.write(pk, gr, serial, rng, **kw))


def _table(buf):
    """oracle.ogg.demux's packet table of a row, as (packet bytes, audio rows) for oracle.decode_ranges"""
    r = ogg.demux(buf, 1 << 20)
    assert r["status"] == 0
    data = b"".join(r["pkt_data"])
    rows, off = [], 0
    for (o, n, g, e, pno), d in zip(r["packets"], r["pkt_data"]):
        rows.append((off, n, g, e, pno))
        off += n
    return np.frombuffer(data, np.uint8), np.array(rows, np.int64).reshape(-1, 5), r


def _starts(buf, hd, length, rng, half):
    """starts at 0, at every few pages' granulepos +- blocksizes[1]/2, near and past the end"""
    hs = 1 if half else 0
    gps = sorted(set(_page_granules(buf, hd["serial"])))
    out = [0, 1]
    for g in gps[::3]:
        t = (g - hd["G0"]) >> hs
        out += [max(t - (BS[1] // 2 >> hs), 0), t, t + (BS[1] // 2 >> hs)]
    out += [max(length - k, 0) for k in (1, 5, 300, 3000)] + [length, length + 1, length + 10 ** 6]
    return out + [int(x) for x in rng.integers(0, max(length, 1), 6)]


def _page_granules(buf, serial):
    out = []
    for p, _ in ogg_links.pages_of(buf):
        ver, flags, g, ser, _, _ = orr._page(buf, p)
        if ser == serial and g != -1 and g != 0:
            out.append(g)
    return out


def _same(got, kept, want_got, want_kept, data, what):
    assert got == want_got, "%s: got %d, plan %d" % (what, got, want_got)
    assert len(kept) == len(want_kept), what
    for j, (a, b) in enumerate(zip(kept, want_kept)):
        assert a["W"] == b["W"] and a["data"] == bytes(data[b["offset"]:b["offset"] + b["bytes"]]), (what, j)
        if j:                                        # "at" means nothing for a block that keeps no sample
            assert a["keep"] == b["keep"] and (a["keep"] == (0, 0) or a["at"] == b["at"]), (what, j, a, b)


def _check_row(buf, rng, what, out_stride=3000):
    data, audio, _ = _table(buf)
    for half in (False, True):
        length, _, blks = dr.blocks(data, audio, BS, MODEBITS, halfrate=half)
        hd = orr.head(buf, BS, MODEBITS, half)
        seeks = 0
        for start in _starts(buf, hd, length, rng, half):
            for n in (0, 1, int(rng.integers(1, out_stride + 1)), out_stride):
                want = dr.plan(blks, start, n)
                r = orr.request(buf, BS, MODEBITS, start, n, half, hd=hd)
                seeks += r["mode"] == "seek"
                _same(r["got"], r["kept"], want[0], want[1], data, "%s half=%s start %d length %d" % (what, half, start, n))
        assert seeks > 0, what


@pytest.mark.parametrize("seed", range(4))
def test_clean_rows_equal_packet_table_plan(seed):
    rng = np.random.default_rng(seed)
    segs = [dict(max_segs=255), dict(max_segs=4), dict(min_segs=1, max_segs=1 + seed * 60)][seed % 3]
    for g0, trim in ((0, 0), (5 * 10 ** 9 + 64, 0), (0, 300)):
        pk, gr = _stream(rng, 220, g0=g0, trim=trim)
        _check_row(_row(rng, pk, gr, **segs), rng, "seed %d g0 %d trim %d" % (seed, g0, trim))


def test_foreign_serial_and_chained_links():
    rng = np.random.default_rng(11)
    pk, gr = _stream(rng, 160)
    mine = ogg.write(pk, gr, 5, rng, max_segs=6)
    pk2, gr2 = _stream(rng, 120)
    other = ogg.write(pk2, gr2, 6, rng, max_segs=6)
    mixed = []
    for i, pg in enumerate(mine):
        mixed.append(pg)
        if i < len(other):
            mixed.append(other[i])
    _check_row(b"".join(mixed), rng, "interleaved")
    chained = b"".join(mine) + b"".join(ogg.write(pk2, gr2, 5, rng, max_segs=9))
    offs = ogg_links.links(chained)
    assert len(offs) == 3
    for k in range(2):
        _check_row(chained[offs[k]:offs[k + 1]], rng, "link %d" % k)


def test_row_errors():
    rng = np.random.default_rng(3)
    pk, gr = _stream(rng, 20)
    pages = ogg.write(pk, gr, 9, rng, max_segs=255)
    assert orr.request(b"".join(pages[1:]), BS, MODEBITS, 0, 10)["got"] == orr.ENOTVORBIS
    assert orr.request(pages[0], BS, MODEBITS, 0, 10)["got"] == orr.EBADHEADER
    assert orr.request(b"", BS, MODEBITS, 0, 10)["got"] == orr.ENOTVORBIS


@pytest.mark.parametrize("damage", ["page removed", "crc flipped"])
def test_positions_follow_granulepos_past_damage(damage):
    rng = np.random.default_rng(21)
    pk, gr = _stream(rng, 400)
    pages = ogg.write(pk, gr, 3, rng, max_segs=8)
    k = len(pages) // 3
    if damage == "page removed":
        bad = pages[:k] + pages[k + 1:]
    else:
        flip = bytearray(pages[k])
        flip[30] ^= 0x40
        bad = pages[:k] + [bytes(flip)] + pages[k + 1:]
    clean, bad = b"".join(pages), b"".join(bad)
    data, audio, r = _table(bad)
    assert ogg.demux(bad, 1 << 20)["holes"] == 1
    length, _, blks = dr.blocks(data, audio, BS, MODEBITS)
    hc, hb = orr.head(clean, BS, MODEBITS), orr.head(bad, BS, MODEBITS)
    assert hc["G0"] == hb["G0"]
    cut = sum(len(p) for p in pages[:k + 2])
    drift = 0
    for start in range(0, gr[-1], 997):
        a, b = orr.request(clean, BS, MODEBITS, start, 1500), orr.request(bad, BS, MODEBITS, start, 1500)
        if b["mode"] != "seek" or b["P"] < cut:
            continue
        assert a["got"] == b["got"] and [x.get("keep") for x in a["kept"]] == [x.get("keep") for x in b["kept"]]
        assert [x.get("at") for x in a["kept"]] == [x.get("at") for x in b["kept"]]
        assert [x["data"] for x in a["kept"]] == [x["data"] for x in b["kept"]], start
        want = dr.plan(blks, start, 1500)
        drift += [x.get("at") for x in want[1]] != [x.get("at") for x in a["kept"]] or want[0] != a["got"]
    assert drift > 0, "the packet-table count does not drift after the lost packets"
