"""The Ogg demux oracle (oracle/ogg.py) and the host-only pieces of Ogg Vorbis file input, without a GPU:
- a seeded RFC 3533 page writer gives back its packets through oracle.ogg.demux, byte for byte, under varied pagings:
  headers alone on the BOS page, packets spanning one to three pages and more, lengths that are multiples of 255,
  zero-length packets, pages where no packet ends (granulepos -1) and 255-segment pages; granulepos lands on the last
  packet that ends on each page, e_o_s on the last packet, packetno counts from 3;
- the rules for damaged files as the header states them: a CRC-flipped page, a removed page, garbage between pages, a
  truncated last page, interleaved pages of a foreign serial, a second chained link, a file with no Vorbis stream and
  max_packets too small;
- four small files worked out by hand from the rules, with their packet tables written out literally (not produced by
  the oracle): granulepos on the last packet ending on a page when a page ends mid-packet, a hole's packetno and the
  skipped leading fragment of the continued page after it, zero-length and 255-byte packets, a page on which no
  packet ends;
- vb200_vorbis_window equals the reference's tabulated windows bit for bit for n = 64 .. 8192;
- the vb200_ogg_stream layout."""
import ctypes as C

import numpy as np
import pytest

from oracle import decode
from oracle import ogg
from vorbis_b200 import abi, lib


def _packets(rng, n):
    """three header-like packets (the first a Vorbis identification magic) and n audio packets of varied lengths"""
    hdr = [b"\x01vorbis" + bytes(rng.integers(0, 256, 23, dtype=np.uint8)),
           b"\x03vorbis" + bytes(rng.integers(0, 256, 300, dtype=np.uint8)),
           b"\x05vorbis" + bytes(rng.integers(0, 256, 1000, dtype=np.uint8))]
    sizes = [0, 1, 254, 255, 256, 510, 765, 1000, 3000, 0, 0, 600]
    audio = []
    for k in range(n):
        m = sizes[k] if k < len(sizes) else int(rng.integers(0, 1500))
        audio.append(bytes(rng.integers(0, 256, m, dtype=np.uint8)))
    return hdr + audio


PAGINGS = [dict(max_segs=255), dict(max_segs=1), dict(max_segs=3), dict(max_segs=17),
           dict(max_segs=255, headers_alone=False), dict(max_segs=5, headers_alone=False)]


def _check_roundtrip(r, pk, granules, pages):
    assert r["status"] == 0 and r["holes"] == 0 and r["dropped"] == 0 and r["foreign"] == 0
    assert r["pages"] == len(pages) and r["chained"] == 0
    assert r["hdr_data"] == pk[:3]
    assert r["pkt_data"] == pk[3:]
    t = ogg.packet_table(r)
    assert (t[:, 4] == np.arange(3, len(pk))).all(), "packetno"
    assert (t[:, 3] == (np.arange(3, len(pk)) == len(pk) - 1)).all(), "e_o_s"
    gp = t[:, 2]
    assert gp[-1] == granules[-1]
    assert ((gp == -1) | (gp == np.array(granules[3:]))).all(), "granulepos from another packet"
    # one granulepos per page that ends an audio packet, -1 on the pages that end none
    page_gp = [int(np.frombuffer(p[6:14], "<i8")[0]) for p in pages]
    ends_audio = sum(1 for g in page_gp if g >= 1000)
    assert (gp != -1).sum() == ends_audio
    return page_gp


@pytest.mark.parametrize("paging", range(len(PAGINGS)))
def test_writer_roundtrip(paging):
    rng = np.random.default_rng(100 + paging)
    pk = _packets(rng, 40)
    granules = [0, 0, 0] + [1000 + 7 * k for k in range(len(pk) - 3)]
    pages = ogg.write(pk, granules, 0x1234 + paging, rng, **PAGINGS[paging])
    r = ogg.demux(b"".join(pages), 1000)
    page_gp = _check_roundtrip(r, pk, granules, pages)
    if PAGINGS[paging].get("headers_alone", True):
        assert pages[0][26] == 1 and pages[0][5] & 2, "identification header alone on the BOS page"
    if PAGINGS[paging]["max_segs"] <= 3:
        assert -1 in page_gp, "a page where no packet ends"


def test_full_pages_and_long_packets():
    """255-segment pages, and packets spanning three pages and more"""
    rng = np.random.default_rng(7)
    pk = _packets(rng, 5)
    pk[4] = bytes(rng.integers(0, 256, 255 * 800, dtype=np.uint8))       # 801 segments: on four pages
    pk.append(bytes(255 * 3))
    granules = [0, 0, 0] + [1000 + k for k in range(len(pk) - 3)]
    pages = ogg.write(pk, granules, 99, rng, min_segs=255, headers_alone=False)
    assert pages[0][26] == 255 and len(pages) >= 4
    _check_roundtrip(ogg.demux(b"".join(pages), 100), pk, granules, pages)


def _file(seed=5, n=30, **kw):
    rng = np.random.default_rng(seed)
    pk = _packets(rng, n)
    granules = [0, 0, 0] + [1000 + 7 * k for k in range(n)]
    return pk, ogg.write(pk, granules, 77, rng, max_segs=kw.pop("max_segs", 4), **kw)


def test_damage_rules():
    pk, pages = _file()
    clean = ogg.demux(b"".join(pages), 1000)
    # a CRC-flipped page is a failed capture, then a sequence hole
    bad = list(pages)
    k = len(pages) // 2
    b = bytearray(bad[k])
    b[-1] ^= 0x40
    bad[k] = bytes(b)
    r = ogg.demux(b"".join(bad), 1000)
    assert r["dropped"] >= 1 and r["holes"] == 1 and r["pages"] == len(pages) - 1 and r["status"] == 0
    assert len(r["packets"]) < len(clean["packets"])
    assert r["pkt_data"][0] == clean["pkt_data"][0]
    # a removed page: one hole, packetno skips one
    r = ogg.demux(b"".join(pages[:k] + pages[k + 1:]), 1000)
    assert r["holes"] == 1 and r["dropped"] == 0
    t = ogg.packet_table(r)
    assert (np.diff(t[:, 4]) >= 1).all() and (np.diff(t[:, 4]) == 2).sum() == 1
    # garbage between pages: dropped captures, nothing else changes
    g = pages[:k] + [b"xxOggSOOgarbage" + bytes(40)] + pages[k:]
    r = ogg.demux(b"".join(g), 1000)
    assert r["dropped"] >= 2 and r["holes"] == 0 and r["pkt_data"] == clean["pkt_data"]
    # a truncated last page is not taken; its packet is lost
    r = ogg.demux(b"".join(pages)[:-3], 1000)
    assert r["pages"] == len(pages) - 1 and not any(x[3] for x in r["packets"])
    # interleaved pages of a foreign serial are skipped and counted
    foreign = ogg.write([b"\x01other" + bytes(40)] * 6, [0] * 6, 5, np.random.default_rng(1), max_segs=1,
                        headers_alone=False)
    mixed = []
    for i, p in enumerate(pages):
        mixed.append(p)
        if i < len(foreign):
            mixed.append(foreign[i])
    r = ogg.demux(b"".join(mixed), 1000)
    assert r["foreign"] == len(foreign) and r["pkt_data"] == clean["pkt_data"]
    # a second chained link: flagged, not read
    r = ogg.demux(b"".join(pages + _file(seed=6)[1]), 1000)
    assert r["chained"] == 1 and r["pkt_data"] == clean["pkt_data"]
    # no Vorbis stream
    r = ogg.demux(b"".join(foreign), 1000)
    assert r["status"] == ogg.ENOTVORBIS and r["foreign"] == len(foreign)
    # max_packets too small
    r = ogg.demux(b"".join(pages), 5)
    assert r["status"] == ogg.EINVAL and r["pkt_data"] == clean["pkt_data"][:5]
    # a hole before the third packet
    r = ogg.demux(b"".join(pages[:1] + pages[2:]), 1000)
    assert r["status"] == ogg.EBADHEADER and r["packets"] == []


def test_vorbis_window_equals_reference_tables():
    if not decode.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    for k in range(8):
        n = 64 << k
        got = lib.vorbis_window(n)
        want = decode.ref_window(n)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "n = %d" % n
    L = lib.load()
    assert L.vb200_vorbis_window(100, None) == -131 and L.vb200_vorbis_window(16384, None) == -131


def test_ogg_stream_layout():
    assert abi.OGG_STREAM_DTYPE.itemsize == 72
    f = abi.OGG_STREAM_DTYPE.fields
    assert f["chained"][1] == 24 and f["hdr_offset"][1] == 32 and f["hdr_bytes"][1] == 56
    L = lib.load()
    assert L.vb200_ogg_demux(1, None, None, 0, None, None, None, None) == -131     # max_packets < 1
    off = np.array([5, 3], np.int64)
    st = np.zeros(1, abi.OGG_STREAM_DTYPE)
    info = np.zeros(1, abi.PACKET_INFO_DTYPE)
    n = np.zeros(1, np.int32)
    rc = L.vb200_ogg_demux(1, None, off.ctypes.data, 1, info.ctypes.data, n.ctypes.data, None, st.ctypes.data)
    assert rc == -131 and b"decreases" in L.vb200_last_error()
    assert C.sizeof(C.c_int64) * 3 == f["hdr_offset"][0].itemsize


# ---- files small enough to work out by hand ------------------------------------------------------------------------
# Headers: 30, 10 and 10 bytes, so the first audio packet starts at offset 50 of the file's own byte range.
H = [b"\x01vorbis" + bytes(range(23)), b"\x03vorbis" + b"abc", b"\x05vorbis" + b"xyz"]


def _pre():
    return [ogg.page(2, 0, 7, 0, [30], H[0]), ogg.page(0, 0, 7, 1, [10, 10], H[1] + H[2])]


def _body(n, seed):
    return bytes((seed + 3 * i) & 255 for i in range(n))


B = _body(300, 1)
# name -> (pages, expected (status, pages, holes), expected rows (offset, bytes, granulepos, e_o_s, packetno))
HAND = {
    # A ends on page 2, B (300 bytes) starts there and ends on page 3 with C: the page granulepos goes to the last packet
    # ending on the page, so A gets 100, B -1, C 200; D alone on the EOS page gets 300 and e_o_s
    "granulepos mid-packet": (
        _pre() + [ogg.page(0, 100, 7, 2, [5, 255], _body(5, 0) + B[:255]),
                  ogg.page(1, 200, 7, 3, [45, 7], B[255:] + _body(7, 2)),
                  ogg.page(4, 300, 7, 4, [3], _body(3, 3))],
        (0, 5, 0),
        [(50, 5, 100, 0, 3), (55, 300, -1, 0, 4), (355, 7, 200, 0, 5), (362, 3, 300, 1, 6)]),
    # page 3 is missing: B's first 255 bytes are dropped, the hole takes packetno 4, and page 4 is continued with nothing
    # pending, so its 10-byte leading fragment is skipped; E lands where B began
    "hole then continued page": (
        _pre() + [ogg.page(0, 100, 7, 2, [5, 255], _body(5, 0) + B[:255]),
                  ogg.page(5, 400, 7, 4, [10, 20], _body(10, 4) + _body(20, 5))],
        (0, 4, 1),
        [(50, 5, 100, 0, 3), (55, 20, 400, 1, 5)]),
    # a zero-length packet, then one of exactly 255 bytes (lacing 255, 0), on the EOS page
    "empty and 255-byte packets": (
        _pre() + [ogg.page(4, 50, 7, 2, [0, 255, 0], _body(255, 6))],
        (0, 3, 0),
        [(50, 0, -1, 0, 3), (50, 255, 50, 1, 4)]),
    # a page on which no packet ends carries granulepos -1; the packet it starts ends on the next page
    "page ending no packet": (
        _pre() + [ogg.page(0, -1, 7, 2, [255], B[:255]), ogg.page(5, 77, 7, 3, [45], B[255:])],
        (0, 4, 0),
        [(50, 300, 77, 1, 3)]),
}


def hand_rows(name):
    return np.array(HAND[name][2], np.int64).reshape(-1, 5)


@pytest.mark.parametrize("name", sorted(HAND))
def test_oracle_on_hand_worked_files(name):
    pages, (status, npages, holes), rows = HAND[name]
    r = ogg.demux(b"".join(pages), 100)
    assert (r["status"], r["pages"], r["holes"], r["dropped"], r["foreign"]) == (status, npages, holes, 0, 0)
    assert r["hdr"] == [(0, 30), (30, 10), (40, 10)] and r["hdr_data"] == H
    assert np.array_equal(ogg.packet_table(r), hand_rows(name))
    if name == "granulepos mid-packet":
        assert r["pkt_data"][1] == B
