"""The Ogg demux rules at the edges stock files never reach, as literal tables worked out by hand (not produced by
oracle/ogg.py), on the oracle alone; tests/test_gpu_ogg_edges.py runs the same files on the device:
- ogg.crc32 equals a bit-at-a-time long division by 0x04c11db7 (and the CRC-32/CKSUM check value without its final
  xor), so the table the oracle and the kernel share is pinned on its own;
- pages of every total length 28..31 (lanes of the kernel's CRC split with empty chunks), 1024..1055 (every residue mod
  32), 32k and 32k +- 1, and 65 307 (255 segments of 255) are accepted; the same pages with one bit flipped at the first
  byte, at the last byte of the first 32nd of the page and the first byte of the second, at the last byte, in the CRC
  field and in a lacing value are one failed capture (plus one per 'O' byte after it) followed by one hole;
- sequence numbers that wrap from 0xFFFFFFFF to 0 leave no hole, 0xFFFFFFFF -> 1 leaves one;
- granulepos 2^32 + 5, 2^40, 2^63 - 1 and -2 are carried exactly on page-final packets;
- empty pages (no segments): mid-stream, while a packet is pending, and as the EOS page (no packet gets e_o_s);
- an EOS page whose last lacing value is 255 (the unfinished packet is not returned);
- a Skeleton-like stream's BOS page before the Vorbis one, and Vorbis pages of version 1 (foreign);
- a continued page after a hole while a packet spanning pages was pending;
- a capture whose lacing or body runs past the end of the file ends the walk;
- runs of 'O' bytes and bad-CRC "OggS" prefixes, with the next page 32, 33 and 64 bytes after a failed capture (the
  edges of the kernel's 32-byte resync windows), and 'O' bytes up to the last byte of the file;
- files of 0, 1 and 26 bytes have no Vorbis stream."""
import numpy as np
import pytest

from oracle import ogg
from test_ogg_demux_oracle import H, _body, _pre

S = 7                                           # the serial of the Vorbis stream in every file below


def _pg(flags, gp, seq, lacing, body, serial=S, version=0):
    return ogg.page(flags, gp, serial, seq, lacing, body, version)


def crc_long_division(data):
    """the Ogg CRC as the remainder of data(x) * x^32 divided by 0x104c11db7, one bit at a time"""
    reg = 0
    for bit in [(b >> (7 - k)) & 1 for b in data for k in range(8)] + [0] * 32:
        top = reg >> 31
        reg = ((reg << 1) | bit) & 0xFFFFFFFF
        if top:
            reg ^= 0x04C11DB7
    return reg


# ---- page lengths for the CRC split -------------------------------------------------------------------------------
CRC_LENGTHS = sorted(set([28, 29, 30, 31] + [1024 + r for r in range(32)] +
                         [32 * k + d for k in (1, 2, 8, 64, 511, 2040) for d in (-1, 0, 1)] + [65307]))


def lacing_of(n):
    """lacing values of a page of n bytes in all (27 + segments + body): one packet ended on it, padded with
    zero-length packets, or 255-byte segments only when the length allows nothing else"""
    nseg = max(1, -(-(n - 27) // 256))
    body = n - 27 - nseg
    q, r = divmod(body, 255)
    lace = [255] * nseg if q == nseg else [255] * q + [r] + [0] * (nseg - q - 1)
    assert len(lace) == nseg and sum(lace) == body and q <= nseg
    return lace


def flip_positions(n):
    """the first byte of the kernel's lane 0 chunk, the last byte of lane 0's and the first of lane 1's chunks, the
    last byte of the page, a byte of the CRC field and the first lacing value"""
    chunk = -(-n // 32)
    return sorted({0, chunk - 1, chunk, n - 1, 22 + n % 4, 27})


def _flip(page, i):
    b = bytearray(page)
    b[i] ^= (b[i] & -b[i]) or 1                 # the lowest set bit: a lacing value only shrinks
    return bytes(b)


def crc_case(n, pos=None):
    """(file, expected (status, pages, dropped, holes, foreign, chained), rows, payloads): the headers, one audio page
    of n bytes (bit-flipped at pos unless None) and an EOS page"""
    lace = lacing_of(n)
    body = bytes((n * 7 + 13 * i) & 255 for i in range(sum(lace)))
    ends = [i for i, v in enumerate(lace) if v < 255]
    gp = 1000 + n if ends else -1
    audio = _pg(0, gp, 2, lace, body)
    assert len(audio) == n
    eos = _pg(5, 9000, 3, [10, 3], bytes(10) + b"eos") if lace[-1] == 255 else _pg(4, 9000, 3, [3], b"eos")
    if pos is not None:
        audio = _flip(audio, pos)
        return (b"".join(_pre() + [audio, eos]), (0, 3, 1 + audio[1:].count(b"O"), 1, 0, 0), [(50, 3, 9000, 1, 4)],
                [b"eos"])
    rows, pay, at, k, cur = [], [], 50, 3, 0
    for i, v in enumerate(lace):
        cur += v
        if v < 255:
            rows.append((at, cur, gp if i == ends[-1] else -1, 0, k))
            pay.append(body[at - 50:at - 50 + cur])
            at, k, cur = at + cur, k + 1, 0
    if cur:
        rows.append((at, cur + 10, -1, 0, k))
        pay.append(body[at - 50:] + bytes(10))
        at, k = at + cur + 10, k + 1
    rows.append((at, 3, 9000, 1, k))
    return b"".join(_pre() + [audio, eos]), (0, 4, 0, 0, 0, 0), rows, pay + [b"eos"]


def crc_cases():
    """[(name, case)] for every length, clean and flipped at each position"""
    out = []
    for n in CRC_LENGTHS:
        out.append(("%d bytes" % n, crc_case(n)))
        out += [("%d bytes, bit flipped at %d" % (n, i), crc_case(n, i)) for i in flip_positions(n)]
    return out


# ---- stream rules, worked out by hand -----------------------------------------------------------------------------
# Headers H: 30, 10 and 10 bytes, so the first audio packet starts at offset 50 of the file's own byte range.
A5, D7, C300, C600, E275, F8 = _body(5, 0), _body(7, 2), _body(300, 1), _body(600, 9), _body(275, 10), _body(8, 11)
G6, G7, G8, G9, G4 = _body(6, 3), _body(7, 4), _body(8, 5), _body(9, 6), _body(4, 7)
BAD = b"OggS" + bytes(23)                       # 27 bytes, no segments, a CRC field of 0 (its CRC is not 0)


def _wrap_pre():
    return [_pg(2, 0, 0xFFFFFFFE, [30], H[0]), _pg(0, 0, 0xFFFFFFFF, [10, 10, 255], H[1] + H[2] + C300[:255])]


def _skeleton(flags, seq, body):
    return ogg.page(flags, 0, 9, seq, [len(body)] if body else [], body)


# name -> (pages, expected (status, pages, dropped, holes, foreign, chained), rows (offset, bytes, granulepos, e_o_s,
# packetno), the packets' bytes)
EDGE = {
    # C starts on the 0xFFFFFFFF page and ends on page 0: the sequence continues, C is whole and gets -1 (A ends later
    # on the same page)
    "sequence wraps": (
        _wrap_pre() + [_pg(1, 100, 0, [45, 5], C300[255:] + A5), _pg(4, 200, 1, [7], D7)],
        (0, 4, 0, 0, 0, 0),
        [(50, 300, -1, 0, 3), (350, 5, 100, 0, 4), (355, 7, 200, 1, 5)], [C300, A5, D7]),
    # 0xFFFFFFFF -> 1: one hole; C's first 255 bytes are dropped, packetno 3 is the hole, the continued page's 45-byte
    # fragment is skipped and A lands where C began
    "sequence wraps with a hole": (
        _wrap_pre() + [_pg(1, 100, 1, [45, 5], C300[255:] + A5), _pg(4, 200, 2, [7], D7)],
        (0, 4, 0, 1, 0, 0),
        [(50, 5, 100, 0, 4), (55, 7, 200, 1, 5)], [A5, D7]),
    # all 64 bits of the granulepos, on the last packet ending on each page; -1 on the others
    "granulepos past 32 bits": (
        _pre() + [_pg(0, 2 ** 32 + 5, 2, [5], A5), _pg(0, 2 ** 40, 3, [6, 7], G6 + G7),
                  _pg(0, 2 ** 63 - 1, 4, [8], G8), _pg(4, -2, 5, [9, 4], G9 + G4)],
        (0, 6, 0, 0, 0, 0),
        [(50, 5, 2 ** 32 + 5, 0, 3), (55, 6, -1, 0, 4), (61, 7, 2 ** 40, 0, 5), (68, 8, 2 ** 63 - 1, 0, 6),
         (76, 9, -1, 0, 7), (85, 4, -2, 1, 8)], [A5, G6, G7, G8, G9, G4]),
    # a page with no segments is taken (and counted) and ends no packet; its granulepos goes nowhere
    "empty page mid-stream": (
        _pre() + [_pg(0, 100, 2, [5], A5), _pg(0, 150, 3, [], b""), _pg(4, 200, 4, [7], D7)],
        (0, 5, 0, 0, 0, 0),
        [(50, 5, 100, 0, 3), (55, 7, 200, 1, 4)], [A5, D7]),
    # ... and leaves a pending packet pending
    "empty page while a packet is pending": (
        _pre() + [_pg(0, 100, 2, [5, 255], A5 + C300[:255]), _pg(1, -1, 3, [], b""), _pg(5, 300, 4, [45], C300[255:])],
        (0, 5, 0, 0, 0, 0),
        [(50, 5, 100, 0, 3), (55, 300, 300, 1, 4)], [A5, C300]),
    # an empty EOS page: no packet gets e_o_s, and the walk ends there (the page after it is not read)
    "empty EOS page": (
        _pre() + [_pg(0, 100, 2, [5], A5), _pg(4, 100, 3, [], b""), _pg(0, 200, 4, [7], D7)],
        (0, 4, 0, 0, 0, 0),
        [(50, 5, 100, 0, 3)], [A5]),
    # the EOS flag belongs to the last segment, which ends no packet: D gets the granulepos but not e_o_s, and the
    # unfinished packet is not returned
    "EOS page ending in lacing 255": (
        _pre() + [_pg(0, 100, 2, [5], A5), _pg(4, 200, 3, [7, 255], D7 + C300[:255])],
        (0, 4, 0, 0, 0, 0),
        [(50, 5, 100, 0, 3), (55, 7, 200, 0, 4)], [A5, D7]),
    # a Skeleton-like stream (serial 9) begins first and interleaves; its EOS page does not end the Vorbis walk
    "other stream's BOS page first": (
        [_skeleton(2, 0, b"fishead\0" + bytes(56)), _pre()[0], _skeleton(0, 1, b"fisbone\0" + bytes(44)), _pre()[1],
         _skeleton(4, 2, b""), _pg(0, 100, 2, [5], A5), _pg(4, 200, 3, [7], D7)],
        (0, 4, 0, 0, 3, 0),
        [(50, 5, 100, 0, 3), (55, 7, 200, 1, 4)], [A5, D7]),
    # a Vorbis identification page of version 1 (serial 8) is not the stream; a version-1 page of serial 7 is foreign
    "pages of version 1": (
        [_pg(2, 0, 0, [30], H[0], serial=8, version=1)] + _pre() +
        [_pg(0, 100, 2, [5], A5), _pg(0, 150, 3, [6], G6, version=1), _pg(4, 200, 3, [7], D7)],
        (0, 4, 0, 0, 2, 0),
        [(50, 5, 100, 0, 3), (55, 7, 200, 1, 4)], [A5, D7]),
    # C (600 bytes) spans pages 2 and 3 and is pending when page 4 (C's end and E's start) is missing: C's 510 bytes
    # are dropped, packetno 4 is the hole, page 5's leading fragment (E's end) is skipped and F lands where C began
    "continued page after a hole": (
        _pre() + [_pg(0, 100, 2, [5, 255], A5 + C600[:255]), _pg(1, -1, 3, [255], C600[255:510]),
                  _pg(5, 300, 5, [20, 8], E275[255:] + F8)],
        (0, 5, 0, 1, 0, 0),
        [(50, 5, 100, 0, 3), (55, 8, 300, 1, 5)], [A5, F8]),
    # a capture whose lacing table (200 segments) runs past the end of the file, valid pages inside its length
    "lacing past the end": (
        _pre() + [_pg(0, 100, 2, [5], A5), b"OggS" + bytes(22) + bytes([200]), _pg(4, 200, 3, [7], D7)],
        (0, 3, 0, 0, 0, 0),
        [(50, 5, 100, 0, 3)], [A5]),
    # a capture whose body (510 bytes) runs past the end of the file
    "body past the end": (
        _pre() + [_pg(0, 100, 2, [5], A5), b"OggS" + bytes(22) + bytes([2, 255, 255]), _pg(4, 200, 3, [7], D7)],
        (0, 3, 0, 0, 0, 0),
        [(50, 5, 100, 0, 3)], [A5]),
    # failed captures: 70 'O' bytes, two bad "OggS" pages, three single 'O' bytes 32, 33 and 64 bytes before the next
    # page, and 40 'O' bytes at the end of the file of which the first 14 have 27 bytes left: 70+2+3+14 = 89 dropped
    "'O' runs and bad captures": (
        _pre() + [_pg(0, 100, 2, [5], A5), b"O" * 70, BAD, b"O" + bytes(31), _pg(0, 150, 3, [6], G6),
                  b"O" + bytes(32), _pg(0, 170, 4, [7], D7), b"O" + bytes(63), BAD, _pg(4, 200, 5, [4], G4),
                  b"O" * 40],
        (0, 6, 89, 0, 0, 0),
        [(50, 5, 100, 0, 3), (55, 6, 150, 0, 4), (61, 7, 170, 0, 5), (68, 4, 200, 1, 6)], [A5, G6, D7, G4]),
}

# too short to hold a page: between ordinary files in the device test
SHORT = [b"", b"O", b"OggS" + bytes(22)]
NOT_VORBIS = (ogg.ENOTVORBIS, 0, 0, 0, 0, 0)


def check_demux(r, expect, rows, payloads, what, hdr=True):
    """a demux result in oracle.ogg.demux's form (offsets from the file's first byte) against a literal table"""
    got = tuple(r[k] for k in ("status", "pages", "dropped", "holes", "foreign", "chained"))
    assert got == expect, "%s: %s" % (what, got)
    if hdr:
        assert r["serial"] == S and r["hdr"] == [(0, 30), (30, 10), (40, 10)] and r["hdr_data"] == H, what
    t = ogg.packet_table(r)
    assert np.array_equal(t, np.array(rows, np.int64).reshape(-1, 5)), "%s: %s" % (what, t.tolist())
    assert r["pkt_data"] == payloads, what


def test_crc32_is_the_long_division():
    assert ogg.crc32(b"123456789") == 0x765E7680 ^ 0xFFFFFFFF           # CRC-32/CKSUM's check value, no final xor
    rng = np.random.default_rng(11)
    for n in list(range(40)) + [255, 1000]:
        b = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        assert ogg.crc32(b) == crc_long_division(b), n
    at = len(b"".join(_pre()))
    for n in [n for n in CRC_LENGTHS if n < 1100] + [65307]:
        pg = bytearray(crc_case(n)[0][at:at + n])                  # the audio page, after the headers' pages
        want = int.from_bytes(pg[22:26], "little")
        pg[22:26] = bytes(4)
        assert crc_long_division(pg) == want, n


def test_crc_page_lengths():
    cases = crc_cases()
    assert len(cases) > 300
    for name, (buf, expect, rows, payloads) in cases:
        check_demux(ogg.demux(buf, 400), expect, rows, payloads, name)


@pytest.mark.parametrize("name", sorted(EDGE))
def test_stream_rules(name):
    pages, expect, rows, payloads = EDGE[name]
    check_demux(ogg.demux(b"".join(pages), 100), expect, rows, payloads, name)


def test_preconditions_of_the_literal_files():
    """what the hand-worked counts assume about the bytes"""
    assert ogg.crc32(BAD) != 0 and b"O" not in BAD[1:]
    assert len(b"".join(EDGE["lacing past the end"][0][3:])) < 27 + 200
    assert len(b"".join(EDGE["body past the end"][0][3:])) < 27 + 2 + 510


def test_short_files():
    for buf in SHORT:
        r = ogg.demux(buf, 10)
        assert tuple(r[k] for k in ("status", "pages", "dropped", "holes", "foreign", "chained")) == NOT_VORBIS
        assert r["hdr"] == [] and r["packets"] == []
