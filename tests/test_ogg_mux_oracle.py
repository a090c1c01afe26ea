"""The Ogg mux oracle (oracle/ogg_mux.py), without a GPU:
- seven cases worked out by hand from libogg's page rules, with their pages written out literally through
  oracle.ogg.page (CRCs included): the header pages, the 4096-byte / 4-packet rule, the 255-value cap, a packet
  continued over pages, zero-length and 255-byte packets, the e_o_s page;
- oracle.ogg.demux of the muxed file gives back every packet, granulepos on page-final packets only, e_o_s on the last;
- seeded cuts through mux_pieces (calls with no new packets, cuts inside a page and inside a packet) give the one-shot
  bytes, and case D cut after packet 4 keeps one packet with 18 of its values on pages;
- the stock encoder's streams (reference build) round-trip."""
import numpy as np
import pytest

from oracle import decode
from oracle import ogg
from oracle import ogg_mux

SERIAL = 0x1234ABCD


def _bytes(rng, n):
    return bytes(rng.integers(0, 256, n, dtype=np.uint8))


def _headers(rng, sizes=(30, 100, 3000)):
    """header packets of these sizes, the first with the identification magic the demux looks for"""
    return [(b"\x01vorbis" if k == 0 else b"") + _bytes(rng, n - (7 if k == 0 else 0)) for k, n in enumerate(sizes)]


def _g(k):
    """granulepos of audio packet k (1-based) in the hand-worked cases"""
    return 1000 * k + 7


def _lace(n):
    return [255] * (n // 255) + [n % 255]


def _case(name):
    """(headers, audio packets, literal pages) of a hand-worked case; pages as (flags, granulepos, lacing, body)"""
    rng = np.random.default_rng(sum(map(ord, name)))
    hs = (30, 100_000 if name == "B" else 100, 3000)
    hdr = _headers(rng, hs)
    sizes = {"A": [1000] * 10, "B": [500], "C": [5000] * 6, "D": [20000] * 5, "E": [10] * 300, "F": [1024] * 8,
             "G": [0, 255, 510]}[name]
    pk = [_bytes(rng, n) for n in sizes]
    blob = b"".join(pk)
    H = hdr[0] + hdr[1] + hdr[2]
    if name == "B":
        lh = _lace(100_000) + _lace(3000)
        head = [(2, 0, [30], hdr[0]), (0, -1, lh[:255], H[30:30 + 65025]), (1, 0, lh[255:], H[30 + 65025:])]
    else:
        head = [(2, 0, [30], hdr[0]), (0, 0, [100] + _lace(3000), hdr[1] + hdr[2])]
    if name == "A":
        per = [255, 255, 255, 235]
        aud = [(0, _g(5), per * 5, blob[:5000]), (4, _g(10), per * 5, blob[5000:])]
    elif name == "B":
        aud = [(4, _g(1), [255, 245], blob)]
    elif name == "C":
        aud = [(0, _g(4), _lace(5000) * 4, blob[:20000]), (4, _g(6), _lace(5000) * 2, blob[20000:])]
    elif name == "D":
        lac = _lace(20000) * 5
        aud = [(0, _g(3), lac[:255], blob[:64590]), (5, _g(5), lac[255:], blob[64590:])]
    elif name == "E":
        aud = [(0, _g(255), [10] * 255, blob[:2550]), (4, _g(300), [10] * 45, blob[2550:])]
    elif name == "F":
        aud = [(0, _g(5), _lace(1024) * 5, blob[:5120]), (4, _g(8), _lace(1024) * 3, blob[5120:])]
    else:
        aud = [(4, _g(3), [0, 255, 0, 255, 255, 0], blob)]
    pages = [ogg.page(f, g, SERIAL, seq, lac, body) for seq, (f, g, lac, body) in enumerate(head + aud)]
    return hdr, pk, pages


CASES = "ABCDEFG"
TOTAL_A = 13292


def hand_case(name):
    """(headers, packets, granules, eos, literal pages) of hand-worked case `name` (also used by the GPU tests)"""
    hdr, pk, pages = _case(name)
    gr = [_g(k + 1) for k in range(len(pk))]
    eos = [k == len(pk) - 1 for k in range(len(pk))]
    return hdr, pk, gr, eos, pages


@pytest.mark.parametrize("name", CASES)
def test_hand_worked_cases(name):
    hdr, pk, gr, eos, want = hand_case(name)
    got = ogg_mux.mux(hdr, pk, gr, eos, SERIAL)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "case %s page %d: %s against %s" % (name, i, g[:32].hex(), w[:32].hex())
    assert len(got) == len(want), "case %s: %d pages, want %d" % (name, len(got), len(want))
    if name == "A":
        assert len(b"".join(got)) == TOTAL_A
    r = ogg.demux(b"".join(got), len(pk) + 1)
    assert r["status"] == 0 and r["hdr_data"] == hdr and r["pkt_data"] == pk


def test_case_d_cut_after_packet_4():
    hdr, pk, gr, eos, want = hand_case("D")
    st, pages, carry = ogg_mux.mux_call(ogg_mux.fresh_carry(SERIAL), hdr, pk[:4], gr[:4], eos[:4])
    assert st == 0 and pages == want[:3]
    assert carry == dict(serial=SERIAL, pageno=3, state=ogg_mux.WRITING, kept=1, kept_segs=18)
    st, pages, carry = ogg_mux.mux_call(carry, None, pk[3:], gr[3:], eos[3:])
    assert st == 0 and pages == want[3:] and pages[0][5] == 5
    assert carry == dict(serial=SERIAL, pageno=4, state=ogg_mux.DONE, kept=0, kept_segs=0)


def seeded_stream(rng, n, eos=True, big=False):
    """headers and n audio packets with sizes that hit the page rules' edges"""
    edge = [0, 1, 254, 255, 256, 509, 510, 511, 764, 765, 766, 4095, 4096, 4097, 1020, 1024]
    if big:
        edge += [65024, 65025, 65026, 70000, 130050]
    sizes = [int(rng.choice(edge)) if rng.random() < 0.5 else int(rng.integers(0, 3000)) for _ in range(n)]
    pk = [_bytes(rng, m) for m in sizes]
    gr = list(np.cumsum(rng.integers(0, 2048, n)).astype(int) + 1)
    return _headers(rng), pk, [int(g) for g in gr], [eos and k == n - 1 for k in range(n)]


def seeded_cuts(rng, n, calls):
    """non-decreasing cut points in [0, n], repeats (calls with no new packets) included"""
    return sorted(int(x) for x in rng.integers(0, n + 1, calls))


@pytest.mark.parametrize("seed", range(12))
def test_demux_of_mux(seed):
    rng = np.random.default_rng(seed)
    hdr, pk, gr, eos = seeded_stream(rng, int(rng.integers(1, 400)), big=seed % 3 == 0)
    pages = ogg_mux.mux(hdr, pk, gr, eos, SERIAL + seed)
    r = ogg.demux(b"".join(pages), len(pk) + 1)
    assert r["status"] == 0 and r["pages"] == len(pages) and r["dropped"] == 0 and r["holes"] == 0
    assert r["hdr_data"] == hdr and r["pkt_data"] == pk
    t = ogg.packet_table(r)
    assert (t[:, 3] == np.array(eos)).all(), "e_o_s on the last packet only"
    # granulepos: the packet's own on the last packet that ends on each page, -1 on every other
    page_ends = []
    for p in pages[2 if len(hdr[1]) + len(hdr[2]) < 255 * 255 else 3:]:
        lac = list(p[27:27 + p[26]])
        page_ends.append(sum(1 for v in lac if v < 255))
    last = np.full(len(pk), False)
    k = 0
    for n in page_ends:
        k += n
        if n:
            last[k - 1] = True
    assert k == len(pk)
    assert (t[:, 2] == np.where(last, gr, -1)).all()


@pytest.mark.parametrize("seed", range(12))
def test_pieces_equal_one_call(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(1, 300))
    hdr, pk, gr, eos = seeded_stream(rng, n, eos=seed % 4 != 3, big=seed % 2 == 0)
    one = ogg_mux.mux(hdr, pk, gr, eos, 77)
    _, whole = ogg_mux.mux_pieces(hdr, pk, gr, eos, 77, [])
    for cuts in (seeded_cuts(rng, n, int(rng.integers(1, 12))), list(range(n + 1)), [0, 0, n, n]):
        pages, carries = ogg_mux.mux_pieces(hdr, pk, gr, eos, 77, cuts)
        assert b"".join(pages) == b"".join(one), "cuts %s" % cuts
        assert carries[-1] == whole[-1]
        assert all(c["kept"] <= 254 for c in carries)
    if not eos[-1]:
        assert whole[-1]["state"] == ogg_mux.WRITING
    else:
        assert whole[-1] == dict(serial=77, pageno=len(one), state=ogg_mux.DONE, kept=0, kept_segs=0)


def test_refusals():
    rng = np.random.default_rng(5)
    hdr, pk, gr, eos = seeded_stream(rng, 10)
    fresh = ogg_mux.fresh_carry(1)
    done = dict(fresh, state=ogg_mux.DONE, pageno=9)
    for carry, h, e in ((fresh, None, eos),                               # fresh without headers
                        (done, hdr, eos),                                 # packets on a done carry
                        (fresh, hdr, [True] + eos[1:]),                   # e_o_s before the last row
                        (dict(fresh, state=1, kept=11), hdr, eos)):       # npkt below kept
        st, pages, c = ogg_mux.mux_call(carry, h, pk, gr, e)
        assert st == ogg_mux.EINVAL and pages == [] and c == carry
    assert ogg_mux.mux_call(done, None, [], [], []) == (0, [], done)


def test_stock_streams_round_trip():
    if not decode.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    from conftest import probe_signal
    for ch, rate, q in [(2, 44100, 0.5), (2, 44100, -0.1)]:
        p = decode.encode(ch, rate, q, probe_signal(ch, rate, 0.7, seed=31))
        pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
        gr = [int(g) for g in p.meta[3:, 2]]
        eos = [bool(e) for e in p.meta[3:, 3]]
        assert eos[-1] and not any(eos[:-1])
        pages = ogg_mux.mux(pk[:3], pk[3:], gr, eos, 5)
        r = ogg.demux(b"".join(pages), len(pk))
        assert r["status"] == 0 and r["hdr_data"] == pk[:3] and r["pkt_data"] == pk[3:]
        got = ogg.packet_table(r)[:, 2]
        assert ((got == -1) | (got == gr)).all() and got[-1] == gr[-1]
