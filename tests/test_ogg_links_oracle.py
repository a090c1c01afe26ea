"""The link rule of vb200_ogg_links (include/vorbis_b200.h) in oracle/ogg_links.py, without a GPU:
- ten small files worked out by hand, with their link offsets written out literally (not produced by the oracle): one
  link, three links of distinct serials, two links of one serial, a multiplexed link whose Vorbis BOS page comes second,
  a truncated link (no EOS page) before a BOS page, garbage and a foreign page between an EOS page and the next BOS
  page, a file that starts with data pages, a damaged BOS page whose link merges into the one before, a failed capture
  whose claimed extent crosses the next link's start (the earlier link's demux ends there), and an empty file;
- concatenating any run of consecutive streams that oracle/ogg_mux.py writes gives back exactly their offsets."""
import numpy as np

from oracle import ogg
from oracle import ogg_links
from oracle import ogg_mux
from test_ogg_demux_oracle import H
from test_ogg_mux_oracle import seeded_stream


def _audio(serial, seq, eos=False, n=20):
    return ogg.page(4 if eos else 0, 1000 + seq, serial, seq, [n], bytes(range(seq, seq + n)))


def _link(serial, eos=True):
    """a 203-byte Vorbis link (155 bytes without its EOS page): the 58-byte BOS page with the identification header,
    a 49-byte page with the other two, two 48-byte audio pages"""
    pages = [ogg.page(2, 0, serial, 0, [30], H[0]), ogg.page(0, 0, serial, 1, [10, 10], H[1] + H[2]),
             _audio(serial, 2), _audio(serial, 3, eos=True)]
    return b"".join(pages if eos else pages[:3])


THEORA_BOS = ogg.page(2, 0, 50, 0, [30], b"\x80theora" + bytes(23))                 # 58 bytes
THEORA_DATA = ogg.page(0, 0, 50, 1, [20], bytes(20))                                  # 48 bytes
GARBAGE = b"junk O junk"                                                              # 11 bytes, no page
# "OggS" and a header that claims one 200-byte segment, with no 'O' after the first byte: 28 bytes whose claimed
# extent is 228 bytes
FAKE = b"OggS" + bytes(22) + bytes([1, 200])


def _damaged_bos(serial):
    b = bytearray(_link(serial))
    b[40] ^= 0x01                                                                     # a byte of the BOS page's body
    return bytes(b)


# name -> (file, its link offsets from the file's first byte, the file's end last)
CASES = {
    "single link": (_link(7), [0, 203]),
    "three serials": (_link(7) + _link(8) + _link(9), [0, 203, 406, 609]),
    "same serial": (_link(7) + _link(7), [0, 203, 406]),
    # Theora BOS 58, Vorbis BOS 58, headers 49, Theora data 48, audio 48 + 48: 309 bytes, then a 203-byte link
    "multiplexed": (THEORA_BOS + _link(7)[:107] + THEORA_DATA + _link(7)[107:] + _link(8), [0, 309, 512]),
    "truncated link": (_link(7, eos=False) + _link(8), [0, 155, 358]),
    "garbage and foreign after EOS": (_link(7) + GARBAGE + THEORA_DATA + _link(8), [0, 262, 465]),
    "data pages first": (_audio(7, 2) + _audio(7, 3) + _link(8), [0, 96, 299]),
    # the middle link's BOS page fails its CRC: its headers page follows link 0's EOS page and starts nothing
    "damaged BOS": (_link(7) + _damaged_bos(8) + _link(9), [0, 406, 609]),
    # the fake header at 155 claims bytes up to 383: the whole-file walk fails its CRC, resyncs at the EOS page (183)
    # and finds link 1 at 231
    "failed capture across the boundary": (_link(7, eos=False) + FAKE + _audio(7, 3, eos=True) + _link(8),
                                           [0, 231, 434]),
    "empty": (b"", [0, 0]),
}


def table(files):
    """(link_first, link_off) of files laid back to back, as vb200_ogg_links writes them, from oracle.ogg_links.links"""
    first, off, at = [0], [], 0
    for f in files:
        starts = ogg_links.links(f)[:-1]
        off += [at + s for s in starts]
        first.append(first[-1] + len(starts))
        at += len(f)
    return np.array(first, np.int64), np.array(off + [at], np.int64)


def literal_table(names):
    first, off, at = [0], [], 0
    for n in names:
        buf, want = CASES[n]
        off += [at + s for s in want[:-1]]
        first.append(first[-1] + len(want) - 1)
        at += len(buf)
    return np.array(first, np.int64), np.array(off + [at], np.int64)


def test_hand_worked_files():
    for name, (buf, want) in CASES.items():
        assert ogg_links.links(buf) == want, "%s: %s" % (name, ogg_links.links(buf))
    names = list(CASES)
    got, lit = table([CASES[n][0] for n in names]), literal_table(names)
    assert np.array_equal(got[0], lit[0]) and np.array_equal(got[1], lit[1])


def test_links_demux():
    """what the demux makes of each case's links"""
    links = lambda name: [CASES[name][0][a:b] for a, b in zip(CASES[name][1], CASES[name][1][1:])]  # noqa: E731
    for name in ("three serials", "same serial", "truncated link", "garbage and foreign after EOS", "damaged BOS"):
        for k, lk in enumerate(links(name)):
            r = ogg.demux(lk, 8)
            assert r["status"] == 0 and r["hdr_data"] == H and r["chained"] == 0, (name, k)
    assert [ogg.demux(lk, 8)["serial"] for lk in links("same serial")] == [7, 7]
    r = ogg.demux(links("multiplexed")[0], 8)
    assert (r["status"], r["serial"], r["foreign"], r["pages"]) == (0, 7, 2, 4)
    r = ogg.demux(links("garbage and foreign after EOS")[0], 8)
    # two failed captures (the garbage's first byte, then its 'O'); the foreign page after them ends the walk
    assert (r["pages"], r["dropped"], r["foreign"]) == (4, 2, 0)
    merged, last = (ogg.demux(lk, 8) for lk in links("damaged BOS"))          # link 8 lost its BOS page
    assert (merged["serial"], merged["pages"], merged["foreign"], last["serial"]) == (7, 4, 0, 9)
    assert merged["dropped"] >= 1
    first = links("data pages first")
    assert ogg.demux(first[0], 8)["status"] == ogg.ENOTVORBIS and ogg.demux(first[1], 8)["serial"] == 8
    assert ogg_links.links(GARBAGE) == [0, len(GARBAGE)] and ogg.demux(GARBAGE, 8)["status"] == ogg.ENOTVORBIS
    # the failed capture across the boundary: link 0's demux ends at the fake header, without its EOS page, where
    # the whole file's demux drops one capture and takes it
    buf = CASES["failed capture across the boundary"][0]
    r0, whole = ogg.demux(links("failed capture across the boundary")[0], 8), ogg.demux(buf, 8)
    assert (r0["pages"], r0["dropped"], len(r0["packets"]), r0["chained"]) == (3, 0, 1, 0)
    assert (whole["pages"], whole["dropped"], len(whole["packets"]), whole["chained"]) == (4, 1, 2, 1)


def test_muxed_streams():
    """N streams from oracle.ogg_mux: every run of consecutive streams, concatenated, gives their offsets"""
    rng = np.random.default_rng(31)
    files = []
    for s in range(7):
        hdr, pk, gr, eos = seeded_stream(rng, int(rng.integers(0, 12)), eos=s != 3)
        files.append(b"".join(ogg_mux.mux(hdr, pk, gr, eos, 0x100 + (s % 2))))   # neighbours share serials
    at = np.concatenate([[0], np.cumsum([len(f) for f in files])])
    for i in range(len(files)):
        for j in range(i + 1, len(files) + 1):
            got = ogg_links.links(b"".join(files[i:j]))
            assert got == list(at[i:j + 1] - at[i]), (i, j, got)
