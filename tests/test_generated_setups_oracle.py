"""Generated Vorbis setups (tests/vorbis_gen.py) against the stock decoder, without a GPU:
- every header set of both corpora is accepted by vorbis_synthesis_headerin, and parses back to its description;
- the structured audio packets decode through vorbis_synthesis with no OV_EBADPACKET, and the reference reads each one
  to its last byte (so to the last partition of the last residue stage) where a channel carries a floor;
- the corpus reaches what the device decoder's limits name (counted on the parsed headers, listed in the message)."""
import numpy as np
import pytest

import vorbis_gen as G
from oracle import decode
from oracle import decode_packets as dp
from oracle import decode_streams as ds

ALL = G.INSIDE + sorted(G.OUTSIDE)
NPKT = 14


def _need():
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def corpus(name, granule=True, page_final=False):
    """(description, structured packets, Packets of the stream) of one generated setup"""
    d = G.setup(name)
    pk, _ = G.packets(d, 1000 + ALL.index(name), NPKT)
    return d, pk, G.stream(d, pk, page_final=page_final, granule=granule)


def headers_of(p):
    return [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:3, :2]]


@pytest.mark.parametrize("name", ALL)
def test_headers_accepted_and_parse_back(name):
    _need()
    d, pk, p = corpus(name)
    W = dp.ref_headers(p, pk)                         # raises where vorbis_synthesis_headerin refuses one
    assert (W >= 0).all()
    h = headers_of(p)
    back = G.read_setup(h[0], h[2])
    for k in ("channels", "bs", "modes", "mappings", "residues"):
        assert back[k] == d[k], k
    for f, g in zip(back["floors"], d["floors"]):
        for k in ("pclass", "mult", "rangebits", "xlist"):
            assert f[k] == g[k], k
    for a, b in zip(back["books"], d["books"]):
        for k in ("dim", "entries", "lengths", "maptype"):
            assert a[k] == b[k], k


@pytest.mark.parametrize("name", ALL)
def test_structured_packets_decode(name):
    _need()
    d, pk, p = corpus(name)
    pcm, rec, modebits = ds.ref_decode(p.buf, p.hdr, p.audio, d["channels"])
    assert modebits == G.ilog(len(d["modes"]) - 1)
    assert (rec[:, 0] == 0).all(), "vorbis_synthesis refused a structured packet: %s" % rec[:, 0]
    assert pcm.shape[1] > 0 and np.isfinite(pcm).all()
    if name in G.OUTSIDE:
        return
    # each packet is read to its end: without its last byte the reference's residue or posts differ.  Where the last
    # codeword's vector is all zeros (quantised values of 0), losing it changes nothing: hence a slack of two packets
    W = dp.ref_headers(p, pk)
    full = dp.ref_staging(p, pk, W, d["bs"], d["channels"])
    cut = [q[:-1] if len(q) > 1 else q for q in pk]
    short = dp.ref_staging(p, cut, W, d["bs"], d["channels"])
    off, _ = dp.layout(W, d["bs"], d["channels"])
    read_to_end, audible = 0, 0
    for k in range(len(pk)):
        audible += bool(full[2][k].any())
        n = d["bs"][W[k]] // 2 * d["channels"]
        a, b = full[0][off[k]:off[k] + n], short[0][off[k]:off[k] + n]
        read_to_end += not np.array_equal(a.view(np.uint32), b.view(np.uint32)) or \
            not np.array_equal(full[1][k], short[1][k])
    assert read_to_end >= audible - 2 and read_to_end > 0, \
        "%d of %d packets with a floor read to their last byte" % (read_to_end, audible)


def _coverage():
    c = {"short": set(), "long": set(), "max_len": 0, "deep_books": 0, "single": 0, "sparse": 0,
         "empty_stage": 0, "maptypes": set(), "mult": set(), "zero_part": 0, "posts_65": 0, "subs": set(),
         "minus1_with_subs3": 0, "res_types": set(), "begin_gt0": 0, "grouping_odd": 0, "classes_64": 0,
         "cascade_gap": 0, "submaps": set(), "chained": 0, "channels": set(), "stages": 0, "stages_to_end": 0,
         "packets_to_end": 0}
    for name in G.INSIDE:
        _, _, p = corpus(name)
        _, enc = G.packets(G.setup(name), 1000 + ALL.index(name), NPKT)    # the packets corpus() wrote
        for k in ("stages", "stages_to_end", "packets_to_end"):
            c[k] += getattr(enc, k)
        h = headers_of(p)
        d = G.read_setup(h[0], h[2])
        c["short"].add(d["bs"][0])
        c["long"].add(d["bs"][1])
        c["channels"].add(d["channels"])
        stage = set()
        for r in d["residues"]:
            for row in r["books"]:
                stage.update(b for b in row if b >= 0)
        for i, b in enumerate(d["books"]):
            L = b["lengths"]
            c["max_len"] = max(c["max_len"], max(L))
            # levels of the device's lookup tables: 10 bits, then 8 per sub-table
            c["deep_books"] += max(L) > 18
            c["single"] += b["entries"] == 1 and L == [1]
            c["sparse"] += b["sparse"] and any(L)
            c["empty_stage"] += not any(L) and i in stage
            if b["maptype"]:
                c["maptypes"].add(b["maptype"])
        used_floors = {f for m in d["mappings"] for f in m["floor"]}
        for i in used_floors:
            f = d["floors"][i]
            c["mult"].add(f["mult"])
            c["zero_part"] += not f["pclass"]
            c["posts_65"] += len(f["xlist"]) + 2 == 65
            for cl in set(f["pclass"]):
                c["subs"].add(f["csubs"][cl])
                c["minus1_with_subs3"] += f["csubs"][cl] == 3 and -1 in f["subbook"][cl]
        for bf, mi in d["modes"]:
            m = d["mappings"][mi]
            c["submaps"].add(m["submaps"])
            cp = m["coupling"]
            c["chained"] += any(a in (x, y) or b in (x, y) for i, (a, b) in enumerate(cp) for (x, y) in cp[:i])
            for s in range(m["submaps"]):
                r = d["residues"][m["residue"][s]]
                bundle = sum(1 for x in m["chmux"] if x == s)
                lim = d["bs"][bf] // 2 * (bundle if r["type"] == 2 else 1)
                n = min(r["end"], lim) - r["begin"]
                if n < r["grouping"]:
                    continue
                c["res_types"].add(r["type"])
                c["begin_gt0"] += r["begin"] > 0
                c["grouping_odd"] += n % r["grouping"] != 0
                c["classes_64"] += len(r["cascade"]) == 64
                c["cascade_gap"] += any(cas != (1 << G.ilog(cas)) - 1 for cas in r["cascade"])   # a clear bit below the top
    return c


def test_corpus_coverage():
    _need()
    c = _coverage()
    sizes = {64, 128, 256, 512, 1024, 2048, 4096, 8192}
    want = [("every block size short", c["short"] >= sizes), ("every block size long", c["long"] >= sizes),
            ("a 32-bit codeword", c["max_len"] == 32), ("a book of >= 3 table levels", c["deep_books"] > 0),
            ("a single-entry book", c["single"] > 0), ("a sparse book", c["sparse"] > 0),
            ("a book without codewords as a stage book", c["empty_stage"] > 0),
            ("lookup types 1 and 2", c["maptypes"] >= {1, 2}), ("floor mult 1-4", c["mult"] >= {1, 2, 3, 4}),
            ("a floor of 0 partitions", c["zero_part"] > 0), ("a floor of 65 posts", c["posts_65"] > 0),
            ("class_subs 0 and 3", c["subs"] >= {0, 3}), ("a -1 subbook under 3 subclass bits", c["minus1_with_subs3"] > 0),
            ("residue types 1 and 2", c["res_types"] >= {1, 2}), ("begin > 0", c["begin_gt0"] > 0),
            ("a grouping that does not divide end - begin", c["grouping_odd"] > 0),
            ("64 classes", c["classes_64"] > 0), ("a cascade with a gap", c["cascade_gap"] > 0),
            ("3 and 4 submaps", c["submaps"] >= {3, 4}), ("chained coupling steps", c["chained"] > 0),
            ("1, 2, 3, 8 and 64 channels", c["channels"] >= {1, 2, 3, 8, 64}),
            ("every residue stage written to its last partition", c["stages"] > 0 and c["stages_to_end"] == c["stages"]),
            ("packets written to the last partition at every stage", c["packets_to_end"] > 0)]
    missing = [what for what, ok in want if not ok]
    assert not missing, "missing %s; reached %s" % (missing, c)


def decode_setup(d):
    """the device-side setup vb200md builds from a decoder of description d (floors, coupling, submaps and the
    reference's windows), for the oracle and for vb200_ctx_create"""
    from test_transform_fp64 import _decode_only_setup
    from vorbis_b200 import abi
    a = dict(_decode_only_setup(*d["bs"]).arrays)
    ch = d["channels"]
    a["channels"] = np.int32(ch)
    a["window0"], a["window1"] = decode.ref_window(d["bs"][0]), decode.ref_window(d["bs"][1])
    a["submaps"] = np.zeros(2, np.int32)
    a["chmux"] = np.zeros((2, abi.MAX_CHANNELS + 1), np.uint8)
    a["coupling_steps"] = np.zeros(2, np.int32)
    a["coupling_mag"] = np.zeros((2, abi.MAX_COUPLING), np.int32)
    a["coupling_ang"] = np.zeros((2, abi.MAX_COUPLING), np.int32)
    for bf, mi in d["modes"][:2]:
        m = d["mappings"][mi]
        a["submaps"][bf] = m["submaps"]
        a["chmux"][bf, :ch] = m["chmux"]
        a["coupling_steps"][bf] = len(m["coupling"])
        for k, (x, y) in enumerate(m["coupling"]):
            a["coupling_mag"][bf, k], a["coupling_ang"][bf, k] = x, y
        for s in range(m["submaps"]):
            f = d["floors"][m["floor"][s]]
            pre = "floor1_%d_%d_" % (bf, s)
            a[pre + "postlist"] = np.array([0, 1 << f["rangebits"]] + f["xlist"], np.int32)
            a[pre + "mult"] = np.int32(f["mult"])
            a[pre + "n"] = np.int32(1 << f["rangebits"])
            for k in ("maxover", "maxunder", "maxerr", "twofitweight", "twofitatten"):
                a[pre + k] = np.float32(0)           # encoder-only fields
    return abi.SetupHolder(a)


@pytest.mark.parametrize("name", G.INSIDE)
def test_oracle_decode_equals_stock(name, oracle_lib):
    """the reference's staging through the oracle's decode_dsp (de-coupling, floor, IMDCT, overlap-add) equals the
    stock decoder's PCM bit for bit: the oracle's transforms pinned to the reference at 64, 128 and 8192 as well"""
    _need()
    from vorbis_b200 import lib as vlib
    d, pk, p = corpus(name, granule=False)           # no granulepos: the stock PCM is every finished sample
    want = decode.stock_decode(p, channels=d["channels"])
    W = dp.ref_headers(p, pk)
    res, posts, present = dp.ref_staging(p, pk, W, d["bs"], d["channels"])
    Wseq = W[None].astype(np.int32)
    co, po, clen, plen = vlib.synthesis_layout(Wseq, list(d["bs"]), d["channels"])
    assert np.array_equal(co[0], dp.layout(W, d["bs"], d["channels"])[0]) and clen == res.size
    got = oracle_lib.Oracle(decode_setup(d)).decode_dsp(Wseq, co, res, posts[None], present[None], po, plen)[0]
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = int((got.view(np.uint32) != want.view(np.uint32)).sum())
    assert bad == 0, "%s: %d of %d samples differ" % (name, bad, want.size)
