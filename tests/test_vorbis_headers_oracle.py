"""vb200_vorbis_headers_parse (vorbis_b200/csrc/vb200_headers.h) against the reference's own reading of the same three
header packets (oracle/ref_headers.c: vorbis_synthesis_headerin x3, vorbis_synthesis_init, then the fields vb200md_setup
reads and the struct vb200md_entropy_new builds):
- stock setups: every one the suite pins (GRID, HIGH and MULTI of tests/test_oracle_vs_ref.py, the 512/4096 setups
  below q0, the four of the Ogg tests) and the managed 128 kbit/s stereo and 64 kbit/s mono encoders.  The parse
  returns 0 and every field equals the reference's, books as multisets of (entry, length, bits, value row as uint32);
- the generated setups of tests/vorbis_gen.py: every INSIDE setup equal to the reference; one_mode, three_modes and
  modes_swapped VB200_EIMPL; floor_wider_than_block, residue_type0 and residue_past_block 0;
- seeded damage: truncations, bit flips, and edits of named fields of the setup header at the bit positions a walk
  of the header records (book counts, dims, entries, codeword lengths and their counts, maptype, q_quant, floor and
  residue book indices, partition and class counts, mapping and mode fields).  The parse fails exactly where the
  reference does, with its code; where the reference accepts, the fields are equal or the result is VB200_EIMPL for a
  reason the reference's state shows; every named field is edited;
- five ordered books of 2^22 entries (a few bytes each): VB200_EIMPL from the table caps, as the reference's state says;
- the same corpus through the parser compiled alone with g++ -fsanitize=address,undefined: no report.
The parse itself is plain host code: none of these needs a GPU."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode, decode_packets as dp, headers as H
from test_gpu_ogg import CASES as OGG_CASES
from test_oracle_vs_ref import GRID
from vorbis_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EIMPL, EBADHEADER, ENOTVORBIS, EVERSION = -130, -133, -132, -134
# every stock setup the suite pins: GRID (which holds HIGH and MULTI), the 512/4096 setups below q0, the Ogg tests' four
STOCK = list(dict.fromkeys(GRID + [(1, 44100, -0.1), (6, 48000, -0.1)] + OGG_CASES))
MANAGED = [(2, 44100, 128000), (1, 44100, 64000)]


def _need():
    if not (H.available() and decode.available() and dp.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def _hdrs(p):
    return [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:3, :2]]


_cache = {}


def stock_headers(ch, rate, q):
    if (ch, rate, q) not in _cache:
        _cache[(ch, rate, q)] = _hdrs(decode.encode(ch, rate, q, probe_signal(ch, rate, 0.2, seed=5)))
    return _cache[(ch, rate, q)]


def managed_headers(ch, rate, br):
    key = ("managed", ch, rate, br)
    if key not in _cache:
        _cache[key] = _hdrs(dp.encode_managed(ch, rate, probe_signal(ch, rate, 0.2, seed=6), nominal_br=br))
    return _cache[key]


def generated_headers(name):
    from test_generated_setups_oracle import corpus, headers_of
    key = ("gen", name)
    if key not in _cache:
        _cache[key] = headers_of(corpus(name)[2])
    return _cache[key]


def mine(h):
    """(code, description) of vb200_vorbis_headers_parse"""
    try:
        v = lib.vorbis_headers(*h)
    except lib.VB200Error as e:
        return e.code, None
    return 0, H.describe(v.c, v.entropy)


def _diff(a, b):
    return [k for k in a if a[k] != b.get(k)]


def check_one(h, what):
    """the parse against the reference on header set h; returns the reference's code (None: not comparable)"""
    rc, why, want, _ = H.ref(*h)
    if rc == H.HANGS:
        return None
    got_rc, got = mine(h)
    if rc:
        assert got_rc == rc, "%s: parse %d, reference %d" % (what, got_rc, rc)
    elif why:
        assert got_rc == EIMPL, "%s: parse %d, reference takes it but %s" % (what, got_rc, H.EIMPL_WHY.get(why, why))
    else:
        assert got_rc == 0, "%s: parse %d, reference 0" % (what, got_rc)
        assert got == want, "%s: fields differ: %s" % (what, _diff(want, got))
    return rc if rc else (EIMPL if why else 0)


@pytest.mark.parametrize("ch,rate,q", STOCK)
def test_stock_setups(ch, rate, q):
    _need()
    assert check_one(stock_headers(ch, rate, q), "stock %s" % ((ch, rate, q),)) == 0


@pytest.mark.parametrize("ch,rate,br", MANAGED)
def test_managed_setups(ch, rate, br):
    _need()
    assert check_one(managed_headers(ch, rate, br), "managed %s" % ((ch, rate, br),)) == 0


def test_generated_setups():
    _need()
    import vorbis_gen as G
    for name in G.INSIDE:
        assert check_one(generated_headers(name), name) == 0, name
    for name in ("one_mode", "three_modes", "modes_swapped"):
        assert check_one(generated_headers(name), name) == EIMPL, name
    for name in ("floor_wider_than_block", "residue_type0", "residue_past_block"):
        assert check_one(generated_headers(name), name) == 0, name


def test_parsed_info():
    _need()
    h = stock_headers(2, 44100, 0.5)
    v = lib.vorbis_headers(*h)
    _, _, _, info = H.ref(*h)
    assert [v.channels, v.rate, *v.bitrates] == info.tolist()
    assert v.blocksizes == [256, 2048] and v.c.n_psy == 0


class _Walk:
    """the bit position, width and name of every field of a well-formed setup header (read as read_setup reads it)"""

    def __init__(self, data):
        self.r = __import__("vorbis_gen").BitReader(data)
        self.fields = []

    def __call__(self, n, name=None):
        if name:
            self.fields.append((self.r.pos, n, name))
        return self.r.read(n)


def setup_fields(setup, channels):
    import vorbis_gen as G
    f = _Walk(setup)
    f(56)
    for _ in range(f(8, "book count") + 1):
        f(24)
        dim, entries = f(16, "book dim"), f(24, "book entries")
        if f(1, "book ordered"):
            n = 0
            f(5, "book minlength")
            while n < entries:
                n += f(G.ilog(entries - n), "book length count")
        else:
            sparse = f(1, "book sparse")
            for _ in range(entries):
                if not sparse or f(1, "book used flag"):
                    f(5, "book length")
        mt = f(4, "book maptype")
        if mt:
            f(64)
            q = f(4, "book q_quant") + 1
            f(1, "book q_sequencep")
            nq = G.maptype1_quantvals(dim, entries) if mt == 1 else entries * dim
            for _ in range(nq):
                f(q)
    for _ in range(f(6, "time count") + 1):
        f(16, "time type")
    for _ in range(f(6, "floor count") + 1):
        f(16, "floor type")
        pcl = [f(4, "floor partition class") for _ in range(f(5, "floor partitions"))]
        cdim = {}
        for c in range(max(pcl, default=-1) + 1):
            cdim[c] = f(3, "floor class dim") + 1
            subs = f(2, "floor class subs")
            if subs:
                f(8, "floor class book")
            for _ in range(1 << subs):
                f(8, "floor subbook")
        f(2, "floor mult")
        rb = f(4, "floor rangebits")
        for c in pcl:
            for _ in range(cdim[c]):
                f(rb, "floor post")
    for _ in range(f(6, "residue count") + 1):
        f(16, "residue type")
        f(24, "residue begin"), f(24, "residue end"), f(24, "residue grouping")
        ncls = f(6, "residue partitions") + 1
        f(8, "residue groupbook")
        cas = []
        for _ in range(ncls):
            c = f(3, "residue cascade")
            if f(1, "residue cascade flag"):
                c |= f(5, "residue cascade high") << 3
            cas.append(c)
        for c in cas:
            for _ in range(bin(c).count("1")):
                f(8, "residue stage book")
    cb = G.ilog(channels - 1)
    for _ in range(f(6, "mapping count") + 1):
        f(16, "mapping type")
        sub = f(4, "mapping submaps") + 1 if f(1, "mapping submap flag") else 1
        if f(1, "mapping coupling flag"):
            for _ in range(f(8, "mapping coupling steps") + 1):
                f(cb, "mapping magnitude"), f(cb, "mapping angle")
        f(2, "mapping reserved")
        if sub > 1:
            for _ in range(channels):
                f(4, "mapping chmux")
        for _ in range(sub):
            f(8), f(8, "mapping floor"), f(8, "mapping residue")
    for _ in range(f(6, "mode count") + 1):
        f(1, "mode blockflag"), f(16, "mode window"), f(16, "mode transform"), f(8, "mode mapping")
    return f.fields


def _set_bits(b, pos, n, v):
    x = int.from_bytes(bytes(b), "little")
    x = (x & ~(((1 << n) - 1) << pos)) | ((v & ((1 << n) - 1)) << pos)
    return bytearray(x.to_bytes(len(b), "little"))


def damaged_corpus(seed=20261017, n=3000):
    """[(what, [id, comment, setup])] of seeded damage on the headers of several setups, and the field names edited"""
    import vorbis_gen as G
    bases = [stock_headers(2, 44100, 0.5), stock_headers(1, 22050, 0.3), stock_headers(6, 48000, 0.2),
             stock_headers(2, 44100, -0.1)] + [generated_headers(nm) for nm in G.INSIDE[:6]]
    fields = []
    for b in bases:
        fl = {}
        for pos, nb, name in setup_fields(b[2], b[0][11]):
            fl.setdefault(name, []).append((pos, nb))
        fields.append(fl)
    rng = np.random.default_rng(seed)
    out, edited = [], set()
    for i in range(n):
        b = bases[i % len(bases)]
        h = [bytearray(x) for x in b]
        kind = rng.integers(0, 5)
        k = int(rng.choice(3, p=[0.15, 0.1, 0.75]))
        if kind == 0:                                      # truncation
            h[k] = h[k][:int(rng.integers(0, len(h[k]) + 1))]
            what = "truncate %d" % k
        elif kind == 1:                                    # bit flips
            for _ in range(int(rng.integers(1, 4))):
                j = int(rng.integers(0, len(h[k]) * 8))
                h[k][j >> 3] ^= 1 << (j & 7)
            what = "flip %d" % k
        else:                                              # a named field of the setup header set to an edge value
            fl = fields[i % len(bases)]
            name = sorted(fl)[int(rng.integers(0, len(fl)))]
            pos, nb = fl[name][int(rng.integers(0, len(fl[name])))]
            old = G.BitReader(bytes(h[2]))
            old.pos = pos
            v = old.read(nb) if nb else 0
            top = (1 << nb) - 1
            new = int(rng.choice([0, 1, top, v + 1, v - 1, int(rng.integers(0, top + 1)) if nb else 0]))
            h[2] = _set_bits(h[2], pos, nb, new)
            edited.add(name)
            what = "%s %d -> %d" % (name, v, new & top)
        out.append(("%d %s" % (i, what), [bytes(x) for x in h]))
    return out, edited


def test_seeded_damage():
    _need()
    counts = {}
    corpus, edited = damaged_corpus()
    for what, h in corpus:
        rc = check_one(h, what)
        counts[rc] = counts.get(rc, 0) + 1
    print("damage outcomes:", counts)
    want = {"book count", "book dim", "book entries", "book length", "book length count", "book maptype",
            "book q_quant", "floor class book", "floor subbook", "floor partitions", "floor partition class",
            "residue groupbook", "residue stage book", "residue partitions", "mapping floor", "mapping residue",
            "mapping submaps", "mode count", "mode mapping", "mode blockflag"}
    assert want <= edited, sorted(want - edited)
    assert counts.get(0, 0) > 20 and counts.get(EBADHEADER, 0) > 500 and counts.get(ENOTVORBIS, 0) > 20
    assert counts.get(EIMPL, 0) > 0


def test_table_caps():
    """five ordered books of 2^22 entries of length 22 (the most a dimension-1 book may state): a few bytes each,
    more than 2^24 codewords together"""
    _need()
    import vorbis_gen as G
    d = G.setup("s64_64_mono")
    d["books"] = d["books"] + [{"dim": 1, "entries": 1 << 22, "lengths": [22] * (1 << 22), "ordered": True,
                                "sparse": False, "maptype": 0}] * 5
    h = [G.ident_header(d), G.comment_header(), G.setup_header(d)]
    assert len(h[2]) < len(generated_headers("s64_64_mono")[2]) + 80          # about 13 bytes per book
    rc, why, _, _ = H.ref(*h)
    assert rc == 0 and why == 16
    assert mine(h)[0] == EIMPL


HARNESS = r"""
#include <cstdio>
#include <vector>
#include "vb200_headers.h"
int main(int argc, char **argv) {
  FILE *f = fopen(argv[1], "rb");
  long n = 0, rc_sum = 0;
  unsigned int len[3];
  while (fread(len, 4, 3, f) == 3) {
    std::vector<std::vector<uint8_t>> p(3);
    for (int k = 0; k < 3; k++) {
      p[k].resize(len[k]);
      if (len[k] && fread(p[k].data(), 1, len[k], f) != len[k]) return 2;
    }
    vb200_vorbis_headers *h = nullptr;
    // exact-size heap copies, so that a read past a packet is a sanitizer report
    std::vector<uint8_t *> c(3);
    for (int k = 0; k < 3; k++) { c[k] = new uint8_t[len[k] ? len[k] : 1]; std::copy(p[k].begin(), p[k].end(), c[k]); }
    int rc = vb200_vorbis_headers_parse(c[0], len[0], c[1], len[1], c[2], len[2], &h);
    if (rc == 0) vb200_vorbis_headers_free(h);
    for (int k = 0; k < 3; k++) delete[] c[k];
    rc_sum += rc; n++;
  }
  printf("%ld %ld\n", n, rc_sum);
  return 0;
}
"""


def test_sanitizers(tmp_path):
    _need()
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not found")
    src, exe, corpus = tmp_path / "h.cc", tmp_path / "h", tmp_path / "corpus.bin"
    src.write_text(HARNESS)
    subprocess.check_call([gxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "vorbis_b200", "csrc"),
                           str(src), "-o", str(exe)])
    cases = [h for _, h in damaged_corpus()[0]] + [stock_headers(2, 44100, 0.5)]
    with open(corpus, "wb") as f:
        for h in cases:
            f.write(np.array([len(x) for x in h], np.uint32).tobytes())
            for x in h:
                f.write(x)
    r = subprocess.run([str(exe), str(corpus)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and not r.stderr, r.stderr[-3000:]
    assert int(r.stdout.split()[0]) == len(cases)
