"""A seeded generator of legal Vorbis I streams, written from the Vorbis I specification:
identification, comment and setup headers from a random setup description, and audio packets written as an encoder
writes them (mode, window flags, floor-1 posts through the class and subclass books, residue classification words
and cascade codewords up to the last partition), plus truncated, bit-flipped and empty variants.  read_setup parses
the header bytes back independently of the description, so the tests measure what the headers really hold.

Two corpora of fixed seeds:
  INSIDE   setups the device decoder takes (two modes with block flags 0 and 1, floor 1 with postlist[1] <=
           blocksize/2, residue types 1 and 2 starting inside the block, mapping 0)
  OUTSIDE  one setup per documented limit the device decoder refuses

TEST INFRASTRUCTURE ONLY."""
import numpy as np

from oracle.decode import META, Packets

QUANT_Q = (256, 128, 86, 64)                     # floor-1 range per mult (spec 7.2.2)


def ilog(v):
    return int(v).bit_length() if v > 0 else 0


# ---- bits, LSb first (the order of oggpack_write) -------------------------------------------------------------------
class BitWriter:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def write(self, v, nbits):
        if nbits == 0:
            return
        self.acc |= (int(v) & ((1 << nbits) - 1)) << self.n
        self.n += nbits
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def bytes(self):
        return bytes(self.out) + (bytes([self.acc & 255]) if self.n else b"")

    def bits(self):
        return 8 * len(self.out) + self.n


class BitReader:
    def __init__(self, data):
        self.v = int.from_bytes(bytes(data), "little")
        self.nbits = 8 * len(data)
        self.pos = 0

    def read(self, nbits):
        if self.pos + nbits > self.nbits:
            raise ValueError("header ends early")
        r = (self.v >> self.pos) & ((1 << nbits) - 1)
        self.pos += nbits
        return r


# ---- codebooks ------------------------------------------------------------------------------------------------------
def canonical_codewords(lengths):
    """spec 3.2.1: each used entry in order takes the numerically lowest free codeword of its length (MSb first).
    Returns {entry: codeword as an int, first bit in the MSb}; raises on an overfull code."""
    free = [(0, 1 << 32)]                          # free intervals of the left-aligned 32-bit codeword space
    out = {}
    for e, L in enumerate(lengths):
        if L <= 0:
            continue
        size = 1 << (32 - L)
        for k, (a, b) in enumerate(free):
            s = -(-a // size) * size
            if s + size <= b:
                rest = [(x, y) for x, y in ((a, s), (s + size, b)) if y > x]
                free[k:k + 1] = rest
                out[e] = s >> (32 - L)
                break
        else:
            raise ValueError("overfull code")
    return out


def stream_bits(code, L):
    """a codeword (first bit in its MSb) as the value oggpack_write(value, L) puts first bit first"""
    return int("{:0{}b}".format(code, L)[::-1], 2) if L else 0


def complete_lengths(rng, n, maxlen=32, deep=0):
    """codeword lengths of a complete prefix code with n leaves (n >= 2), at most maxlen bits; deep > 0 forces one
    leaf that deep"""
    leaves = [0]
    if deep:
        while len(leaves) < n and leaves[-1] < deep:
            d = leaves.pop()
            leaves += [d + 1, d + 1]
    while len(leaves) < n:
        cand = [i for i, d in enumerate(leaves) if d < maxlen]
        i = cand[int(rng.integers(len(cand)))]
        d = leaves.pop(i)
        leaves += [d + 1, d + 1]
    leaves = np.array(leaves)
    rng.shuffle(leaves)
    return [int(x) for x in leaves]


def maptype1_quantvals(dim, entries):
    v = max(1, int(round(entries ** (1.0 / dim))))
    while v ** dim > entries:
        v -= 1
    while (v + 1) ** dim <= entries:
        v += 1
    return v


def make_book(rng, dim, entries, maptype=1, ordered=False, sparse=0.0, none_used=False, lengths=None, deep=0,
              maxlen=16):
    """a book description; lengths 0 = unused entry.  sparse: the share of unused entries"""
    if lengths is None:
        if none_used:
            lengths = [0] * entries
        elif entries == 1:
            lengths = [1]
        else:
            used = entries if not sparse else max(2, entries - int(sparse * entries))
            ls = complete_lengths(rng, used, maxlen, deep)
            lengths = ls + [0] * (entries - used)
            if sparse:
                lengths = [int(x) for x in rng.permutation(lengths)]
    ordered = ordered and all(L > 0 for L in lengths)        # the length-ordered layout has no unused entries
    if ordered:
        lengths = sorted(lengths)
    book = {"dim": dim, "entries": entries, "lengths": list(lengths), "ordered": ordered,
            "sparse": any(L == 0 for L in lengths), "maptype": maptype}
    if maptype:
        qbits = int(rng.integers(1, 9))
        nq = maptype1_quantvals(dim, entries) if maptype == 1 else entries * dim
        book.update(min=(int(rng.integers(0, 2)), int(rng.integers(1 << 18, 1 << 21)), 788 - 21 - int(rng.integers(3, 9))),
                    delta=(0, int(rng.integers(1 << 16, 1 << 21)), 788 - 21 - int(rng.integers(4, 10))),
                    qbits=qbits, seqp=int(rng.integers(0, 2)),
                    quant=[int(x) for x in rng.integers(0, 1 << qbits, nq)])
    return book


def balanced_lengths(rng, n):
    """codeword lengths of a complete prefix code with n >= 2 leaves at two adjacent depths, shuffled (fast for the
    large lattice books, where complete_lengths' random splits are slow)"""
    L = ilog(n - 1)
    ls = [L - 1] * ((1 << L) - n) + [L] * (2 * n - (1 << L))
    return [int(x) for x in rng.permutation(ls)]


def lattice_book(rng, dim, quantvals, delta, sparse=0.0):
    """a map-type-1 book on the full centred integer lattice an encoder's residue search assumes: quantvals (odd) ^ dim
    entries, minval -(quantvals >> 1) * delta, an integer delta, and each digit's value list in the order of
    local_book_besterror's index (0, -delta, +delta, -2 delta, ...), so that the decoder reads back the vector the
    encoder subtracted.  sparse: the share of entries left without a codeword"""
    entries, ze = quantvals ** dim, quantvals >> 1
    used = entries if not sparse else max(2, entries - int(sparse * entries))
    ls = balanced_lengths(rng, used) if used > 1 else [1]
    lengths = [int(x) for x in rng.permutation(ls + [0] * (entries - used))]
    quant = [ze - (m + 1) // 2 if m & 1 else ze + m // 2 for m in range(quantvals)]
    return {"dim": dim, "entries": entries, "lengths": lengths, "ordered": False, "sparse": used < entries,
            "maptype": 1, "min": (1, ze * delta, 788) if ze else (0, 0, 0), "delta": (0, delta, 788),
            "qbits": max(1, ilog(quantvals - 1)), "seqp": 0, "quant": quant}


def _float32(w, sign, mant, exp):
    w.write(mant | (exp << 21) | (sign << 31), 32)


def write_book(w, b):
    w.write(0x564342, 24)
    w.write(b["dim"], 16)
    w.write(b["entries"], 24)
    L = b["lengths"]
    w.write(1 if b["ordered"] else 0, 1)
    if b["ordered"]:
        cur = min(L)
        w.write(cur - 1, 5)
        i = 0
        while i < len(L):
            num = sum(1 for x in L if x == cur)
            w.write(num, ilog(len(L) - i))
            i += num
            cur += 1
    else:
        w.write(1 if b["sparse"] else 0, 1)
        for x in L:
            if b["sparse"]:
                w.write(1 if x else 0, 1)
                if x:
                    w.write(x - 1, 5)
            else:
                w.write(x - 1, 5)
    w.write(b["maptype"], 4)
    if b["maptype"]:
        _float32(w, *b["min"])
        _float32(w, *b["delta"])
        w.write(b["qbits"] - 1, 4)
        w.write(b["seqp"], 1)
        for q in b["quant"]:
            w.write(q, b["qbits"])


def read_book(r):
    if r.read(24) != 0x564342:
        raise ValueError("codebook sync")
    dim, entries = r.read(16), r.read(24)
    ordered = r.read(1)
    if ordered:
        cur, L = r.read(5) + 1, []
        while len(L) < entries:
            num = r.read(ilog(entries - len(L)))
            L += [cur] * num
            cur += 1
        sparse = False
    else:
        sparse = r.read(1)
        L = []
        for _ in range(entries):
            if sparse and not r.read(1):
                L.append(0)
            else:
                L.append(r.read(5) + 1)
    b = {"dim": dim, "entries": entries, "lengths": L, "ordered": bool(ordered), "sparse": any(x == 0 for x in L),
         "maptype": r.read(4)}
    if b["maptype"]:
        r.read(64)
        b["qbits"] = r.read(4) + 1
        b["seqp"] = r.read(1)
        nq = maptype1_quantvals(dim, entries) if b["maptype"] == 1 else entries * dim
        b["quant"] = [r.read(b["qbits"]) for _ in range(nq)]
    return b


class Coder:
    """codeword writer of one book: entry -> (value for BitWriter.write, length)"""

    def __init__(self, b):
        cw = canonical_codewords(b["lengths"])
        self.words = {e: (stream_bits(c, b["lengths"][e]), b["lengths"][e]) for e, c in cw.items()}
        self.used = sorted(self.words)

    def put(self, w, e):
        v, L = self.words[e]
        w.write(v, L)


# ---- headers --------------------------------------------------------------------------------------------------------
def _magic(w, kind):
    w.write(kind, 8)
    for c in b"vorbis":
        w.write(c, 8)


def ident_header(d):
    w = BitWriter()
    _magic(w, 1)
    w.write(0, 32)
    w.write(d["channels"], 8)
    w.write(d["rate"], 32)
    for _ in range(3):
        w.write(0, 32)
    w.write(ilog(d["bs"][0] - 1), 4)
    w.write(ilog(d["bs"][1] - 1), 4)
    w.write(1, 1)
    return w.bytes()


def comment_header():
    w = BitWriter()
    _magic(w, 3)
    vendor = b"vorbis_gen"
    w.write(len(vendor), 32)
    for c in vendor:
        w.write(c, 8)
    w.write(0, 32)
    w.write(1, 1)
    return w.bytes()


def setup_header(d):
    w = BitWriter()
    _magic(w, 5)
    w.write(len(d["books"]) - 1, 8)
    for b in d["books"]:
        write_book(w, b)
    w.write(0, 6)
    w.write(0, 16)                                   # one time-domain placeholder, type 0
    w.write(len(d["floors"]) - 1, 6)
    for f in d["floors"]:
        w.write(1, 16)
        w.write(len(f["pclass"]), 5)
        for c in f["pclass"]:
            w.write(c, 4)
        for c in range(max(f["pclass"], default=-1) + 1):
            w.write(f["cdim"][c] - 1, 3)
            w.write(f["csubs"][c], 2)
            if f["csubs"][c]:
                w.write(f["cbook"][c], 8)
            for k in range(1 << f["csubs"][c]):
                w.write(f["subbook"][c][k] + 1, 8)
        w.write(f["mult"] - 1, 2)
        w.write(f["rangebits"], 4)
        for x in f["xlist"]:
            w.write(x, f["rangebits"])
    w.write(len(d["residues"]) - 1, 6)
    for rs in d["residues"]:
        w.write(rs["type"], 16)
        w.write(rs["begin"], 24)
        w.write(rs["end"], 24)
        w.write(rs["grouping"] - 1, 24)
        w.write(len(rs["cascade"]) - 1, 6)
        w.write(rs["groupbook"], 8)
        for c in rs["cascade"]:
            w.write(c & 7, 3)
            w.write(1 if c > 7 else 0, 1)
            if c > 7:
                w.write(c >> 3, 5)
        for c, cas in enumerate(rs["cascade"]):
            for s in range(8):
                if cas >> s & 1:
                    w.write(rs["books"][c][s], 8)
    w.write(len(d["mappings"]) - 1, 6)
    cb = ilog(d["channels"] - 1)
    for m in d["mappings"]:
        w.write(0, 16)
        w.write(1 if m["submaps"] > 1 else 0, 1)
        if m["submaps"] > 1:
            w.write(m["submaps"] - 1, 4)
        w.write(1 if m["coupling"] else 0, 1)
        if m["coupling"]:
            w.write(len(m["coupling"]) - 1, 8)
            for a, b in m["coupling"]:
                w.write(a, cb)
                w.write(b, cb)
        w.write(0, 2)
        if m["submaps"] > 1:
            for c in m["chmux"]:
                w.write(c, 4)
        for s in range(m["submaps"]):
            w.write(0, 8)
            w.write(m["floor"][s], 8)
            w.write(m["residue"][s], 8)
    w.write(len(d["modes"]) - 1, 6)
    for bf, mp in d["modes"]:
        w.write(bf, 1)
        w.write(0, 16)
        w.write(0, 16)
        w.write(mp, 8)
    w.write(1, 1)
    return w.bytes()


def read_setup(ident, setup):
    """the headers parsed back: a description of the same shape as the generator's"""
    r = BitReader(ident)
    r.read(56 + 32)
    d = {"channels": r.read(8), "rate": r.read(32)}
    r.read(96)
    d["bs"] = (1 << r.read(4), 1 << r.read(4))
    r = BitReader(setup)
    r.read(56)
    d["books"] = [read_book(r) for _ in range(r.read(8) + 1)]
    for _ in range(r.read(6) + 1):
        r.read(16)
    d["floors"] = []
    for _ in range(r.read(6) + 1):
        if r.read(16) != 1:
            raise ValueError("floor type")
        f = {"pclass": [r.read(4) for _ in range(r.read(5))], "cdim": {}, "csubs": {}, "cbook": {}, "subbook": {}}
        for c in range(max(f["pclass"], default=-1) + 1):
            f["cdim"][c], f["csubs"][c] = r.read(3) + 1, r.read(2)
            f["cbook"][c] = r.read(8) if f["csubs"][c] else -1
            f["subbook"][c] = [r.read(8) - 1 for _ in range(1 << f["csubs"][c])]
        f["mult"], f["rangebits"] = r.read(2) + 1, r.read(4)
        f["xlist"] = [r.read(f["rangebits"]) for c in f["pclass"] for _ in range(f["cdim"][c])]
        d["floors"].append(f)
    d["residues"] = []
    for _ in range(r.read(6) + 1):
        rs = {"type": r.read(16), "begin": r.read(24), "end": r.read(24), "grouping": r.read(24) + 1}
        ncls, rs["groupbook"] = r.read(6) + 1, r.read(8)
        rs["cascade"] = []
        for _ in range(ncls):
            c = r.read(3)
            if r.read(1):
                c |= r.read(5) << 3
            rs["cascade"].append(c)
        rs["books"] = [[r.read(8) if cas >> s & 1 else -1 for s in range(8)] for cas in rs["cascade"]]
        d["residues"].append(rs)
    d["mappings"] = []
    cb = ilog(d["channels"] - 1)
    for _ in range(r.read(6) + 1):
        r.read(16)
        m = {"submaps": r.read(4) + 1 if r.read(1) else 1}
        m["coupling"] = [(r.read(cb), r.read(cb)) for _ in range(r.read(8) + 1)] if r.read(1) else []
        r.read(2)
        m["chmux"] = [r.read(4) for _ in range(d["channels"])] if m["submaps"] > 1 else [0] * d["channels"]
        m["floor"], m["residue"] = [], []
        for _ in range(m["submaps"]):
            r.read(8)
            m["floor"].append(r.read(8))
            m["residue"].append(r.read(8))
        d["mappings"].append(m)
    d["modes"] = []
    for _ in range(r.read(6) + 1):
        bf = r.read(1)
        r.read(32)
        d["modes"].append((bf, r.read(8)))
    return d


# ---- random setups --------------------------------------------------------------------------------------------------
class Gen:
    """one setup description under construction"""

    def __init__(self, seed, bs, channels, rate=44100):
        self.rng = np.random.default_rng(seed)
        self.d = {"channels": channels, "rate": rate, "bs": tuple(bs), "books": [], "floors": [], "residues": [],
                  "mappings": [], "modes": []}

    def book(self, *a, **k):
        self.d["books"].append(make_book(self.rng, *a, **k))
        return len(self.d["books"]) - 1

    def lattice(self, *a, **k):
        self.d["books"].append(lattice_book(self.rng, *a, **k))
        return len(self.d["books"]) - 1

    def floor(self, n, mult=None, partitions=None, dims=None, subs=None, minus_one=False, pclass=None):
        """a floor-1 setup over [0, n) (n a power of two): partitions of classes with the given dims and subclass
        bits (partition i of class pclass[i], default i % classes); minus_one puts a -1 subbook in every class with
        subclasses"""
        rng = self.rng
        mult = mult or int(rng.integers(1, 5))
        q = QUANT_Q[mult - 1]
        nparts = int(rng.integers(1, 6)) if partitions is None else partitions
        ncls = min(nparts, int(rng.integers(1, 4))) if dims is None else len(dims)
        dims = dims or [int(rng.integers(1, 5)) for _ in range(ncls)]
        subs = subs or [int(rng.integers(0, 4)) for _ in range(ncls)]
        pclass = pclass or [int(i % ncls) for i in range(nparts)]
        f = {"pclass": pclass, "cdim": {}, "csubs": {}, "cbook": {}, "subbook": {}, "mult": mult,
             "rangebits": ilog(n - 1)}
        for c in range(max(pclass, default=-1) + 1):
            f["cdim"][c], f["csubs"][c] = dims[c], subs[c]
            f["cbook"][c] = -1
            if subs[c]:
                f["cbook"][c] = self.book(1, min(1 << (subs[c] * dims[c]), 64), maptype=0,
                                          ordered=bool(rng.integers(0, 2)))
            sb = []
            for k in range(1 << subs[c]):
                if (minus_one and subs[c] and k == 1) or rng.random() < 0.1:
                    sb.append(-1)
                else:
                    sb.append(self.book(1, int(rng.integers(2, q + 40)), maptype=0, sparse=0.2 * rng.random()))
            f["subbook"][c] = sb
        npost = sum(dims[c] for c in pclass)
        assert npost + 1 <= n, "more posts than floor range"
        f["xlist"] = [int(x) for x in rng.choice(np.arange(1, n), npost, replace=False)]
        self.d["floors"].append(f)
        return len(self.d["floors"]) - 1

    def residue(self, type_, begin, end, grouping, classes, ppw=1, stage_books=None, cascade=None):
        rng = self.rng
        gb = self.book(ppw, classes ** ppw, maptype=0, ordered=bool(rng.integers(0, 2)))
        stage_books = stage_books or [self.book(int(rng.choice([1, 2, 3, 4, 5, 8])), int(rng.integers(2, 90)),
                                                maptype=int(rng.integers(1, 3)), sparse=0.15 * rng.integers(0, 2),
                                                ordered=bool(rng.integers(0, 2)))
                                      for _ in range(3)]
        rs = {"type": type_, "begin": begin, "end": end, "grouping": grouping, "groupbook": gb, "cascade": [],
              "books": []}
        for c in range(classes):
            cas = cascade[c % len(cascade)] if cascade else int(rng.integers(0, 8))
            rs["cascade"].append(cas)
            rs["books"].append([int(rng.choice(stage_books)) if cas >> s & 1 else -1 for s in range(8)])
        self.d["residues"].append(rs)
        return len(self.d["residues"]) - 1

    def mapping(self, floors, residues, chmux=None, coupling=()):
        m = {"submaps": len(floors), "floor": list(floors), "residue": list(residues),
             "chmux": list(chmux) if chmux is not None else [0] * self.d["channels"], "coupling": list(coupling)}
        self.d["mappings"].append(m)
        return len(self.d["mappings"]) - 1

    def simple(self, W, type_=None, submaps=1, coupling=(), **kw):
        """a floor, a residue and a mapping for block flag W with `submaps` submaps"""
        rng, ch = self.rng, self.d["channels"]
        half = self.d["bs"][W] // 2
        fl, rs = [], []
        for s in range(submaps):
            fl.append(self.floor(half, partitions=int(rng.integers(0, 4)) if half < 32 else None))
            t = type_ or int(rng.integers(1, 3))
            bundle = max(1, sum(1 for c in range(ch) if c % submaps == s))
            lim = half * (bundle if t == 2 else 1)
            g = int(rng.choice([1, 2, 3, 4, 8, 16, 32]))
            begin = int(rng.integers(0, max(1, lim // 4)))
            rs.append(self.residue(t, begin, int(rng.integers(begin, lim + 1)), g, int(rng.integers(1, 9)),
                                   ppw=int(rng.integers(1, 3))))
        return self.mapping(fl, rs, [c % submaps for c in range(ch)], coupling)

    def modes(self, m0, m1):
        self.d["modes"] = [(0, m0), (1, m1)]
        return self.d


def _coupling_chain(ch):
    return [(i, i + 1) for i in range(ch - 1)]


def _setup(name):
    """the fixed setups; each exercises something named in its comment"""
    if name == "s64_64_mono":                             # smallest block, no partitions in the floors
        g = Gen(1, (64, 64), 1)
        fa = g.floor(32, mult=1, partitions=0)
        ra = g.residue(1, 0, 32, 4, 3)
        fb = g.floor(32, mult=2, partitions=2, dims=[3], subs=[1])
        rb = g.residue(2, 2, 30, 3, 4)
        return g.modes(g.mapping([fa], [ra]), g.mapping([fb], [rb]))
    if name == "s64_128_64ch":                            # 64 channels, chained coupling, 4 submaps
        g = Gen(2, (64, 128), 64)
        m0 = g.simple(0, submaps=4, coupling=_coupling_chain(64)[:40])
        m1 = g.simple(1, submaps=4, coupling=_coupling_chain(64))
        return g.modes(m0, m1)
    if name == "s128_256_stereo_65posts":                 # 65 posts, class with 3 subclass bits and a -1 subbook
        g = Gen(3, (128, 256), 2)
        f0 = g.floor(64, mult=4, partitions=8, dims=[8, 7], subs=[3, 0], minus_one=True, pclass=[0] * 7 + [1])
        r0 = g.residue(2, 5, 128, 7, 64, ppw=1)           # 64 classes, grouping 7 does not divide 123
        f1 = g.floor(128, mult=3, partitions=8, dims=[8, 7], subs=[2, 3], minus_one=True)
        r1 = g.residue(1, 3, 128, 6, 5, ppw=2, cascade=[0b101, 0b011, 0b110, 0b100])
        return g.modes(g.mapping([f0], [r0], coupling=[(0, 1)]), g.mapping([f1], [r1], coupling=[(1, 0)]))
    if name == "s256_512_3ch":                            # 3 channels in one type-2 bundle, odd grouping
        g = Gen(4, (256, 512), 3)
        sb = [g.book(d, 40, maptype=1) for d in (3, 5, 7)]
        f0, f1 = g.floor(128), g.floor(256)
        r0 = g.residue(2, 1, 384, 5, 4, stage_books=sb, cascade=[0b1, 0b101, 0b111, 0b10])
        r1 = g.residue(2, 0, 1000, 9, 3, stage_books=sb, cascade=[0b11, 0b100, 0b1])  # end past the block
        return g.modes(g.mapping([f0], [r0], coupling=[(0, 2)]), g.mapping([f1], [r1], coupling=[(0, 2), (2, 1)]))
    if name == "s512_1024_8ch":                           # 8 channels, 3 submaps
        g = Gen(5, (512, 1024), 8)
        return g.modes(g.simple(0, submaps=3, coupling=[(0, 1), (1, 2), (5, 6)]), g.simple(1, submaps=2))
    if name == "s1024_2048_stereo_books":                 # 32-bit codewords, deep tables, single-entry and empty books
        g = Gen(6, (1024, 2048), 2)
        deep = g.book(2, 200, maptype=2, lengths=None, deep=32, maxlen=32)
        mid = g.book(1, 40, maptype=1, deep=21, maxlen=24, ordered=True)
        single = g.book(4, 1, maptype=1)
        empty = g.book(3, 9, maptype=1, none_used=True)
        sb = [deep, mid, single, empty]
        f0, f1 = g.floor(512, mult=2), g.floor(1024, mult=3)
        r0 = g.residue(1, 16, 512, 16, 4, stage_books=sb, cascade=[0b1, 0b11, 0b101, 0b1111])
        r1 = g.residue(2, 7, 2048, 24, 6, ppw=2, stage_books=sb, cascade=[0b1, 0b10, 0b100, 0b1000, 0b101, 0b11])
        return g.modes(g.mapping([f0], [r0]), g.mapping([f1], [r1], coupling=[(0, 1)]))
    if name == "s2048_4096_mono":
        g = Gen(7, (2048, 4096), 1)
        return g.modes(g.simple(0, type_=1), g.simple(1, type_=2))
    if name == "s4096_8192_stereo":
        g = Gen(8, (4096, 8192), 2)
        return g.modes(g.simple(0, coupling=[(1, 0)]), g.simple(1, type_=2, coupling=[(0, 1)]))
    if name == "s8192_8192_mono":
        g = Gen(9, (8192, 8192), 1)
        return g.modes(g.simple(0, type_=1), g.simple(1, type_=1))
    if name == "s64_8192_stereo":                        # both extremes in one stream
        g = Gen(10, (64, 8192), 2)
        return g.modes(g.simple(0, submaps=2), g.simple(1, submaps=2, coupling=[(0, 1)]))
    if name == "s128_128_3ch_4sub":                       # 4 submaps on 3 channels (one submap unused)
        g = Gen(11, (128, 128), 3)
        m0 = g.simple(0, submaps=4)
        m1 = g.simple(1, submaps=3, coupling=[(2, 0), (0, 1)])
        return g.modes(m0, m1)
    raise KeyError(name)


INSIDE = ["s64_64_mono", "s64_128_64ch", "s128_256_stereo_65posts", "s256_512_3ch", "s512_1024_8ch",
          "s1024_2048_stereo_books", "s2048_4096_mono", "s4096_8192_stereo", "s8192_8192_mono", "s64_8192_stereo",
          "s128_128_3ch_4sub"]

# limit -> how the device side refuses it: "context" (the driver cannot open: no device context for the setup) or
# "entropy" (the context refuses the entropy setup: the driver keeps the host path)
OUTSIDE = {"floor_wider_than_block": "context", "one_mode": "context", "three_modes": "context",
           "modes_swapped": "context", "residue_type0": "entropy", "residue_past_block": "entropy"}


def _outside(name):
    g = Gen(100 + sorted(OUTSIDE).index(name), (256, 2048), 2)
    if name == "floor_wider_than_block":                 # the short mode's floor spans 512 lines of a 128-line half
        f0, f1 = g.floor(512), g.floor(1024)
        r0, r1 = g.residue(1, 0, 128, 8, 3), g.residue(2, 0, 2048, 16, 3)
        return g.modes(g.mapping([f0], [r0]), g.mapping([f1], [r1]))
    m0, m1 = g.simple(0), g.simple(1)
    if name == "one_mode":
        g.d["modes"] = [(1, m1)]
    elif name == "three_modes":
        g.d["modes"] = [(0, m0), (1, m1), (1, m1)]
    elif name == "modes_swapped":
        g.d["modes"] = [(1, m1), (0, m0)]
    else:
        g.modes(m0, m1)
        rs = g.d["residues"][g.d["mappings"][m0]["residue"][0]]
        if name == "residue_type0":
            rs["type"] = 0
        else:                                            # begins past the short block's 128 lines
            rs["type"], rs["begin"], rs["end"] = 1, 200, 300
    return g.d


def setup(name):
    return _outside(name) if name in OUTSIDE else _setup(name)


# ---- audio packets --------------------------------------------------------------------------------------------------
class Encoder:
    """structured audio packets of one setup description"""

    def __init__(self, d):
        self.d = d
        self.coders = [Coder(b) for b in d["books"]]
        self.modebits = ilog(len(d["modes"]) - 1)
        # the walk's own count: residue stages walked, those that wrote up to the last partition, and packets whose
        # every stage did (and that had a stage to walk)
        self.stages = self.stages_to_end = self.packets_to_end = 0

    def _entry(self, rng, b, below=None):
        used = self.coders[b].used
        if below is not None:
            used = [e for e in used if e < below]
        return int(used[int(rng.integers(len(used)))])

    def _floor(self, w, rng, f):
        q = QUANT_Q[f["mult"] - 1]
        w.write(1, 1)
        w.write(int(rng.integers(q)), ilog(q - 1))
        w.write(int(rng.integers(q)), ilog(q - 1))
        for c in f["pclass"]:
            cdim, bits = f["cdim"][c], f["csubs"][c]
            cval = 0
            if bits:
                cval = self._entry(rng, f["cbook"][c])
                self.coders[f["cbook"][c]].put(w, cval)
            for _ in range(cdim):
                book = f["subbook"][c][cval & ((1 << bits) - 1)]
                cval >>= bits
                if book >= 0:                            # values below the range keep every post inside it
                    self.coders[book].put(w, self._entry(rng, book, q))

    def _vectors(self, w, rng, book, nvals):
        dim = self.d["books"][book]["dim"]
        if not self.coders[book].used:
            return
        for _ in range(-(-nvals // dim)):
            self.coders[book].put(w, self._entry(rng, book))

    def _residue(self, w, rng, rs, rows, half):
        two = rs["type"] == 2
        lim = half * len(rows) if two else half
        end = min(rs["end"], lim)
        n = end - rs["begin"]
        if n <= 0 or not rows:
            return True
        g, P = rs["grouping"], len(rs["cascade"])
        parts, ppw = n // g, self.d["books"][rs["groupbook"]]["dim"]
        per = 1 if two else len(rows)
        cls = np.zeros((per, max(parts, 1)), np.int64)
        stages = max((ilog(c) for c in rs["cascade"]), default=0)
        for s in range(stages):
            i = 0
            while i < parts:
                if s == 0:
                    for j in range(per):
                        digits = [int(rng.integers(P)) for _ in range(ppw)]
                        temp = 0
                        for k in range(ppw):
                            temp = temp * P + digits[k]
                            if i + k < parts:
                                cls[j, i + k] = digits[k]
                        self.coders[rs["groupbook"]].put(w, temp)
                for _ in range(ppw):
                    if i >= parts:
                        break
                    for j in range(per):
                        book = rs["books"][cls[j, i]][s]
                        if book < 0:
                            continue
                        if two:
                            off, ch = i * g + rs["begin"], len(rows)
                            self._vectors(w, rng, book, ((off + g) // ch - off // ch) * ch)
                        else:
                            self._vectors(w, rng, book, g)
                    i += 1
            self.stages += 1
            self.stages_to_end += i == parts
        return parts == 0 or stages == 0 or i == parts

    def packet(self, rng, mode, lW, nW):
        d = self.d
        w = BitWriter()
        w.write(0, 1)
        w.write(mode, self.modebits)
        bf, mp = d["modes"][mode]
        if bf:
            w.write(lW, 1)
            w.write(nW, 1)
        m = d["mappings"][mp]
        ch = d["channels"]
        nz = [bool(rng.random() < 0.85) for _ in range(ch)]
        for c in range(ch):
            f = d["floors"][m["floor"][m["chmux"][c]]]
            if nz[c]:
                self._floor(w, rng, f)
            else:
                w.write(0, 1)
        for a, b in m["coupling"]:
            if nz[a] or nz[b]:
                nz[a] = nz[b] = True
        half = d["bs"][bf] // 2
        walked, ok = self.stages, True
        for s in range(m["submaps"]):
            rs = d["residues"][m["residue"][s]]
            bundle = [c for c in range(ch) if m["chmux"][c] == s]
            if rs["type"] == 2:
                rows = bundle if any(nz[c] for c in bundle) else []
            else:
                rows = [c for c in bundle if nz[c]]
            ok &= self._residue(w, rng, rs, rows, half)
        self.packets_to_end += ok and self.stages > walked
        return w.bytes()


def packets(d, seed, n):
    """n structured audio packets of a two-mode setup with a random block-flag sequence (consistent window flags)"""
    rng = np.random.default_rng(seed)
    enc = Encoder(d)
    modes = d["modes"]
    flags = [int(x) for x in rng.integers(0, 2, n)]
    out = []
    for k in range(n):
        mode = next(i for i, (bf, _) in enumerate(modes) if bf == flags[k]) if len(modes) > 1 else 0
        bf = modes[mode][0]
        lW = flags[k - 1] if k else 0
        nW = flags[k + 1] if k + 1 < n else bf
        out.append(enc.packet(rng, mode, lW, nW))
    return out, enc


def damaged(pkts, seed, header_bits):
    """cuts at random byte lengths, random bit flips after the header bits, and empty packets"""
    rng = np.random.default_rng(seed)
    out = []
    for p in pkts:
        if len(p) > 1:
            out.append(p[:int(rng.integers(1, len(p)))])
        a = bytearray(p)
        nb = 8 * len(a)
        if nb > header_bits:
            for bit in rng.integers(header_bits, nb, int(rng.integers(1, 6))):
                a[bit >> 3] ^= 1 << (bit & 7)
            out.append(bytes(a))
    out.append(b"")
    return out


def stream(d, audio, page_final=False, granule=True):
    """Packets of the three headers and the audio packets: granulepos the finished sample count (on every packet, or
    on every fourth and the last as Ogg pages carry it, or on none), the last packet ending 3 samples early, e_o_s on
    it"""
    hdr = [ident_header(d), comment_header(), setup_header(d)]
    allp = hdr + list(audio)
    meta = np.zeros((len(allp), META), np.int64)
    off = 0
    bs = d["bs"]
    total, prev = 0, None
    for k, p in enumerate(allp):
        meta[k, 0], meta[k, 1], meta[k, 4] = off, len(p), k
        off += len(p)
        meta[k, 2] = 0 if k < 3 else -1
        if k >= 3:
            W = _flag(d, p)
            if W is not None:
                if prev is not None:
                    total += bs[prev] // 4 + bs[W] // 4
                prev = W
            last = k == len(allp) - 1
            if granule and (not page_final or last or (k - 3) % 4 == 3):
                meta[k, 2] = max(total - 3, 0) if last else total
            meta[k, 3] = 1 if last else 0
    return Packets(np.frombuffer(b"".join(allp) + b"\0", np.uint8).copy(), meta)


def _flag(d, p):
    """the block flag of a parsable audio packet, else None"""
    if not p:
        return None
    r = BitReader(p)
    try:
        if r.read(1):
            return None
        mode = r.read(ilog(len(d["modes"]) - 1))
        if mode >= len(d["modes"]):
            return None
        bf = d["modes"][mode][0]
        if bf:
            r.read(2)
        return bf
    except ValueError:
        return None


def header_bits(d):
    return 1 + ilog(len(d["modes"]) - 1) + 2
