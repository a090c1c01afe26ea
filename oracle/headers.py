"""The reference's reading of three header packets: ctypes loader of
  oracle/_ref/libvorbis_ref_headers.so   ref_headers.c + the stock reference objects + the decode driver
                                         (vorbis_b200/host/vb200_decode.c, for vb200md_entropy_new)
oracle/Makefile builds it where the reference sources exist; like the rest of oracle/_ref it travels.  Also
`describe`, the comparable form of a (vb200_setup, vb200_entropy_setup, modebits) that both the reference's and the
product's parse are reduced to.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os

import numpy as np

from vorbis_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libvorbis_ref_headers.so")
HANGS = -1000          # rh_open: vorbis_synthesis_init would not return (maptype 1, dimension 0)
EIMPL_WHY = {1: "modes", 2: "floor0", 4: "submaps", 8: "dim", 16: "tables past the caps"}


def available():
    return os.path.exists(LIB)


_L = None


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        vp = C.c_void_p
        L.rh_open.restype = vp
        L.rh_open.argtypes = [C.c_char_p, C.c_long, C.c_char_p, C.c_long, C.c_char_p, C.c_long,
                              C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.rh_setup.restype = C.POINTER(abi.Setup)
        L.rh_setup.argtypes = [vp]
        L.rh_entropy.restype = C.POINTER(abi.EntropySetup)
        L.rh_entropy.argtypes = [vp]
        L.rh_modebits.argtypes = [vp]
        L.rh_info.argtypes = [vp, np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")]
        L.rh_close.argtypes = [vp]
        _L = L
    return _L


def ref(id_, comment, setup):
    """(rc, eimpl bits, description or None, info [channels, rate, bitrate upper, nominal, lower]) of the reference"""
    L = _lib()
    rc, why = C.c_int(0), C.c_int(0)
    h = L.rh_open(bytes(id_), len(id_), bytes(comment), len(comment), bytes(setup), len(setup), C.byref(rc),
                  C.byref(why))
    if not h:
        return rc.value, 0, None, None
    try:
        info = np.zeros(5, np.int64)
        L.rh_info(h, info)
        d = None
        if not why.value:
            d = describe(L.rh_setup(h).contents, L.rh_entropy(h).contents)
        return 0, why.value, d, info
    finally:
        L.rh_close(h)


def _arr(p, n, dt):
    if not p or n <= 0:
        return np.zeros(0, dt)
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(np.ctypeslib.as_ctypes_type(dt))), shape=(n,)).copy()


def describe(s, es):
    """a plain dict of every field vb200md_setup and vb200md_entropy_new give (abi.Setup, abi.EntropySetup); books as
    sorted lists of (entry, length, bits, value row as uint32 bytes)"""
    ch = s.channels
    d = {"channels": ch, "rate": s.rate, "blocksizes": list(s.blocksizes), "n_psy": s.n_psy,
         "modebits": es.modebits, "nbooks": es.nbooks}
    for w in range(2):
        d["window%d" % w] = _arr(C.cast(s.window[w], C.c_void_p).value, s.blocksizes[w] // 2, np.float32).view(
            np.uint32).tolist()
        n = s.coupling_steps[w]
        d["coupling%d" % w] = (n, list(s.coupling_mag[w])[:n], list(s.coupling_ang[w])[:n])
        sm = s.submaps[w]
        d["submaps%d" % w] = sm
        d["chmux%d" % w] = list(s.chmux[w])[:ch]
        d["residue_types%d" % w] = [s.residue[w][j].type for j in range(abi.MAX_SUBMAPS)]
        for j in range(sm):
            f = s.floor1[w][j]
            d["floor1_%d_%d" % (w, j)] = (f.posts, list(f.postlist)[:f.posts], f.mult, f.n, f.maxover, f.maxunder,
                                          f.maxerr, f.twofitweight, f.twofitatten)
            fd = es.floor[w][j]
            d["floor_%d_%d" % (w, j)] = (fd.type, fd.partitions, list(fd.partitionclass), list(fd.class_dim),
                                         list(fd.class_subs), list(fd.class_book),
                                         [list(r) for r in fd.class_subbook])
            r = es.residue[w][j]
            d["residue_%d_%d" % (w, j)] = (r.type, r.begin, r.end, r.grouping, r.partitions, r.partvals, r.groupbook,
                                           [list(x) for x in r.stagebook])
    books = []
    for i in range(es.nbooks):
        b = es.books[i]
        n, dim = b.used, b.dim
        ln, bits, ent = _arr(b.length, n, np.uint8), _arr(b.bits, n, np.uint32), _arr(b.entry, n, np.int32)
        val = _arr(b.value, n * dim, np.float32).view(np.uint32).reshape(n, dim) if b.value else None
        rows = sorted((int(ent[k]), int(ln[k]), int(bits[k]), val[k].tobytes() if val is not None else None)
                      for k in range(n))
        books.append((dim, n, val is not None, rows))
    d["books"] = books
    return d
