"""The reference's encoder functions on a setup read from three header packets: ctypes loader of
  oracle/_ref/libvorbis_ref_genenc.so   ref_gen_encode.c + the stock reference objects + the multi-stream encode
                                        driver (vorbis_b200/host/vb200_mapping0.c, for vb200ms_entropy_setup_build)
oracle/Makefile builds it where the reference sources exist; like the rest of oracle/_ref it travels.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os

import numpy as np

from vorbis_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libvorbis_ref_genenc.so")
FLOOR1_STRIDE = abi.FLOOR1_STRIDE
# rge_open's refusals: the preconditions under which libvorbis's encoder stays inside its own arrays
REFUSED = {1: "stage book not map type 1 or dim outside 1..8", 2: "rint(q_delta) < 1",
           4: "lattice not full and centred", 8: "dim-8 stage book with unused entries",
           16: "floor past 65 posts or wider than the block", 32: "residue past 64 partitions or past its rows",
           64: "modes / mappings / codewords"}


def available():
    return os.path.exists(LIB)


_L = None
_ip = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_lp = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
_fp = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_bp = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        vp = C.c_void_p
        L.rge_open.restype = vp
        L.rge_open.argtypes = [C.c_char_p, C.c_long, C.c_char_p, C.c_long, C.c_char_p, C.c_long, _fp, C.c_int, _ip,
                               C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.rge_close.argtypes = [vp]
        L.rge_vb200_setup.restype = C.POINTER(abi.Setup)
        L.rge_vb200_setup.argtypes = [vp]
        L.rge_entropy.restype = C.POINTER(abi.EncodeEntropySetup)
        L.rge_entropy.argtypes = [vp]
        L.rge_modebits.argtypes = [vp]
        L.rge_counts.argtypes = [vp, _lp]
        L.rge_book.argtypes = [vp, C.c_int, _lp]
        L.rge_fit.argtypes = [vp, C.c_int, C.c_int, C.c_long, _fp, _fp, _ip, _ip]
        L.rge_encode.argtypes = [vp, C.c_int, C.c_int, C.c_long, _ip, _bp, C.c_long, _lp, _ip, _ip]
        L.rge_classify.argtypes = [vp, C.c_int, C.c_long, _ip, _ip, _ip, C.c_int]
        L.rge_packets.restype = C.c_long
        L.rge_packets.argtypes = [vp, C.c_int, C.c_long, _ip, _ip, _ip, _ip, _bp, C.c_long, _lp, _lp]
        _L = L
    return _L


class SetupView:
    """a vb200_setup the reference handle holds, as lib.Context and pyoracle.Oracle take it (.c, .channels,
    .blocksize); its windows are the reference's static tables"""

    def __init__(self, s):
        self.c = abi.Setup()
        C.memmove(C.addressof(self.c), C.addressof(s), C.sizeof(self.c))
        self.channels = self.c.channels

    def blocksize(self, W):
        return int(self.c.blocksizes[W])


class Encoder:
    """rge_open on three header packets and the encoder fields the headers do not carry:
    floors [nfloors][5] = maxover, maxunder, maxerr, twofitweight, twofitatten; classmetric [nresidues][2][64].
    .refused: the RGE_* bits of the preconditions the setup breaks (0: the handle serves as the reference)."""

    def __init__(self, id_, comment, setup, floors, classmetric):
        self.L = _lib()
        ff = np.ascontiguousarray(floors, np.float32).reshape(-1, 5)
        cm = np.ascontiguousarray(classmetric, np.int32).reshape(-1, 2, 64)
        rc, why = C.c_int(0), C.c_int(0)
        self.h = self.L.rge_open(bytes(id_), len(id_), bytes(comment), len(comment), bytes(setup), len(setup), ff,
                                 ff.shape[0], cm, cm.shape[0], C.byref(rc), C.byref(why))
        if not self.h:
            raise RuntimeError("rge_open failed (%d)" % rc.value)
        self.refused = why.value
        if self.refused:
            return
        self.setup = SetupView(self.L.rge_vb200_setup(self.h).contents)
        self.channels, self.bs = self.setup.channels, [self.setup.blocksize(0), self.setup.blocksize(1)]
        self.modebits = self.L.rge_modebits(self.h)

    def entropy(self):
        """the abi.EncodeEntropySetup vb200ms_entropy_setup_build made (its arrays live in this handle)"""
        return self.L.rge_entropy(self.h).contents

    def book(self, i):
        """(dim, entries, minval, delta, quantvals) of the encoder's codebook i"""
        out = np.zeros(5, np.int64)
        self.L.rge_book(self.h, i, out)
        return tuple(int(x) for x in out)

    def counts(self):
        """{"fallback": stage-0 vectors on an unused lattice entry, "dropped": floor values written with no bits,
        "nullfit": fits that returned NULL} since the handle opened"""
        out = np.zeros(3, np.int64)
        self.L.rge_counts(self.h, out)
        return dict(zip(("fallback", "dropped", "nullfit"), (int(x) for x in out)))

    def fit(self, W, submap, logmdct, logmask):
        n = self.bs[W] // 2
        a = np.ascontiguousarray(logmdct, np.float32).reshape(-1, n)
        b = np.ascontiguousarray(logmask, np.float32).reshape(-1, n)
        posts = np.zeros((a.shape[0], FLOOR1_STRIDE), np.int32)
        nz = np.zeros(a.shape[0], np.int32)
        self.L.rge_fit(self.h, W, submap, a.shape[0], a, b, posts, nz)
        return posts, nz

    def encode(self, W, submap, posts):
        """floor1_encode on posts at the fit scale (all-zero rows: no floor): (posts it leaves, ilogmask, return
        values, packed bits as bytes per row)"""
        n = self.bs[W] // 2
        p = np.array(posts, np.int32).reshape(-1, FLOOR1_STRIDE)
        rows, cap = p.shape[0], 4096
        bits = np.zeros(rows * cap, np.uint8)
        nbits = np.zeros(rows, np.int64)
        ilog = np.zeros((rows, n), np.int32)
        ret = np.zeros(rows, np.int32)
        self.L.rge_encode(self.h, W, submap, rows, p, bits, cap, nbits, ilog, ret)
        packed = [bytes(bits[r * cap:r * cap + (int(nbits[r]) + 7) // 8]) for r in range(rows)]
        return p, ilog, ret, packed

    def classify(self, W, iwork, nonzero, stride):
        ch, n = self.channels, self.bs[W] // 2
        iw = np.ascontiguousarray(iwork, np.int32).reshape(-1, ch, n)
        nz = np.ascontiguousarray(nonzero, np.int32).reshape(-1, ch)
        classes = np.full((iw.shape[0], ch, stride), -1, np.int32)
        self.L.rge_classify(self.h, W, iw.shape[0], iw, nz, classes, stride)
        return classes

    def packets(self, W, desc, posts, nonzero, iwork):
        """the reference's packets for blocks of size W: desc [nb][2] lW, nW (or a BLOCKDESC array); posts at the
        quantised scale.  Returns (packets as bytes, the posts floor1_encode leaves)"""
        if desc.dtype.names:
            desc = np.stack([desc["lW"], desc["nW"]], 1)
        desc = np.ascontiguousarray(desc, np.int32)
        nb, ch = desc.shape[0], self.channels
        posts = np.array(posts, np.int32).reshape(nb, ch, FLOOR1_STRIDE)
        nonzero = np.ascontiguousarray(nonzero, np.int32)
        iwork = np.array(iwork, np.int32)
        cap = max(1 << 16, nb * 65536)
        out = np.zeros(cap, np.uint8)
        off, nbytes = np.zeros(nb, np.int64), np.zeros(nb, np.int64)
        if self.L.rge_packets(self.h, W, nb, desc, posts, nonzero, iwork, out, cap, off, nbytes) < 0:
            raise RuntimeError("reference packet writing failed")
        return [bytes(out[off[i]:off[i] + nbytes[i]]) for i in range(nb)], posts

    def close(self):
        if self.h:
            self.L.rge_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
