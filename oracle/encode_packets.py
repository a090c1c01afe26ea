"""Checkers of the device entropy coder: ctypes loader of
  oracle/_ref/libvorbis_ref_encpackets.so      ref_encode_packets.c + the stock reference objects: the reference's own
                                               floor1_encode and residue class / forward on given posts and residue
  oracle/_ref/libvorbis_dropin_encpackets.so   the same file + the multi-stream encode driver
                                               (vorbis_b200/host/vb200_mapping0.c) + the drop-in reference objects
oracle/Makefile builds both where the reference sources exist; like the rest of oracle/_ref they travel.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libvorbis_dropin_encpackets.so")
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref_encpackets.so")
FLOOR1_STRIDE = 65


def available():
    return os.path.exists(LIB) and os.path.exists(REF_LIB)


_L = {}
_ip = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_lp = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
_bp = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")


def _lib(dropin=False):
    if dropin not in _L:
        L = C.CDLL(LIB if dropin else REF_LIB)
        if dropin:
            L.rep_open.restype = C.c_void_p
            L.rep_open.argtypes = [C.c_int, C.c_int, C.c_long, C.c_float, C.c_int]
            L.rep_ctx.restype = C.c_void_p
            L.rep_ctx.argtypes = [C.c_void_p]
            L.rep_on_device.argtypes = [C.c_void_p]
            L.rep_close.argtypes = [C.c_void_p]
            L.rep_blocksize.argtypes = [C.c_void_p, C.c_int]
            L.rep_setup_new.restype = C.c_void_p
            L.rep_setup_new.argtypes = [C.c_void_p]
            L.rep_setup_free.argtypes = [C.c_void_p]
            L.rep_ms_encode.restype = C.c_long
            L.rep_ms_encode.argtypes = [C.c_int, C.c_int, C.c_long, C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_long,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        else:
            L.rep_ref_packets.restype = C.c_long
            L.rep_ref_packets.argtypes = [C.c_int, C.c_long, C.c_float, C.c_int, C.c_long, _ip, _ip, _ip, _ip, _bp,
                                          C.c_long, _lp, _lp, _lp]
        _L[dropin] = L
    return _L[dropin]


def ref_packets(ch, rate, q, W, desc, posts, nonzero, iwork):
    """checker (a): the reference's packets for blocks of size W given lW / nW (desc [nblocks][2] or a
    BLOCKDESC array), posts at the quantised scale, nonzero and iwork.  Returns (packets: list of bytes, the posts
    floor1_encode leaves, stage-0 lattice hits on unused entries)."""
    if desc.dtype.names:
        desc = np.stack([desc["lW"], desc["nW"]], 1)
    desc = np.ascontiguousarray(desc, np.int32)
    nb = desc.shape[0]
    posts = np.array(posts, np.int32).reshape(nb, ch, FLOOR1_STRIDE)
    nonzero = np.ascontiguousarray(nonzero, np.int32)
    iwork = np.array(iwork, np.int32)
    cap = max(1 << 16, nb * 65536)
    out = np.zeros(cap, np.uint8)
    off = np.zeros(nb, np.int64)
    nbytes = np.zeros(nb, np.int64)
    hits = np.zeros(1, np.int64)
    if _lib().rep_ref_packets(ch, rate, q, W, nb, desc, posts, nonzero, iwork, out, cap, off, nbytes, hits) < 0:
        raise RuntimeError("reference packet writing failed")
    return [bytes(out[off[i]:off[i] + nbytes[i]]) for i in range(nb)], posts, int(hits[0])


class Driver:
    """checker (b): a multi-stream encode driver vb200ms_open(ns, ch, rate, q); .ctx is a lib.Context on its device
    context, which carries the driver's entropy setup"""

    def __init__(self, ch, rate, q, ns=1, device=0):
        from vorbis_b200 import lib
        self.L = _lib(True)
        self.m = self.L.rep_open(ns, ch, rate, q, device)
        if not self.m:
            raise RuntimeError("vb200ms_open failed")
        self.on_device = bool(self.L.rep_on_device(self.m))
        self.ctx = lib.Context.wrap(self.L.rep_ctx(self.m), ch,
                                    [self.L.rep_blocksize(self.m, 0), self.L.rep_blocksize(self.m, 1)])

    def setup_copy(self):
        """(abi.EncodeEntropySetup copy, keep-alive) of the setup the driver registered, for editing"""
        from vorbis_b200 import abi
        p = self.L.rep_setup_new(self.m)
        if not p:
            raise RuntimeError("setup build failed")
        src = abi.EncodeEntropySetup.from_address(p)
        es = abi.EncodeEntropySetup()
        C.memmove(C.addressof(es), p, C.sizeof(es))
        books = (abi.EncCodebook * max(src.nbooks, 1))()
        C.memmove(books, C.cast(src.books, C.c_void_p).value, C.sizeof(abi.EncCodebook) * src.nbooks)
        es.books = C.cast(books, C.POINTER(abi.EncCodebook))
        self.L.rep_setup_free(p)
        return es, books

    def close(self):
        if self.m:
            if self.ctx is not None:
                self.ctx.h = None
            self.L.rep_close(self.m)
            self.m = None


def ms_encode(pcm, ch, rate, q, host_entropy=False, device=0):
    """checker (c): pcm [ns][ch][n] through one driver, host path forced or not: (blocks, [(count, bytes, hash)],
    the path it took: True = device)"""
    pcm = np.ascontiguousarray(pcm, np.float32)
    ns, n = pcm.shape[0], pcm.shape[2]
    hashes = (C.c_uint64 * ns)()
    nbytes = (C.c_long * ns)()
    counts = (C.c_long * ns)()
    on = C.c_int(0)
    blocks = _lib(True).rep_ms_encode(ns, ch, rate, q, device, 1 if host_entropy else 0, pcm.ctypes.data, n,
                                      C.addressof(hashes), C.addressof(nbytes), C.addressof(counts), C.addressof(on))
    if blocks < 0:
        raise RuntimeError("multi-stream encode failed (%d)" % blocks)
    return blocks, [(counts[i], nbytes[i], hashes[i]) for i in range(ns)], bool(on.value)
