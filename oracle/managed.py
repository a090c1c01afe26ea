"""Bitrate-managed encoder runs for the tests: build recipes and ctypes loaders of
  oracle/_ref/libvorbis_ref_managed.so     the stock reference encoder from vorbis_encode_init (ref_managed.c)
  oracle/_ref/libvorbis_dropin_managed.so  N such encoders through the managed multi-stream driver
                                           (vorbis_b200/host/vb200_mapping0.c, vb200ms_open_managed)
Both link the objects oracle/Makefile compiles from the unmodified reference sources (targets `ref` and `dropin`)
and are only built where those exist; like the rest of oracle/_ref they travel.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.halfrate import DROPIN_OBJS, OBJ, PARITY, REF_OBJS, REF_SRC, _stale

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref_managed.so")
DROPIN_LIB = os.path.join(HERE, "_ref", "libvorbis_dropin_managed.so")


def build(cc="gcc"):
    """the two libraries where oracle/Makefile's objects exist"""
    if not os.path.exists(os.path.join(REF_SRC, "lib", "mdct.c")):
        return
    inc = os.path.join(os.path.dirname(HERE), "include")
    refinc = ["-I" + os.path.join(HERE, "shim"), "-I" + os.path.join(REF_SRC, "include"),
              "-I" + os.path.join(REF_SRC, "lib"), "-I" + inc]
    src = os.path.join(HERE, "ref_managed.c")
    for lib, objs, extra, tail in (
            (REF_LIB, REF_OBJS, [], ["-lm"]),
            (DROPIN_LIB, DROPIN_OBJS, ["-DVB200_DROPIN"],
             ["-fopenmp", "-L" + os.path.join(os.path.dirname(HERE), "vorbis_b200"), "-lvorbis_b200",
              "-Wl,-rpath,$ORIGIN/../../vorbis_b200", "-lm"])):
        paths = [os.path.join(OBJ, o) for o in objs]
        if not all(os.path.exists(p) for p in paths):
            continue
        if not _stale(lib, paths + [src]):
            continue
        obj = lib[:-3] + ".o"
        subprocess.check_call([cc] + PARITY + ["-Wall"] + refinc + extra + ["-c", src, "-o", obj])
        subprocess.check_call([cc, "-shared", "-Wl,-Bsymbolic", "-o", lib, obj] + paths + tail)
        os.remove(obj)


def available():
    return os.path.exists(REF_LIB) and os.path.exists(DROPIN_LIB)


_libs = {}


def _lib(dropin):
    if dropin not in _libs:
        L = C.CDLL(DROPIN_LIB if dropin else REF_LIB)
        L.ref_managed_stock_summary.restype = C.c_long
        L.ref_managed_stock_summary.argtypes = [C.c_int, C.c_long, C.c_long, C.c_long, C.c_long, C.c_void_p, C.c_long,
                                                C.c_void_p, C.c_void_p, C.c_void_p]
        if dropin:
            L.ref_ms_encode_managed.restype = C.c_long
            L.ref_ms_encode_managed.argtypes = [C.c_int, C.c_int, C.c_long, C.c_long, C.c_long, C.c_long, C.c_int,
                                                C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p]
        _libs[dropin] = L
    return _libs[dropin]


def stock_summary(ch, rate, max_br, nominal_br, min_br, pcm):
    """one stock managed encoder on pcm [ch][n]: (blocks, count, bytes, hash)"""
    L = _lib(False)
    pcm = np.ascontiguousarray(pcm, np.float32)
    h, b, c = C.c_uint64(0), C.c_long(0), C.c_long(0)
    nb = L.ref_managed_stock_summary(ch, rate, max_br, nominal_br, min_br, pcm.ctypes.data, pcm.shape[1],
                                     C.byref(h), C.byref(b), C.byref(c))
    if nb < 0:
        raise RuntimeError("stock managed encoder failed")
    return nb, c.value, b.value, h.value


def ms_encode(ch, rate, max_br, nominal_br, min_br, pcm, device=0):
    """pcm [nstreams][ch][n] through the managed multi-stream driver: (blocks, rounds, launches, per-stream
    (count, bytes, hash))"""
    L = _lib(True)
    pcm = np.ascontiguousarray(pcm, np.float32)
    ns = pcm.shape[0]
    hashes, nbytes, counts = (C.c_uint64 * ns)(), (C.c_long * ns)(), (C.c_long * ns)()
    rounds, launches = C.c_long(0), C.c_uint64(0)
    nb = L.ref_ms_encode_managed(ns, ch, rate, max_br, nominal_br, min_br, device, pcm.ctypes.data, pcm.shape[2],
                                 hashes, nbytes, counts, C.byref(rounds), C.byref(launches))
    if nb < 0:
        raise RuntimeError("managed multi-stream driver failed")
    return nb, rounds.value, launches.value, [(counts[i], nbytes[i], hashes[i]) for i in range(ns)]
