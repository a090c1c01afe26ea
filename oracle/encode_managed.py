"""Checker of the managed multi-stream driver's entropy path: build recipe and ctypes loader of
  oracle/_ref/libvorbis_dropin_encmanaged.so   ref_encode_managed.c + the multi-stream encode driver
                                               (vorbis_b200/host/vb200_mapping0.c) + the drop-in reference objects
Built only where oracle/Makefile's objects exist; like the rest of oracle/_ref it travels.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.halfrate import DROPIN_OBJS, OBJ, PARITY, REF_SRC, _stale

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_ref", "libvorbis_dropin_encmanaged.so")


def build(cc="gcc"):
    if not os.path.exists(os.path.join(REF_SRC, "lib", "mdct.c")):
        return
    inc = os.path.join(ROOT, "include")
    refinc = ["-I" + os.path.join(HERE, "shim"), "-I" + os.path.join(REF_SRC, "include"),
              "-I" + os.path.join(REF_SRC, "lib"), "-I" + inc]
    src = os.path.join(HERE, "ref_encode_managed.c")
    paths = [os.path.join(OBJ, o) for o in DROPIN_OBJS]
    if not all(os.path.exists(p) for p in paths) or not _stale(LIB, paths + [src]):
        return
    obj = LIB[:-3] + ".o"
    subprocess.check_call([cc] + PARITY + ["-Wall"] + refinc + ["-DVB200_DROPIN", "-c", src, "-o", obj])
    subprocess.check_call([cc, "-shared", "-Wl,-Bsymbolic", "-o", LIB, obj] + paths +
                          ["-fopenmp", "-L" + os.path.join(ROOT, "vorbis_b200"), "-lvorbis_b200",
                           "-Wl,-rpath,$ORIGIN/../../vorbis_b200", "-lm"])
    os.remove(obj)


def available():
    return os.path.exists(LIB)


_L = []


def _lib():
    if not _L:
        L = C.CDLL(LIB)
        L.rep_ms_encode_managed.restype = C.c_long
        L.rep_ms_encode_managed.argtypes = [C.c_int, C.c_int, C.c_long, C.c_long, C.c_long, C.c_long, C.c_int, C.c_int,
                                            C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p]
        _L.append(L)
    return _L[0]


def ms_encode(ch, rate, max_br, nominal_br, min_br, pcm, host_entropy=None, device=0):
    """pcm [nstreams][ch][n] through the managed multi-stream driver, the host entropy path forced (host_entropy
    True) or as the driver chooses it (None / False): (blocks, rounds, launches, per-stream (count, bytes, hash), the
    path it took: True = device)"""
    pcm = np.ascontiguousarray(pcm, np.float32)
    ns = pcm.shape[0]
    hashes, nbytes, counts = (C.c_uint64 * ns)(), (C.c_long * ns)(), (C.c_long * ns)()
    rounds, launches, on = C.c_long(0), C.c_uint64(0), C.c_int(0)
    nb = _lib().rep_ms_encode_managed(ns, ch, rate, max_br, nominal_br, min_br, device, 1 if host_entropy else 0,
                                      pcm.ctypes.data, pcm.shape[2], hashes, nbytes, counts, C.byref(rounds),
                                      C.byref(launches), C.byref(on))
    if nb < 0:
        raise RuntimeError("managed multi-stream driver failed")
    return nb, rounds.value, launches.value, [(counts[i], nbytes[i], hashes[i]) for i in range(ns)], bool(on.value)
