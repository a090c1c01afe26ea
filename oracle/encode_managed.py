"""Checker of the managed multi-stream driver's entropy path: ctypes loader of
  oracle/_ref/libvorbis_dropin_encmanaged.so   ref_encode_managed.c + the multi-stream encode driver
                                               (vorbis_b200/host/vb200_mapping0.c) + the drop-in reference objects
oracle/Makefile builds it where the reference sources exist; like the rest of oracle/_ref it travels.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libvorbis_dropin_encmanaged.so")


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
