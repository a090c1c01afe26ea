"""Checkers of vb200_decode_streams_packets: ctypes loaders of
  oracle/libvb_oracle_decode_streams.so   the plain-C restatement of its per-stream plan (vb_oracle_decode_streams.c);
                                          builds anywhere gcc exists
  oracle/_ref/libvorbis_ref_plan.so       ref_decode_plan.c + the stock reference objects: the stock decoder's PCM and
                                          its state after every vorbis_synthesis_blockin, at full and half rate
oracle/Makefile builds both; the second only where the reference sources exist, and like the rest of oracle/_ref it
travels.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.decode import META

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_LIB = os.path.join(HERE, "libvb_oracle_decode_streams.so")
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref_plan.so")
REF_REC = 8                    # status, W, samples, granulepos, pcm_returned, pcm_current, sequence, sample_count
ORACLE_REC = 11                # the same, then lo, hi, fin
STATE_WORDS = 6                # sizeof(vbo_ds_state) / 8


def ref_available():
    return os.path.exists(REF_LIB)


_L = {}
_lp = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")


def _lib(ref):
    if ref not in _L:
        if ref:
            L = C.CDLL(REF_LIB)
            L.rdsp_decode.restype = C.c_long
            L.rdsp_decode.argtypes = [C.c_void_p, _lp, _lp, C.c_long, C.c_int, C.c_void_p, C.c_long, _lp,
                                      C.POINTER(C.c_int)]
        else:
            subprocess.check_call(["make", "-s", "-C", HERE, os.path.basename(ORACLE_LIB), "CC=gcc"])
            L = C.CDLL(ORACLE_LIB)
            L.vbo_ds_init.argtypes = [_lp, C.c_void_p, C.c_int]
            L.vbo_ds_run.argtypes = [_lp, C.c_void_p, _lp, C.c_long, C.c_int, C.c_void_p, C.c_int, _lp]
            L.vbo_ds_init.restype = L.vbo_ds_run.restype = None
        _L[ref] = L
    return _L[ref]


def ref_decode(buf, hdr, audio, channels, halfrate=False, cap=1 << 21):
    """the stock decoder on header rows hdr and audio rows (meta int64 [n][5] into buf): (pcm float [ch][n],
    rec int64 [npkt][REF_REC], modebits)"""
    buf = np.ascontiguousarray(buf, np.uint8)
    audio = np.ascontiguousarray(audio, np.int64).reshape(-1, META)
    out = np.zeros((channels, cap), np.float32)
    rec = np.zeros((max(len(audio), 1), REF_REC), np.int64)
    mb = C.c_int(0)
    n = _lib(True).rdsp_decode(buf.ctypes.data, np.ascontiguousarray(hdr, np.int64), audio, len(audio),
                               1 if halfrate else 0, out.ctypes.data, cap, rec, C.byref(mb))
    if n < 0 or n > cap:
        raise RuntimeError("reference decode failed")
    return out[:, :n], rec[:len(audio)], mb.value


class Plan:
    """the oracle's state of one stream, carried from run to run"""

    def __init__(self, bs, modebits, halfrate=False):
        self.bs = np.array(bs, np.int32)
        self.modebits, self.hs = modebits, 1 if halfrate else 0
        self.state = np.zeros(STATE_WORDS, np.int64)
        self.restart()

    def restart(self):
        _lib(False).vbo_ds_init(self.state, self.bs.ctypes.data, self.hs)

    def run(self, buf, audio):
        """audio meta rows into buf -> rec int64 [npkt][ORACLE_REC]"""
        buf = np.ascontiguousarray(buf, np.uint8)
        audio = np.ascontiguousarray(audio, np.int64).reshape(-1, META)
        rec = np.zeros((max(len(audio), 1), ORACLE_REC), np.int64)
        _lib(False).vbo_ds_run(self.state, buf.ctypes.data, audio, len(audio), self.modebits, self.bs.ctypes.data,
                               self.hs, rec)
        return rec[:len(audio)]


def s16_of(pcm):
    """examples/decoder_example.c:250-262 on float [ch][n] -> int16 [n][ch]"""
    v = np.floor(pcm.astype(np.float32) * np.float32(32767.0) + np.float32(0.5)).astype(np.int64)
    return np.clip(v, -32768, 32767).astype(np.int16).T.copy()
