"""The LPC extrapolation of vorbis_analysis_wrote for the tests: ctypes loaders of
  oracle/libvb_oracle_lpc.so   vb_oracle_lpc.c: the plain-C restatement of the filter fit and the predictor
  oracle/_ref/libvorbis_ref.so the reference's own vorbis_lpc_from_data / vorbis_lpc_predict (compiled unmodified by
                               oracle/Makefile, lpc is in REFSRC; built only where the reference sources exist)
and timeline(), which builds the v->pcm a stock encoder sees from its input and write schedule: the preamble from the
write that crossed blocksizes[1] samples, the input, and the tail from the drained planner's base at the end write,
which the carried planner of oracle/resume.py supplies.  oracle/Makefile builds both libraries.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_LIB = os.path.join(HERE, "libvb_oracle_lpc.so")
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref.so")
PRE, TAIL = 16, 32

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")


_libs = {}


def _oracle():
    if "o" not in _libs:
        L = C.CDLL(ORACLE_LIB)
        L.vbo_lpc_filter.argtypes = [f32p, C.c_long, C.c_int, f32p]
        L.vbo_lpc_run.argtypes = [f32p, f32p, C.c_int, f32p, C.c_long]
        _libs["o"] = L
    return _libs["o"]


def ref_available():
    return os.path.exists(REF_LIB)


def _ref():
    if "r" not in _libs:
        L = C.CDLL(REF_LIB)
        L.vorbis_lpc_from_data.argtypes = [f32p, f32p, C.c_int, C.c_int]
        L.vorbis_lpc_from_data.restype = C.c_float
        L.vorbis_lpc_predict.argtypes = [f32p, f32p, C.c_int, f32p, C.c_long]
        _libs["r"] = L
    return _libs["r"]


def extrapolate(x, m, count):
    """the oracle: (coefficients [m], count samples continuing x) for the window x"""
    x = np.ascontiguousarray(x, np.float32)
    coef = np.zeros(m, np.float32)
    _oracle().vbo_lpc_filter(x, len(x), m, coef)
    out = np.zeros(max(count, 1), np.float32)
    _oracle().vbo_lpc_run(coef, np.ascontiguousarray(x[len(x) - m:]), m, out, count)
    return coef, out[:count]


def ref_extrapolate(x, m, count):
    """the reference's vorbis_lpc_from_data then vorbis_lpc_predict, as vorbis_analysis_wrote calls them"""
    x = np.ascontiguousarray(x, np.float32).copy()
    coef = np.zeros(m, np.float32)
    _ref().vorbis_lpc_from_data(x, coef, len(x), m)
    out = np.zeros(max(count, 1), np.float32)
    _ref().vorbis_lpc_predict(coef, np.ascontiguousarray(x[len(x) - m:]), m, out, count)
    return coef, out[:count]


def crossing(writes, bs1):
    """P: the samples written when the preamble is made (the first write after which more than blocksizes[1] have been
    written), or None when the end write makes it"""
    total = 0
    for w in writes:
        total += int(w)
        if w > 0 and total > bs1:
            return total
    return None


def drained_base(ora, bs, tl, P):
    """the base of a stock encoder drained on the timeline tl (without eof) once its preamble exists: the carried
    planner fed the whole timeline; 0 when the end write makes the preamble (nothing was planned before)"""
    from oracle import resume as R
    if P is None:
        return 0
    pl = R.Planner(bs, tl.shape[0])
    while True:
        base = pl.c.base
        if not len(pl.feed(ora, tl[:, base:], tl.shape[1] - base, 0, 4096)):
            return base


def timeline(ora, bs, pcm, writes):
    """the stock encoder's timeline [ch][bs1/2 + n + 3*bs1] and eof for input pcm [ch][n] written in the given
    pieces (summing to n) then vorbis_analysis_wrote(v, 0)"""
    ch, n = pcm.shape
    half = bs[1] // 2
    tl = np.zeros((ch, half + n + 3 * bs[1]), np.float32)
    tl[:, half:half + n] = pcm
    P = crossing(writes, bs[1])
    p = n if P is None else P
    if p > 2 * PRE:
        for c in range(ch):
            _, pre = extrapolate(pcm[c, :p][::-1], PRE, half)
            tl[c, :half] = pre[::-1]
    eof = half + n
    base = drained_base(ora, bs, tl[:, :eof], P)
    if eof - base > 2 * TAIL:
        w = min(eof - base, bs[1])
        for c in range(ch):
            _, tail = extrapolate(tl[c, eof - w:eof], TAIL, 3 * bs[1])
            tl[c, eof:] = tail
    return tl, eof
