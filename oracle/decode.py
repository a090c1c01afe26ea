"""Decode runs for the tests and tools/decode_throughput.py: build recipes and ctypes loaders of
  oracle/_ref/libvorbis_ref_decode.so     the stock reference encoder and decoder (ref_decode_streams.c)
  oracle/_ref/libvorbis_dropin_decode.so  many decoders through the multi-stream decode driver
                                          (vorbis_b200/host/vb200_decode.c, vb200md_*)
Both link the objects oracle/Makefile compiles from the unmodified reference sources (targets `ref` and `dropin`)
and are only built where those exist; like the rest of oracle/_ref they travel.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.halfrate import DROPIN_OBJS, OBJ, PARITY, REF_OBJS, REF_SRC, _stale

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref_decode.so")
DROPIN_LIB = os.path.join(HERE, "_ref", "libvorbis_dropin_decode.so")
DRIVER = os.path.join(ROOT, "vorbis_b200", "host", "vb200_decode.c")
META = 5                       # offset, bytes, granulepos, e_o_s, packetno


def build(cc="gcc"):
    """the two libraries where oracle/Makefile's objects exist"""
    if not os.path.exists(os.path.join(REF_SRC, "lib", "mdct.c")):
        return
    inc = os.path.join(ROOT, "include")
    refinc = ["-I" + os.path.join(HERE, "shim"), "-I" + os.path.join(REF_SRC, "include"),
              "-I" + os.path.join(REF_SRC, "lib"), "-I" + inc]
    src = os.path.join(HERE, "ref_decode_streams.c")
    for lib, objs, srcs, extra, tail in (
            (REF_LIB, REF_OBJS, [src], ["-fopenmp"], ["-fopenmp", "-lm"]),
            (DROPIN_LIB, DROPIN_OBJS, [src, DRIVER], ["-DVB200_DROPIN", "-fopenmp"],
             ["-fopenmp", "-L" + os.path.join(ROOT, "vorbis_b200"), "-lvorbis_b200",
              "-Wl,-rpath,$ORIGIN/../../vorbis_b200", "-lm"])):
        paths = [os.path.join(OBJ, o) for o in objs]
        if not all(os.path.exists(p) for p in paths):
            continue
        if not _stale(lib, paths + srcs + [os.path.join(inc, "vorbis_b200.h")]):
            continue
        own = []
        for i, s in enumerate(srcs):
            obj = lib[:-3] + ".%d.o" % i
            subprocess.check_call([cc] + PARITY + ["-Wall"] + refinc + extra + ["-c", s, "-o", obj])
            own.append(obj)
        subprocess.check_call([cc, "-shared", "-Wl,-Bsymbolic", "-o", lib] + own + paths + tail)
        for obj in own:
            os.remove(obj)


def available():
    return os.path.exists(REF_LIB) and os.path.exists(DROPIN_LIB)


_libs = {}
_lp = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")


def _lib(dropin):
    if dropin not in _libs:
        L = C.CDLL(DROPIN_LIB if dropin else REF_LIB)
        L.rds_encode.restype = C.c_long
        L.rds_encode.argtypes = [C.c_int, C.c_long, C.c_float, C.c_void_p, C.c_long, C.c_void_p, C.c_long, _lp,
                                 C.c_long]
        L.rds_stock_decode.restype = C.c_long
        L.rds_stock_decode.argtypes = [C.c_void_p, _lp, _lp, C.c_long, C.c_int, C.c_void_p, C.c_long]
        L.rds_stock_decode_many.restype = C.c_long
        L.rds_stock_decode_many.argtypes = [C.c_int, C.c_void_p, _lp, _lp, _lp, _lp]
        if dropin:
            L.rds_md_run.restype = C.c_long
            L.rds_md_run.argtypes = [C.c_int, C.c_void_p, _lp, _lp, _lp, _lp, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p, C.c_long, _lp, C.c_void_p]
        _libs[dropin] = L
    return _libs[dropin]


class Packets:
    """the packets of one encoded stream: buf uint8, meta int64 [n][META] (3 headers first)"""

    def __init__(self, buf, meta):
        self.buf, self.meta = buf, meta

    @property
    def hdr(self):
        return np.ascontiguousarray(self.meta[:3])

    @property
    def audio(self):
        return np.ascontiguousarray(self.meta[3:])


def encode(ch, rate, quality, pcm):
    """the stock encoder's packets for pcm [ch][n]"""
    L = _lib(False)
    pcm = np.ascontiguousarray(pcm, np.float32)
    cap, maxn = 1 << 26, 1 << 18
    buf = np.zeros(cap, np.uint8)
    meta = np.zeros((maxn, META), np.int64)
    n = L.rds_encode(ch, rate, quality, pcm.ctypes.data, pcm.shape[1], buf.ctypes.data, cap, meta, maxn)
    if n < 0:
        raise RuntimeError("reference encode failed")
    meta = meta[:n].copy()
    end = int(meta[-1, 0] + meta[-1, 1])
    return Packets(buf[:end].copy(), meta)


def stock_decode(p, audio=None, channels=1, s16=False, cap=1 << 22):
    """the stock decoder on header packets p.hdr and audio rows (default p.audio): float [ch][n] or int16 [n][ch]"""
    L = _lib(False)
    audio = p.audio if audio is None else np.ascontiguousarray(audio, np.int64)
    out = np.zeros((cap, channels), np.int16) if s16 else np.zeros((channels, cap), np.float32)
    n = L.rds_stock_decode(p.buf.ctypes.data, p.hdr, audio, len(audio), 1 if s16 else 0, out.ctypes.data, cap)
    if n < 0:
        raise RuntimeError("reference decode failed")
    return out[:n] if s16 else out[:, :n]


def join(streams):
    """streams: (buf, audio meta rows, header meta rows) of one codec setup -> one buffer for all of them, the
    headers of the first: (buf, hdr, meta, first, npkt)"""
    bufs, metas, first, npkt, off, row = [], [], [], [], 0, 0
    for buf, audio, _ in streams:
        m = np.array(audio, np.int64).reshape(-1, META)
        m[:, 0] += off
        bufs.append(buf)
        metas.append(m)
        first.append(row)
        npkt.append(len(m))
        off += len(buf)
        row += len(m)
    return (np.concatenate(bufs), np.ascontiguousarray(streams[0][2], np.int64), np.concatenate(metas),
            np.array(first, np.int64), np.array(npkt, np.int64))


def stock_decode_many(joined):
    buf, hdr, meta, first, npkt = joined
    n = _lib(False).rds_stock_decode_many(len(first), buf.ctypes.data, hdr, meta, first, npkt)
    if n < 0:
        raise RuntimeError("reference decode failed")
    return n


def md_run(joined, sched, channels, s16=False, restart=-1, cap=1 << 21, device=0, keep=True):
    """the streams of join() through vb200md: (per-stream PCM (slot ns: the restarted stream's second run),
    stats dict)"""
    L = _lib(True)
    buf, hdr, meta, first, npkt = joined
    ns = len(first)
    sched = np.ascontiguousarray(sched, np.int32).reshape(-1, ns)
    out = None
    if keep:
        out = (np.zeros((ns + 1, cap, channels), np.int16) if s16 else np.zeros((ns + 1, channels, cap), np.float32))
    ln = np.zeros(ns + 1, np.int64)
    stats = np.zeros(6, np.float64)
    rc = L.rds_md_run(ns, buf.ctypes.data, hdr, meta, first, npkt, sched.ctypes.data, sched.shape[0], 1 if s16 else 0,
                      device, restart, None if out is None else out.ctypes.data, cap, ln, stats.ctypes.data)
    if rc < 0:
        raise RuntimeError("multi-stream decode driver failed (%d)" % rc)
    pcm = None
    if keep:
        pcm = [out[s][:ln[s]] if s16 else out[s][:, :ln[s]] for s in range(ns + 1)]
    return pcm, {"rounds": int(stats[0]), "blocks": int(stats[1]), "max_launches_per_round": int(stats[2]),
                 "launches": int(stats[3]), "device_s": float(stats[4]), "host_s": float(stats[5]),
                 "samples": ln[:ns].copy()}
