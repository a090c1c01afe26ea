"""Checkers of the device entropy decode: ctypes loader of
  oracle/_ref/libvorbis_ref_packets.so      ref_decode_packets.c + the stock reference objects: the managed
                                            encoder and the reference's staging
  oracle/_ref/libvorbis_dropin_packets.so   the same + the multi-stream decode driver
                                            (vorbis_b200/host/vb200_decode.c) + the drop-in reference objects
oracle/Makefile builds both where the reference sources exist; like the rest of oracle/_ref they travel.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import ctypes as C
import os

import numpy as np

from oracle.decode import META, Packets

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libvorbis_dropin_packets.so")
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref_packets.so")
FLOOR1_STRIDE = 65


def available():
    return os.path.exists(LIB) and os.path.exists(REF_LIB)


_L = {}
_lp = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
_ip = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_fp = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_bp = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")


def _lib(dropin=False):
    if dropin not in _L:
        L = C.CDLL(LIB if dropin else REF_LIB)
        L.rdp_encode_managed.restype = C.c_long
        L.rdp_encode_managed.argtypes = [C.c_int, C.c_long, C.c_long, C.c_long, C.c_long, C.c_void_p, C.c_long,
                                         C.c_void_p, C.c_long, _lp, C.c_long]
        L.rdp_ref_headers.restype = C.c_long
        L.rdp_ref_headers.argtypes = [_bp, _lp, _bp, _lp, _ip, C.c_long, _ip]
        L.rdp_ref_staging.restype = C.c_long
        L.rdp_ref_staging.argtypes = [_bp, _lp, _bp, _lp, _ip, C.c_long, _lp, _fp, _ip, _ip]
        if dropin:
            L.rdp_open.restype = C.c_void_p
            L.rdp_open.argtypes = [_bp, _lp, C.c_int]
            L.rdp_ctx.restype = C.c_void_p
            L.rdp_ctx.argtypes = [C.c_void_p]
            L.rdp_on_device.argtypes = [C.c_void_p]
            L.rdp_close.argtypes = [C.c_void_p]
            L.rdp_md_run.restype = C.c_long
            L.rdp_md_run.argtypes = [C.c_int, C.c_void_p, _lp, _lp, _lp, _lp, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p, C.c_long, _lp, C.c_void_p]
        _L[dropin] = L
    return _L[dropin]


def encode_managed(ch, rate, pcm, max_br=-1, nominal_br=128000, min_br=-1):
    """the stock managed encoder's packets (vorbis_encode_init) for pcm [ch][n]"""
    pcm = np.ascontiguousarray(pcm, np.float32)
    cap, maxn = 1 << 26, 1 << 18
    buf = np.zeros(cap, np.uint8)
    meta = np.zeros((maxn, META), np.int64)
    n = _lib().rdp_encode_managed(ch, rate, max_br, nominal_br, min_br, pcm.ctypes.data, pcm.shape[1],
                                  buf.ctypes.data, cap, meta, maxn)
    if n < 0:
        raise RuntimeError("reference managed encode failed")
    meta = meta[:n].copy()
    return Packets(buf[:int(meta[-1, 0] + meta[-1, 1])].copy(), meta)


def _packed(pkts):
    """list of bytes -> (data uint8, off int64, bytes int32)"""
    lens = np.array([len(p) for p in pkts], np.int32)
    off = np.zeros(len(pkts), np.int64)
    off[1:] = np.cumsum(lens)[:-1]
    data = np.frombuffer(b"".join(pkts) + b"\0", np.uint8).copy()
    return data, off, lens


def layout(W, bs, ch):
    """coef_off of packets with flags W (-1: none) packed back to back, and the total"""
    n = np.where(W < 0, 0, np.where(W == 1, bs[1], bs[0]) // 2 * ch).astype(np.int64)
    off = np.zeros(len(W), np.int64)
    off[1:] = np.cumsum(n)[:-1]
    return off, int(n.sum())


def ref_headers(p, pkts):
    data, off, lens = _packed(pkts)
    W = np.zeros(len(pkts), np.int32)
    if _lib().rdp_ref_headers(p.buf, p.hdr, data, off, lens, len(pkts), W) < 0:
        raise RuntimeError("headers do not parse")
    return W


def ref_staging(p, pkts, W, bs, ch):
    """the reference's staging of packets pkts (list of bytes) whose flags are W: (res, posts, present)"""
    data, off, lens = _packed(pkts)
    coef_off, total = layout(W, bs, ch)
    res = np.zeros(max(total, 1), np.float32)
    posts = np.zeros((len(pkts), ch, FLOOR1_STRIDE), np.int32)
    present = np.zeros((len(pkts), ch), np.int32)
    if _lib().rdp_ref_staging(p.buf, p.hdr, data, off, lens, len(pkts), coef_off, res, posts, present) < 0:
        raise RuntimeError("reference staging failed")
    return res, posts, present


class Driver:
    """a one-stream decode driver on p's headers; .ctx is a lib.Context on its device context"""

    def __init__(self, p, device=0):
        from vorbis_b200 import lib
        self.L = _lib(True)
        self.m = self.L.rdp_open(p.buf, p.hdr, device)
        if not self.m:
            raise RuntimeError("vb200md_open failed")
        self.on_device = bool(self.L.rdp_on_device(self.m))
        ident = p.buf[int(p.meta[0, 0]):int(p.meta[0, 0] + p.meta[0, 1])]
        self.channels = int(ident[11])                      # the identification header, doc/04-codec.tex
        self.bs = [1 << int(ident[28] & 15), 1 << int(ident[28] >> 4)]
        self.ctx = lib.Context.wrap(self.L.rdp_ctx(self.m), self.channels, self.bs)

    def close(self):
        if self.m:
            self.ctx.h = None
            self.L.rdp_close(self.m)
            self.m = None


class _OggPacket(C.Structure):
    _fields_ = [("packet", C.c_void_p), ("bytes", C.c_long), ("b_o_s", C.c_long), ("e_o_s", C.c_long),
                ("granulepos", C.c_int64), ("packetno", C.c_int64)]


def open_error(p, device=0):
    """what vb200md_open_err reports for p's headers: 0 (the driver opened, and is closed again) or the OV_* code"""
    L = _lib(True)
    L.vb200md_open_err.restype = C.c_void_p
    L.vb200md_open_err.argtypes = [C.c_int, C.POINTER(_OggPacket), C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.vb200md_close.argtypes = [C.c_void_p]
    hdr = (_OggPacket * 3)()
    for k in range(3):
        o, n = int(p.meta[k, 0]), int(p.meta[k, 1])
        hdr[k] = _OggPacket(p.buf.ctypes.data + o, n, 1 if k == 0 else 0, 0, 0, k)
    err = C.c_int(0)
    m = L.vb200md_open_err(1, hdr, 0, device, C.byref(err))
    if m:
        L.vb200md_close(m)
    return err.value


def dev_staging(ctx, pkts, W, bs, ch):
    """vb200_decode_entropy on the packets with W >= 0, in the layout of ref_staging"""
    data, off, lens = _packed(pkts)
    coef_off, total = layout(W, bs, ch)
    keep = np.nonzero(W >= 0)[0]
    res = np.zeros(max(total, 1), np.float32)
    posts = np.zeros((len(pkts), ch, FLOOR1_STRIDE), np.int32)
    present = np.zeros((len(pkts), ch), np.int32)
    if len(keep):
        r, po, pr = ctx.decode_entropy(W[keep], off[keep], lens[keep], data, coef_off[keep], res.size)
        res[:] = r
        posts[keep] = po
        present[keep] = pr
    return res, posts, present


def md_run(joined, sched, channels, s16=False, host_entropy=False, cap=1 << 21, device=0, keep=True):
    """oracle.decode.md_run without restart, the host entropy path forced or not: (per-stream PCM or None, stats)"""
    buf, hdr, meta, first, npkt = joined
    ns = len(first)
    sched = np.ascontiguousarray(sched, np.int32).reshape(-1, ns)
    out = None
    if keep:
        out = np.zeros((ns, cap, channels), np.int16) if s16 else np.zeros((ns, channels, cap), np.float32)
    ln = np.zeros(ns, np.int64)
    stats = np.zeros(7, np.float64)
    rc = _lib(True).rdp_md_run(ns, buf.ctypes.data, hdr, meta, first, npkt, sched.ctypes.data, sched.shape[0],
                           1 if s16 else 0, device, 1 if host_entropy else 0, None if out is None else out.ctypes.data,
                           cap, ln,
                           stats.ctypes.data)
    if rc < 0:
        raise RuntimeError("multi-stream decode driver failed (%d)" % rc)
    pcm = None if out is None else [out[s][:ln[s]] if s16 else out[s][:, :ln[s]] for s in range(ns)]
    return pcm, {"rounds": int(stats[0]), "blocks": int(stats[1]), "max_launches_per_round": int(stats[2]),
                 "launches": int(stats[3]), "device_s": float(stats[4]), "host_s": float(stats[5]),
                 "entropy_on_device": bool(stats[6]), "samples": ln.copy()}
