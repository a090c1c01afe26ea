"""The bitrate manager and whole streams' packets for the tests: build recipes and ctypes loaders of
  oracle/libvb_oracle_bitrate.so             the CPU oracle's restatement of vorbis_bitrate_addblock
                                             (vb_oracle_bitrate.c); builds anywhere gcc exists
  oracle/_ref/libvorbis_ref_bitrate.so       ref_bitrate.c + the stock reference objects: ref_bitrate_info,
                                             ref_bitrate_replay and ref_stream_capture
  oracle/_ref/libvorbis_dropin_bitrate.so    the same file + the managed multi-stream driver: a device context with
                                             the setup and entropy setup of a managed encoder
The two reference libraries link the objects oracle/Makefile compiles from the unmodified reference sources and are
only built where those exist; like the rest of oracle/_ref they travel.

TEST INFRASTRUCTURE ONLY: imported by tests/, tools/ and tests/golden/make_golden_bitrate.py, never by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.halfrate import DROPIN_OBJS, OBJ, PARITY, REF_OBJS, REF_SRC, _stale
from vorbis_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ORACLE_LIB = os.path.join(HERE, "libvb_oracle_bitrate.so")
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref_bitrate.so")
DROPIN_LIB = os.path.join(HERE, "_ref", "libvorbis_dropin_bitrate.so")
NB = abi.PACKETBLOBS
BRANCHES = ("slew down", "slew up", "min loop", "max loop", "truncation", "padding")


def build(cc="gcc"):
    """the oracle library always; the two reference libraries where oracle/Makefile's objects exist"""
    inc = os.path.join(ROOT, "include")
    osrc = os.path.join(HERE, "vb_oracle_bitrate.c")
    if _stale(ORACLE_LIB, [osrc, os.path.join(inc, "vorbis_b200.h")]):
        subprocess.check_call([cc] + PARITY + ["-std=gnu99", "-Wall", "-I" + inc, "-shared", "-o", ORACLE_LIB, osrc,
                                               "-lm"])
    if not os.path.exists(os.path.join(REF_SRC, "lib", "mdct.c")):
        return
    refinc = ["-I" + os.path.join(HERE, "shim"), "-I" + os.path.join(REF_SRC, "include"),
              "-I" + os.path.join(REF_SRC, "lib"), "-I" + inc]
    src = os.path.join(HERE, "ref_bitrate.c")
    for lib, objs, extra, tail in (
            (REF_LIB, REF_OBJS, [], ["-lm"]),
            (DROPIN_LIB, DROPIN_OBJS, ["-DVB200_DROPIN"],
             ["-fopenmp", "-L" + os.path.join(ROOT, "vorbis_b200"), "-lvorbis_b200",
              "-Wl,-rpath,$ORIGIN/../../vorbis_b200", "-lm"])):
        paths = [os.path.join(OBJ, o) for o in objs]
        if not all(os.path.exists(p) for p in paths):
            continue
        if not _stale(lib, paths + [src, os.path.join(inc, "vorbis_b200.h")]):
            continue
        obj = lib[:-3] + ".o"
        subprocess.check_call([cc] + PARITY + ["-Wall"] + refinc + extra + ["-c", src, "-o", obj])
        subprocess.check_call([cc, "-shared", "-Wl,-Bsymbolic", "-o", lib, obj] + paths + tail)
        os.remove(obj)


def ref_available(dropin=False):
    return os.path.exists(DROPIN_LIB if dropin else REF_LIB)


class Config(C.Structure):
    """rbr_config of ref_bitrate.c: how a stock encoder is opened"""
    _fields_ = [("mode", C.c_int32), ("channels", C.c_int32), ("rate", C.c_int64), ("quality", C.c_double),
                ("max_br", C.c_int64), ("nominal_br", C.c_int64), ("min_br", C.c_int64), ("rm2", C.c_int32),
                ("pad", C.c_int32), ("rm2_reservoir_bits", C.c_int64), ("rm2_bias", C.c_double),
                ("rm2_damp", C.c_double)]


def vbr(ch, rate, q):
    return Config(mode=0, channels=ch, rate=rate, quality=q)


def managed(ch, rate, max_br=-1, nominal_br=-1, min_br=-1, reservoir_bits=None, bias=None, damp=None):
    """vorbis_encode_init(ch, rate, max, nominal, min); given reservoir_bits, the reservoir bits, bias and average
    damping replaced through OV_ECTL_RATEMANAGE2_SET before vorbis_encode_setup_init"""
    cf = Config(mode=1, channels=ch, rate=rate, max_br=max_br, nominal_br=nominal_br, min_br=min_br)
    if reservoir_bits is not None:
        cf.rm2, cf.rm2_reservoir_bits, cf.rm2_bias, cf.rm2_damp = 1, reservoir_bits, bias, damp
    return cf


def config_array(cf):
    """a Config as a plain int64/float64 record for the fixture"""
    return np.array([cf.mode, cf.channels, cf.rate, cf.quality, cf.max_br, cf.nominal_br, cf.min_br, cf.rm2,
                     cf.rm2_reservoir_bits, cf.rm2_bias, cf.rm2_damp], np.float64)


# the configurations the tests replay: ABR (nominal only), CBR, max only, min only, and CBR with a small reservoir,
# another bias and another damping through OV_ECTL_RATEMANAGE2_SET (reaches truncation and padding)
CONFIGS = {
    "abr": managed(2, 44100, nominal_br=128000),
    "cbr": managed(2, 44100, 128000, 128000, 128000),
    "max": managed(2, 44100, max_br=128000),
    "min": managed(1, 22050, min_br=48000),
    "cbr_small": managed(2, 44100, 128000, 128000, 128000, reservoir_bits=4000, bias=0.3, damp=0.5),
}


def size_sequences(rng, nseq, bs, target_bits, max_len=48):
    """random sequences of block flags and the 15 packets' bit counts per block: a loudness that drifts, drops to near
    silence or bursts, and curves that grow with the blob index.  Returns (lens, W, bits [total][15])."""
    lens = rng.integers(1, max_len + 1, nseq).astype(np.int32)
    total = int(lens.sum())
    W = (rng.random(total) < 0.7).astype(np.int32)
    spl = bs[1] // bs[0]
    level = np.exp(rng.normal(0, 0.5, total))
    level[rng.random(total) < 0.08] = 0.02
    level[rng.random(total) < 0.08] *= 6
    base = target_bits * np.where(W == 1, 1.0, 1.0 / spl) * level
    k = np.arange(NB)
    growth = rng.uniform(1.03, 1.15, (total, 1)) ** (k - 7)
    bits = base[:, None] * growth * rng.uniform(0.9, 1.1, (total, NB))
    bits = np.sort(np.maximum(bits, 9), axis=1)
    return lens, W, np.round(bits).astype(np.int32)


def target_bits(info, bs, rate):
    """a long block's share of the configuration's highest rate, in bits"""
    return max(info.avg_rate, info.max_rate, info.min_rate) * bs[1] / 2 / rate


def info_from_arrays(i_int, i_float):
    return abi.BitrateInfo(*[int(v) for v in i_int], *[float(v) for v in i_float])


# ---- the oracle -------------------------------------------------------------------------------------------
_olib = None


def _oracle_lib():
    global _olib
    if _olib is None:
        build()
        L = C.CDLL(ORACLE_LIB)
        L.vbo_bitrate_run.argtypes = [C.POINTER(abi.BitrateInfo), C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _olib = L
    return _olib


def vbo_bitrate_addblock(info, rate, bs, W, bits, state=None, branches=None):
    """the oracle over one stream's blocks: W [nb], bits [nb][15] -> (choice [nb], bytes [nb], state after every block
    (abi.BITRATE_STATE_DTYPE [nb])).  state: a BITRATE_STATE_DTYPE scalar array, advanced in place (None: fresh).
    branches: an int64 [6] array the branch counts are added to (BRANCHES)."""
    W = np.ascontiguousarray(W, np.int32)
    bits = np.ascontiguousarray(bits, np.int32).reshape(len(W), NB)
    nb = len(W)
    choice = np.zeros(max(nb, 1), np.int32)
    nbytes = np.zeros(max(nb, 1), np.int64)
    after = np.zeros(max(nb, 1), abi.BITRATE_STATE_DTYPE)
    br = np.zeros(len(BRANCHES), np.int64) if branches is None else branches
    if _oracle_lib().vbo_bitrate_run(C.byref(info), rate, bs[0], bs[1], nb, W.ctypes.data, bits.ctypes.data,
                                     None if state is None else state.ctypes.data, choice.ctypes.data,
                                     nbytes.ctypes.data, after.ctypes.data, br.ctypes.data):
        raise ValueError("not a managed bitrate setup")
    return choice[:nb], nbytes[:nb], after[:nb]


# ---- the reference ----------------------------------------------------------------------------------------
_rlibs = {}


def _ref_lib(dropin=False):
    if dropin not in _rlibs:
        L = C.CDLL(DROPIN_LIB if dropin else REF_LIB)
        if dropin:
            L.rbr_open_managed.restype = C.c_void_p
            L.rbr_open_managed.argtypes = [C.c_int, C.c_long, C.c_long, C.c_long, C.c_long, C.c_int]
            L.rbr_ctx.restype = C.c_void_p
            L.rbr_ctx.argtypes = [C.c_void_p]
            L.rbr_close.argtypes = [C.c_void_p]
        else:
            L.ref_bitrate_info.argtypes = [C.POINTER(Config), C.POINTER(abi.BitrateInfo), C.c_void_p]
            L.ref_bitrate_replay.argtypes = [C.POINTER(Config), C.c_uint64, C.c_int, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
            L.ref_stream_capture.restype = C.c_long
            L.ref_stream_capture.argtypes = [C.POINTER(Config), C.c_void_p, C.c_long, C.c_long, C.c_void_p, C.c_long,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_long]
        _rlibs[dropin] = L
    return _rlibs[dropin]


def ref_bitrate_info(cf):
    """(abi.BitrateInfo of ci->bi, [blocksizes]) of the encoder cf opens"""
    info = abi.BitrateInfo()
    bs = np.zeros(2, np.int32)
    if _ref_lib().ref_bitrate_info(C.byref(cf), C.byref(info), bs.ctypes.data):
        raise RuntimeError("the reference refused the configuration")
    return info, [int(bs[0]), int(bs[1])]


def ref_bitrate_replay(cf, lens, W, bits, seed=1):
    """sequences of lens[i] blocks (W, bits concatenated), each from a fresh state, through the reference's own
    vorbis_bitrate_addblock / flushpacket: (choice, bytes, content_ok, state after every block)"""
    lens = np.ascontiguousarray(lens, np.int32)
    W = np.ascontiguousarray(W, np.int32)
    bits = np.ascontiguousarray(bits, np.int32).reshape(len(W), NB)
    t = len(W)
    assert lens.sum() == t
    choice = np.zeros(max(t, 1), np.int32)
    nbytes = np.zeros(max(t, 1), np.int64)
    ok = np.zeros(max(t, 1), np.int32)
    after = np.zeros(max(t, 1), abi.BITRATE_STATE_DTYPE)
    if _ref_lib().ref_bitrate_replay(C.byref(cf), seed, len(lens), lens.ctypes.data, W.ctypes.data, bits.ctypes.data,
                                     choice.ctypes.data, nbytes.ctypes.data, ok.ctypes.data, after.ctypes.data):
        raise RuntimeError("reference replay failed")
    return choice[:t], nbytes[:t], ok[:t], after[:t]


def ref_stream_capture(cf, pcm, chunk=1024):
    """one stream pcm [ch][n] through a stock encoder: {"timeline" [ch][len], "eof", "packets": [bytes],
    "granulepos", "e_o_s", "packetno"} (audio packets only)"""
    pcm = np.ascontiguousarray(pcm, np.float32)
    ch, n = pcm.shape
    L = _ref_lib()
    tl_cap = n + 8 * 8192
    tl = np.zeros((ch, tl_cap), np.float32)
    maxn = n // 32 + 64
    cap = max(1 << 20, n * ch * 4)
    out = np.zeros(cap, np.uint8)
    nbytes, gp, pno = (np.zeros(maxn, np.int64) for _ in range(3))
    eos = np.zeros(maxn, np.int32)
    tl_len, eof = C.c_int64(0), C.c_int64(0)
    np_ = L.ref_stream_capture(C.byref(cf), pcm.ctypes.data, n, chunk, tl.ctypes.data, tl_cap, C.byref(tl_len),
                               C.byref(eof), out.ctypes.data, cap, nbytes.ctypes.data, gp.ctypes.data, eos.ctypes.data,
                               pno.ctypes.data, maxn)
    if np_ < 0:
        raise RuntimeError("stock encode failed (%d)" % np_)
    off = np.concatenate([[0], np.cumsum(nbytes[:np_])])
    return {"timeline": tl[:, :tl_len.value].copy(), "eof": int(eof.value),
            "packets": [bytes(out[off[i]:off[i + 1]]) for i in range(np_)],
            "granulepos": gp[:np_].copy(), "e_o_s": eos[:np_].copy(), "packetno": pno[:np_].copy()}


class ManagedDriver:
    """a managed multi-stream driver vb200ms_open_managed(1, ch, rate, max, nominal, min); .ctx is a lib.Context on
    its device context, which carries the managed encoder's setup and entropy setup"""

    def __init__(self, ch, rate, max_br, nominal_br, min_br, device=0):
        from vorbis_b200 import lib
        self.L = _ref_lib(True)
        self.m = self.L.rbr_open_managed(ch, rate, max_br, nominal_br, min_br, device)
        if not self.m:
            raise RuntimeError("vb200ms_open_managed failed or took the host entropy path")
        cf = managed(ch, rate, max_br, nominal_br, min_br)
        _, bs = ref_bitrate_info(cf)
        self.ctx = lib.Context.wrap(self.L.rbr_ctx(self.m), ch, bs)

    def close(self):
        if self.m:
            self.ctx.h = None
            self.L.rbr_close(self.m)
            self.m = None
