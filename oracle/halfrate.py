"""Half-rate decode (vorbis_synthesis_halfrate) for the tests: build recipes and ctypes loaders of
  oracle/libvb_oracle_halfrate.so          the CPU oracle's half-rate synthesis (vb_oracle_halfrate.c)
  oracle/_ref/libvorbis_ref_halfrate.so    the reference's own encoder / half-rate decoder (ref_halfrate.c)
  oracle/_ref/libvorbis_dropin_halfrate.so the same decoder with mdct_backward bound to the CUDA shim
The two reference libraries link the objects oracle/Makefile compiles from the unmodified reference sources
(targets `ref` and `dropin`) and are only built where those exist; like the rest of oracle/_ref they travel.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tests/golden/make_golden_halfrate.py, never by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from vorbis_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
OBJ = os.path.join(REF_DIR, "obj")
ORACLE_LIB = os.path.join(HERE, "libvb_oracle_halfrate.so")
REF_LIB = os.path.join(REF_DIR, "libvorbis_ref_halfrate.so")
DROPIN_LIB = os.path.join(REF_DIR, "libvorbis_dropin_halfrate.so")
REF_SRC = os.environ.get("REF", "/root/reference")

# oracle/Makefile: PARITY flags, REFSRC, REFINC, and the object sets of libvorbis_ref.so / libvorbis_dropin.so
PARITY = ["-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-fvisibility=default"]
REFSRC = ["mdct", "window", "smallft", "psy", "block", "analysis", "synthesis", "envelope", "floor1", "floor0",
          "res0", "codebook", "sharedbook", "info", "registry", "bitrate", "lpc", "lsp", "lookup", "vorbisenc"]
REF_OBJS = [s + ".o" for s in REFSRC] + ["mapping0.o", "ref_driver.o", "bitpack.o"]
DROPIN_OBJS = ([s + ".o" for s in REFSRC if s != "block"] +
               ["block_shim.o", "mapping0_shim.o", "vb200_ref_shim.o", "vb200_mapping0.o", "bitpack.o"])

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")


def _stale(target, sources):
    return not os.path.exists(target) or any(os.path.getmtime(s) > os.path.getmtime(target) for s in sources)


def build(cc="gcc"):
    """the oracle library always; the two reference libraries where oracle/Makefile's objects exist"""
    inc = os.path.join(os.path.dirname(HERE), "include")
    deps = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.startswith("vb_oracle") or f == "floor1_db_table.h"]
    if _stale(ORACLE_LIB, deps):
        subprocess.check_call([cc] + PARITY + ["-std=gnu99", "-Wall", "-I" + inc, "-I" + HERE, "-shared", "-o",
                                               ORACLE_LIB, os.path.join(HERE, "vb_oracle_halfrate.c"), "-lm"])
    if not os.path.exists(os.path.join(REF_SRC, "lib", "mdct.c")):
        return
    refinc = ["-I" + os.path.join(HERE, "shim"), "-I" + os.path.join(REF_SRC, "include"),
              "-I" + os.path.join(REF_SRC, "lib"), "-I" + inc]
    src = os.path.join(HERE, "ref_halfrate.c")
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


# ---- the oracle ---------------------------------------------------------------------------------------
_olib = None


def _oracle_lib():
    global _olib
    if _olib is None:
        build()
        L = C.CDLL(ORACLE_LIB)
        L.vbohs_create.restype = C.c_void_p
        L.vbohs_create.argtypes = [C.POINTER(abi.Setup), C.c_void_p]
        L.vbohs_destroy.argtypes = [C.c_void_p]
        L.vbohs_mdct_backward.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p]
        L.vbohs_synthesis.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i64p, f32p, i64p, f32p, C.c_int64]
        L.vbohs_decode_dsp.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i64p, f32p, i32p, i32p, i64p, f32p,
                                       C.c_int64]
        _olib = L
    return _olib


class Oracle:
    """The CPU oracle in half-rate mode for one setup (abi.SetupHolder).  windows: the half windows of
    blocksizes[w]/2 (SetupHolder.halfrate_windows()); None = closed form."""

    @classmethod
    def create(cls, setup, windows=None):
        """None where vorbis_synthesis_halfrate refuses (blocksizes[0] <= 64)"""
        L = _oracle_lib()
        keep, ptrs = abi.halfrate_window_ptrs(windows)
        h = L.vbohs_create(C.byref(setup.c), ptrs)
        if not h:
            return None
        self = cls()
        self.L, self.h, self.setup = L, h, setup
        self.channels = setup.channels
        self.bs = [setup.blocksize(0), setup.blocksize(1)]
        return self

    def close(self):
        if getattr(self, "h", None):
            self.L.vbohs_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def mdct_backward(self, W, x):
        """mdct_backward at N = blocksizes[W]/2: [nvec][N/2] -> [nvec][N]"""
        N = self.bs[W] // 2
        x = np.ascontiguousarray(x, np.float32).reshape(-1, N // 2)
        out = np.empty((x.shape[0], N), np.float32)
        self.L.vbohs_mdct_backward(self.h, W, x.shape[0], x, out)
        return out

    def synthesis(self, Wseq, coef_off, coef, pcm_off, pcm_stride):
        """layout of vorbis_b200.lib.synthesis_layout(..., halfrate=True)"""
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        pcm = np.zeros((ns, self.channels, pcm_stride), np.float32)
        self.L.vbohs_synthesis(self.h, ns, nblk, Wseq, np.ascontiguousarray(coef_off, np.int64),
                               np.ascontiguousarray(coef, np.float32), np.ascontiguousarray(pcm_off, np.int64),
                               pcm, pcm_stride)
        return pcm

    def decode_dsp(self, Wseq, coef_off, res, posts, present, pcm_off, pcm_stride):
        """de-couple + floor multiply (full size) + half-rate IMDCT and overlap-add; res is not modified"""
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        res = np.array(res, np.float32)
        pcm = np.zeros((ns, self.channels, pcm_stride), np.float32)
        self.L.vbohs_decode_dsp(self.h, ns, nblk, Wseq, np.ascontiguousarray(coef_off, np.int64), res,
                                np.ascontiguousarray(posts, np.int32).reshape(-1),
                                np.ascontiguousarray(present, np.int32).reshape(-1),
                                np.ascontiguousarray(pcm_off, np.int64), pcm, pcm_stride)
        return pcm


# ---- the reference ------------------------------------------------------------------------------------
def ref_available(dropin=False):
    return os.path.exists(DROPIN_LIB if dropin else REF_LIB)


_rlibs = {}


def _ref_lib(dropin):
    if dropin not in _rlibs:
        L = C.CDLL(DROPIN_LIB if dropin else REF_LIB)
        L.refhs_encode.argtypes = [C.c_int, C.c_long, C.c_float, f32p, C.c_long, C.c_void_p, C.c_long, C.c_void_p,
                                   C.c_int]
        L.refhs_decode.restype = C.c_long
        L.refhs_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, f32p, C.c_long, i32p, C.c_int,
                                   C.POINTER(C.c_int), f32p, f32p]
        _rlibs[dropin] = L
    return _rlibs[dropin]


def ref_encode(ch, rate, quality, pcm):
    """the stock reference encoder's packets (3 headers, then audio) for pcm [ch][n]: (bytes, sizes int64)"""
    L = _ref_lib(False)
    pcm = np.ascontiguousarray(pcm, np.float32)
    cap, maxn = 1 << 24, 1 << 16
    buf = np.zeros(cap, np.uint8)
    sizes = np.zeros(maxn, np.int64)
    n = L.refhs_encode(ch, rate, quality, pcm, pcm.shape[1], buf.ctypes.data, cap, sizes.ctypes.data, maxn)
    if n < 0:
        raise RuntimeError("reference encode failed")
    return buf[:int(sizes[:n].sum())].copy(), sizes[:n].copy()


def ref_decode(packets, bs, channels, pcm_cap, halfrate=True, dropin=False):
    """decode ref_encode's packets with the reference's API loop (dropin: mdct_backward through the CUDA shim),
    after vorbis_synthesis_halfrate(vi, 1) when halfrate.  Returns pcm [ch][n], the block flags and the two
    half windows the decoder's overlap-add used (window0, window1)."""
    L = _ref_lib(dropin)
    buf, sizes = packets
    buf = np.ascontiguousarray(buf, np.uint8)
    sizes = np.ascontiguousarray(sizes, np.int64)
    pcm = np.zeros((channels, pcm_cap), np.float32)
    maxblocks = len(sizes)
    Wseq = np.zeros(maxblocks, np.int32)
    nb = C.c_int(0)
    win = [np.zeros(bs[w] // 4, np.float32) for w in (0, 1)]
    got = L.refhs_decode(buf.ctypes.data, sizes.ctypes.data, len(sizes), 1 if halfrate else 0, pcm, pcm_cap, Wseq,
                         maxblocks, C.byref(nb), win[0], win[1])
    if got < 0:
        raise RuntimeError("reference decode failed")
    return {"pcm": pcm[:, :got], "W": Wseq[:nb.value], "window0": win[0], "window1": win[1]}
