"""The carried block planner for the tests: build recipes and ctypes loaders of
  oracle/libvb_oracle_resume.so        vb_oracle_resume.c: the plain-C restatement of the planner that
                                       vb200_encode_streams_packets[_managed]_resume carry from call to call
  oracle/_ref/libvorbis_ref_resume.so  ref_resume.c + the stock reference objects: the reference's planner state
                                       after every vorbis_analysis_blockout of a stream written in chunks
The reference library links the objects oracle/Makefile compiles from the unmodified reference sources and is only
built where those exist; like the rest of oracle/_ref it travels.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.halfrate import OBJ, PARITY, REF_OBJS, REF_SRC, _stale
from vorbis_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ORACLE_LIB = os.path.join(HERE, "libvb_oracle_resume.so")
REF_LIB = os.path.join(HERE, "_ref", "libvorbis_ref_resume.so")
REC_FIELDS = ("write", "base", "current", "cursor", "curmark", "kept", "centerW", "W", "lW", "nW", "blocktype")


def build(cc="gcc"):
    inc = os.path.join(ROOT, "include")
    osrc = os.path.join(HERE, "vb_oracle_resume.c")
    if _stale(ORACLE_LIB, [osrc, os.path.join(inc, "vorbis_b200.h")]):
        subprocess.check_call([cc] + PARITY + ["-std=gnu99", "-Wall", "-I" + inc, "-shared", "-o", ORACLE_LIB, osrc])
    if not os.path.exists(os.path.join(REF_SRC, "lib", "mdct.c")):
        return
    paths = [os.path.join(OBJ, o) for o in REF_OBJS]
    src = os.path.join(HERE, "ref_resume.c")
    if not all(os.path.exists(p) for p in paths) or not _stale(REF_LIB, paths + [src]):
        return
    refinc = ["-I" + os.path.join(HERE, "shim"), "-I" + os.path.join(REF_SRC, "include"),
              "-I" + os.path.join(REF_SRC, "lib"), "-I" + inc]
    obj = REF_LIB[:-3] + ".o"
    subprocess.check_call([cc] + PARITY + ["-Wall"] + refinc + ["-c", src, "-o", obj])
    subprocess.check_call([cc, "-shared", "-Wl,-Bsymbolic", "-o", REF_LIB, obj] + paths + ["-lm"])
    os.remove(obj)


class Carry(C.Structure):
    """vbo_carry of vb_oracle_resume.c"""
    _fields_ = [("base", C.c_int64), ("kept", C.c_int64), ("centerW", C.c_int64), ("cursor", C.c_int64),
                ("curmark", C.c_int64), ("current", C.c_int64), ("W", C.c_int32), ("lW", C.c_int32),
                ("done", C.c_int32), ("pad", C.c_int32)]


_libs = {}


def _load(path):
    if path not in _libs:
        _libs[path] = C.CDLL(path)
    return _libs[path]


def ref_available():
    return os.path.exists(REF_LIB)


class Planner:
    """one stream's carried planner: feed(ora, buf, pcm_len, eof, max_blocks) analyses the envelope steps the carry
    has not seen (with the pyoracle.Oracle `ora` and the carried envelope state) and plans; returns the plan rows"""

    def __init__(self, bs, ch, cap=4096):
        self.L = _load(ORACLE_LIB)
        self.L.vbo_carry_init.argtypes = [C.c_int, C.POINTER(Carry)]
        self.L.vbo_plan_blocks_resume.argtypes = [C.c_int, C.c_int, C.POINTER(Carry), C.c_void_p, C.c_int, C.c_void_p,
                                                  C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p]
        self.bs, self.cap = bs, cap
        self.c = Carry()
        self.L.vbo_carry_init(bs[1], C.byref(self.c))
        self.window = np.zeros(cap, np.uint8)
        self.env = np.zeros((1, abi.ve_state_words(ch)), np.int32)

    def feed(self, ora, buf, pcm_len, eof=0, max_blocks=1 << 20):
        first = self.c.current // 64
        count = max(0, pcm_len // 64 - 4 - first)
        ret = np.zeros(max(count, 1), np.uint8)
        if count and not self.c.done:
            pad = np.zeros((1, buf.shape[0], max(buf.shape[1], 64 * (first + count) + 64)), np.float32)
            pad[0, :, :buf.shape[1]] = buf
            r, self.env = ora.envelope_search(pad, first, count, self.env)
            ret[:count] = r[0]
        plan = np.zeros(max(max_blocks, 1) if max_blocks < 4096 else 4096, abi.STREAM_BLOCK_DTYPE)
        nb = self.L.vbo_plan_blocks_resume(self.bs[0], self.bs[1], C.byref(self.c), self.window.ctypes.data, self.cap,
                                           ret.ctypes.data, count, pcm_len, eof, min(max_blocks, len(plan)),
                                           plan.ctypes.data)
        assert nb >= 0, "mark window overflow"
        return plan[:nb]


def ref_resume_capture(ch, rate, q, pcm, chunk):
    """the stock VBR encoder on pcm [ch][n] written in chunks: {"timeline", "eof", "write_end" [writes],
    "rec" [blocks] structured by REC_FIELDS}"""
    L = _load(REF_LIB)
    f = L.ref_resume_capture
    f.restype = C.c_long
    f.argtypes = [C.c_int, C.c_long, C.c_double, C.c_void_p, C.c_long, C.c_long, C.c_void_p, C.c_long, C.c_void_p,
                  C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_long]
    pcm = np.ascontiguousarray(pcm, np.float32)
    n = pcm.shape[1]
    cap = n + 8 * 8192
    tl = np.zeros((ch, cap), np.float32)
    tl_len, eof = np.zeros(1, np.int64), np.zeros(1, np.int64)
    maxw = n // max(chunk, 1) + 4
    wend = np.zeros(maxw, np.int64)
    maxn = n // 64 + 64
    rec = np.zeros((maxn, len(REC_FIELDS)), np.int64)
    nb = f(ch, rate, q, pcm.ctypes.data, n, chunk, tl.ctypes.data, cap, tl_len.ctypes.data, eof.ctypes.data,
           wend.ctypes.data, maxw, rec.ctypes.data, maxn)
    assert nb >= 0
    nw = -(-n // chunk) + 1                            # the writes of PCM, then vorbis_analysis_wrote(v, 0)
    return {"timeline": tl[:, :tl_len[0]].copy(), "eof": int(eof[0]), "write_end": wend[:nw],
            "rec": {k: rec[:nb, i] for i, k in enumerate(REC_FIELDS)}}
