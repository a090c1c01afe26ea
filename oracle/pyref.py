"""ctypes loader for oracle/_ref/libvorbis_ref.so — the UNMODIFIED reference sources
compiled by oracle/Makefile, driven through oracle/ref_driver.c.

TEST INFRASTRUCTURE ONLY: imported by tests/, tests/golden/make_golden.py,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg; never
by the product package.
"""
import ctypes as C
import os

import numpy as np

from vorbis_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_ref", "libvorbis_ref.so")
DROPIN_PATH = os.path.join(HERE, "_ref", "libvorbis_dropin.so")
if os.environ.get("VB200_DROPIN_EMU"):      # development aid (tools/cuemu): the drop-in linked against the host emulation
    DROPIN_PATH = os.path.join(HERE, "_ref", "libvorbis_dropin_emu.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")


def available():
    return os.path.exists(LIB_PATH)


def coupling_hooks_available():
    """whether the built library has ref_set_coupling and ref_get_headers (Ref.set_coupling, Ref.headers); a library
    built from an older ref_driver.c has neither, and every other entry point still works"""
    return available() and all(hasattr(lib(), k) for k in ("ref_set_coupling", "ref_get_headers"))


class Capture(C.Structure):
    _fields_ = [
        ("maxblocks", C.c_int), ("Nmax", C.c_int), ("nblocks", C.c_int),
        ("W", C.c_void_p), ("lW", C.c_void_p), ("nW", C.c_void_p), ("blocktype", C.c_void_p),
        ("ampmax_in", C.c_void_p), ("ampmax_out", C.c_void_p),
        ("pcm", C.c_void_p), ("windowed", C.c_void_p), ("fft", C.c_void_p), ("mdct_raw", C.c_void_p),
        ("logfft", C.c_void_p), ("logmdct", C.c_void_p), ("noise", C.c_void_p), ("tone", C.c_void_p),
        ("logmask", C.c_void_p), ("mdct_m1", C.c_void_p), ("local_ampmax", C.c_void_p),
        ("global_ampmax", C.c_void_p), ("ilogmask", C.c_void_p), ("iwork_out", C.c_void_p),
        ("nonzero_in", C.c_void_p), ("nonzero_out", C.c_void_p),
        ("fit_posts", C.c_void_p), ("enc_posts", C.c_void_p),
        ("dec_coef", C.c_void_p), ("dec_imdct", C.c_void_p),
    ]


_lib = None
_dropin = None


def dropin_available():
    return os.path.exists(DROPIN_PATH)


def dropin_lib():
    """The reference encoder/decoder whose mapping0 hot callees are redirected to the CUDA
    shims (vorbis_b200/host/vb200_ref_shim.c); same driver entry points as lib()."""
    global _dropin
    if _dropin is None:
        L = C.CDLL(DROPIN_PATH)
        _declare(L)
        L.vb200shim_attach.argtypes = [C.c_void_p, C.c_int]
        L.vb200shim_launches.restype = C.c_ulonglong
        L.ref_use_block_seam.argtypes = [C.c_int]
        _dropin = L
    return _dropin


def _declare(L):
    L.ref_open.restype = C.c_void_p
    L.ref_open.argtypes = [C.c_int, C.c_long, C.c_float]
    L.ref_open_managed.restype = C.c_void_p
    L.ref_open_managed.argtypes = [C.c_int, C.c_long, C.c_long]
    L.ref_close.argtypes = [C.c_void_p]
    L.ref_vd.restype = C.c_void_p
    L.ref_vd.argtypes = [C.c_void_p]
    L.ref_blocksize.argtypes = [C.c_void_p, C.c_int]
    L.ref_get_packets.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_int]
    if hasattr(L, "ref_get_headers"):
        L.ref_get_headers.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p]
    L.ref_encode_capture.argtypes = [C.c_void_p, f32p, C.c_long, C.POINTER(Capture), C.POINTER(C.c_long)]
    L.ref_decode_capture.restype = C.c_long
    L.ref_decode_capture.argtypes = [C.c_void_p, C.POINTER(Capture), f32p, C.c_long, C.c_void_p]


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB_PATH)
        _declare(L)
        L.ref_open.restype = C.c_void_p
        L.ref_open.argtypes = [C.c_int, C.c_long, C.c_float]
        L.ref_open_managed.restype = C.c_void_p
        L.ref_open_managed.argtypes = [C.c_int, C.c_long, C.c_long]
        L.ref_close.argtypes = [C.c_void_p]
        L.ref_blocksize.argtypes = [C.c_void_p, C.c_int]
        L.ref_get_setup.argtypes = [C.c_void_p, C.POINTER(abi.Setup)]
        if hasattr(L, "ref_set_coupling"):
            L.ref_set_coupling.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i32p]
        L.ref_get_table.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
        L.ref_mdct_forward.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p]
        L.ref_mdct_backward.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p]
        L.ref_apply_window.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, f32p]
        L.ref_drft_forward.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p]
        L.ref_noisemask.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p]
        L.ref_tonemask.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p, f32p, f32p]
        L.ref_offset_and_mix.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, f32p, f32p, f32p, f32p, f32p]
        L.ref_couple_quantize_normalize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    f32p, i32p, i32p]
        L.ref_ampmax_decay.restype = C.c_float
        L.ref_ampmax_decay.argtypes = [C.c_void_p, C.c_float, C.c_int]
        L.ref_encode_capture.argtypes = [C.c_void_p, f32p, C.c_long, C.POINTER(Capture), C.POINTER(C.c_long)]
        L.ref_decode_capture.restype = C.c_long
        L.ref_decode_capture.argtypes = [C.c_void_p, C.POINTER(Capture), f32p, C.c_long, C.c_void_p]
        L.ref_blockin_sequence.restype = C.c_long
        L.ref_blockin_sequence.argtypes = [C.c_void_p, C.c_int, i32p, f32p, C.c_int, f32p, C.c_long]
        L.ref_phaseA_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, C.c_void_p, f32p, f32p, f32p, f32p]
        L.ref_residue_classify.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i32p, i32p, C.c_int]
        L.ref_floor1_inverse2.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i32p, f32p]
        L.ref_set_timeline.argtypes = [C.c_void_p, C.c_long]
        L.ref_get_timeline.argtypes = [C.POINTER(C.c_long), C.POINTER(C.c_long)]
        L.ref_envelope_marks.restype = C.c_long
        L.ref_envelope_marks.argtypes = [C.c_void_p, f32p, C.c_long, i32p, C.c_long, C.c_void_p, f32p]
        L.ref_encode_dsp_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, C.c_void_p, i32p, i32p, i32p, f32p]
        L.ref_encode_dsp_managed_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, C.c_void_p, i32p, i32p, i32p, f32p]
        _lib = L
    return _lib


_CAP_F_N = ["pcm", "windowed", "fft", "dec_imdct"]
_CAP_F_n = ["mdct_raw", "logfft", "logmdct", "noise", "tone", "logmask", "mdct_m1", "dec_coef"]
_CAP_I_n = ["ilogmask", "iwork_out"]


class Ref:
    """One reference encoder instance: vorbis_encode_init_vbr(channels, rate, quality).
    dropin=True uses the CUDA-shimmed build and attaches the device context."""

    def __init__(self, channels=2, rate=44100, quality=0.5, dropin=False, device=0, nominal_bitrate=None):
        """nominal_bitrate (bits/s): a bitrate-managed encoder (vorbis_encode_init) instead of VBR quality"""
        self.L = dropin_lib() if dropin else lib()
        self.h = (self.L.ref_open(channels, rate, quality) if nominal_bitrate is None
                  else self.L.ref_open_managed(channels, rate, int(nominal_bitrate)))
        if not self.h:
            raise RuntimeError("reference refused setup (ch=%d rate=%d q=%g)" % (channels, rate, quality))
        self.channels, self.rate, self.quality = channels, rate, quality
        self.bs = [self.L.ref_blocksize(self.h, 0), self.L.ref_blocksize(self.h, 1)]
        self.dropin = dropin
        if dropin:
            rc = self.L.vb200shim_attach(self.L.ref_vd(self.h), device)
            if rc:
                raise RuntimeError("vb200shim_attach failed: %d" % rc)

    def packets(self):
        """bytes of every packet produced by encode_capture (list of bytes objects)"""
        cap = 1 << 24
        buf = (C.c_ubyte * cap)()
        sizes = (C.c_long * 100000)()
        n = self.L.ref_get_packets(self.h, buf, cap, sizes, 100000)
        assert n >= 0
        out, off = [], 0
        raw = bytes(buf)
        for i in range(n):
            out.append(raw[off:off + sizes[i]])
            off += sizes[i]
        return out

    def headers(self):
        """the identification, comment and setup header packets encode_capture wrote (list of 3 bytes objects)"""
        cap = 1 << 20
        buf = (C.c_ubyte * cap)()
        sizes = (C.c_long * 3)()
        if self.L.ref_get_headers(self.h, buf, cap, sizes) != 3:
            raise RuntimeError("no headers: run encode_capture first")
        raw, off, out = bytes(buf), 0, []
        for n in sizes:
            out.append(raw[off:off + n])
            off += n
        return out

    def close(self):
        if self.h and getattr(self, "dropin", False):
            self.L.vb200shim_detach()
        if self.h:
            self.L.ref_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def setup(self):
        s = abi.Setup()
        if self.L.ref_get_setup(self.h, C.byref(s)):
            raise RuntimeError("ref_get_setup failed")
        return abi.SetupHolder.from_struct(s)

    def set_coupling(self, W, steps):
        """replace the coupling map of mode W by steps = [(mag, ang), ...] (ref_set_coupling): setup(), the stage
        calls, the batched chains and the headers of encode_capture then use it.  The map is not checked."""
        mag = np.ascontiguousarray([m for m, _ in steps] or [0], np.int32)
        ang = np.ascontiguousarray([a for _, a in steps] or [0], np.int32)
        if self.L.ref_set_coupling(self.h, W, len(steps), mag, ang):
            raise RuntimeError("ref_set_coupling refused W=%d with %d steps" % (W, len(steps)))

    def table(self, W, which):
        N = self.bs[W]
        if which == 1:
            out = np.zeros(N // 4, np.int32)
        else:
            out = np.zeros(2 * N, np.float32)
        k = self.L.ref_get_table(self.h, W, which, out.ctypes.data, out.size)
        assert k > 0
        return out[:k].copy()

    # ---- stage calls ---------------------------------------------------------
    def mdct_forward(self, W, x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1, self.bs[W])
        out = np.empty((x.shape[0], self.bs[W] // 2), np.float32)
        self.L.ref_mdct_forward(self.h, W, x.shape[0], x, out)
        return out

    def mdct_backward(self, W, x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1, self.bs[W] // 2)
        out = np.empty((x.shape[0], self.bs[W]), np.float32)
        self.L.ref_mdct_backward(self.h, W, x.shape[0], x, out)
        return out

    def apply_window(self, W, x, lW=None, nW=None):
        x = np.array(x, np.float32).reshape(-1, self.bs[W])
        lWa = None if lW is None else np.ascontiguousarray(lW, np.int32)
        nWa = None if nW is None else np.ascontiguousarray(nW, np.int32)
        self.L.ref_apply_window(self.h, W, x.shape[0],
                                None if lWa is None else lWa.ctypes.data,
                                None if nWa is None else nWa.ctypes.data, x)
        return x

    def drft_forward(self, W, x):
        x = np.array(x, np.float32).reshape(-1, self.bs[W])
        self.L.ref_drft_forward(self.h, W, x.shape[0], x)
        return x

    def noisemask(self, look, logmdct):
        x = np.ascontiguousarray(logmdct, np.float32)
        x = x.reshape(-1, x.shape[-1])
        out = np.empty_like(x)
        self.L.ref_noisemask(self.h, look, x.shape[0], x, out)
        return out

    def tonemask(self, look, logfft, gmax, lmax):
        x = np.ascontiguousarray(logfft, np.float32)
        x = x.reshape(-1, x.shape[-1])
        out = np.empty_like(x)
        g = np.ascontiguousarray(np.broadcast_to(np.asarray(gmax, np.float32), (x.shape[0],)))
        l = np.ascontiguousarray(np.broadcast_to(np.asarray(lmax, np.float32), (x.shape[0],)))
        self.L.ref_tonemask(self.h, look, x.shape[0], x, g, l, out)
        return out

    def offset_and_mix(self, look, sel, noise, tone, mdct, logmdct):
        noise = np.ascontiguousarray(noise, np.float32)
        noise = noise.reshape(-1, noise.shape[-1])
        tone = np.ascontiguousarray(tone, np.float32).reshape(noise.shape)
        mdct = np.array(mdct, np.float32).reshape(noise.shape)
        logmdct = np.ascontiguousarray(logmdct, np.float32).reshape(noise.shape)
        logmask = np.empty_like(noise)
        self.L.ref_offset_and_mix(self.h, look, noise.shape[0], sel, noise, tone, mdct, logmdct, logmask)
        return logmask, mdct

    def couple_quantize_normalize(self, W, blocktype, blobno, mdct, iwork, nonzero):
        mdct = np.array(mdct, np.float32)
        iwork = np.array(iwork, np.int32)
        nonzero = np.array(nonzero, np.int32)
        nb = mdct.shape[0]
        self.L.ref_couple_quantize_normalize(self.h, W, blocktype, blobno, nb, mdct, iwork, nonzero)
        return iwork, nonzero

    def ampmax_decay(self, amp, W):
        return float(self.L.ref_ampmax_decay(self.h, float(amp), W))

    def phaseA_batch(self, W, pcm, desc):
        ch, N = self.channels, self.bs[W]
        pcm = np.ascontiguousarray(pcm, np.float32).reshape(-1, ch, N)
        nb = pcm.shape[0]
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        mdct = np.empty((nb, ch, N // 2), np.float32)
        logmdct = np.empty_like(mdct)
        logmask = np.empty_like(mdct)
        amp = np.empty(nb, np.float32)
        self.L.ref_phaseA_batch(self.h, W, nb, pcm, desc.ctypes.data, mdct, logmdct, logmask, amp)
        return mdct, logmdct, logmask, amp

    def residue_classify(self, W, iwork, nonzero, stride):
        """the reference's res{0,1,2}_class per submap (lib/mapping0.c:660-672) on [block][ch][n] ints"""
        ch, n = self.channels, self.bs[W] // 2
        iwork = np.ascontiguousarray(iwork, np.int32).reshape(-1, ch, n)
        nonzero = np.ascontiguousarray(nonzero, np.int32).reshape(-1, ch)
        classes = np.zeros((iwork.shape[0], ch, stride), np.int32)
        self.L.ref_residue_classify(self.h, W, iwork.shape[0], iwork, nonzero, classes, stride)
        return classes

    def floor1_inverse2(self, W, posts, present, data):
        """the reference's floor1_inverse2 (lib/floor1.c:1041) on rows [block][channel]"""
        posts = np.ascontiguousarray(posts, np.int32).reshape(-1, 65)
        present = np.ascontiguousarray(present, np.int32).reshape(-1)
        data = np.array(data, np.float32).reshape(posts.shape[0], self.bs[W] // 2)
        self.L.ref_floor1_inverse2(self.h, W, posts.shape[0], posts, present, data)
        return data

    def envelope_marks(self, pcm):
        """pcm [ch][S] float -> (marks int32 [steps+2], steps, state words, stream [ch][bs1/2+S]) from the
        reference's own _ve_envelope_search on a fresh dsp state (lib/envelope.c:216).  The reference's
        stream buffer starts with blocksizes[1]/2 samples of preamble (v->pcm_current = v->centerW at
        init, lib/block.c:283-284; zeros, later overwritten by _preextrapolate_helper's reverse LPC
        extrapolation): step j covers samples 64j.. of the returned stream."""
        pcm = np.ascontiguousarray(pcm, np.float32)
        ch, S = pcm.shape
        cap = (S + self.bs[1] // 2) // 64 + 8
        marks = np.zeros(cap, np.int32)
        state = np.zeros(abi.ve_state_words(ch), np.int32)
        stream = np.zeros((ch, self.bs[1] // 2 + S), np.float32)
        steps = int(self.L.ref_envelope_marks(self.h, pcm, S, marks, cap, state.ctypes.data, stream))
        return marks[:steps + 2], steps, state, stream

    def encode_dsp_batch(self, W, pcm, desc):
        """the reference's own functions in mapping0_forward's order: Phase A, floor1_fit, floor1_encode,
        _vp_couple_quantize_normalize (blob PACKETBLOBS/2); independent blocks, desc[].ampmax on entry"""
        ch, N = self.channels, self.bs[W]
        pcm = np.ascontiguousarray(pcm, np.float32).reshape(-1, ch, N)
        nb = pcm.shape[0]
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        out = {"posts": np.zeros((nb, ch, 65), np.int32), "nonzero": np.zeros((nb, ch), np.int32),
               "iwork": np.zeros((nb, ch, N // 2), np.int32), "ampmax_out": np.zeros(nb, np.float32)}
        self.L.ref_encode_dsp_batch(self.h, W, nb, pcm, desc.ctypes.data, out["posts"], out["nonzero"],
                                    out["iwork"], out["ampmax_out"])
        return out

    def encode_dsp_managed_batch(self, W, pcm, desc):
        """bitrate-managed mapping0_forward with the reference's own functions (ref_encode_dsp_managed_batch):
        blob-major posts [15][nb][ch][65], nonzero [15][nb][ch], iwork [15][nb][ch][n]"""
        ch, N = self.channels, self.bs[W]
        pcm = np.ascontiguousarray(pcm, np.float32).reshape(-1, ch, N)
        nb = pcm.shape[0]
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        NB = abi.PACKETBLOBS
        out = {"posts": np.zeros((NB, nb, ch, 65), np.int32), "nonzero": np.zeros((NB, nb, ch), np.int32),
               "iwork": np.zeros((NB, nb, ch, N // 2), np.int32), "ampmax_out": np.zeros(nb, np.float32)}
        self.L.ref_encode_dsp_managed_batch(self.h, W, nb, pcm, desc.ctypes.data, out["posts"], out["nonzero"],
                                            out["iwork"], out["ampmax_out"])
        return out

    # ---- full API capture ----------------------------------------------------
    def _mkcap(self, maxblocks, fields):
        ch, Nmax = self.channels, self.bs[1]
        cap = Capture()
        cap.maxblocks, cap.Nmax = maxblocks, Nmax
        arr = {}
        for name in ("W", "lW", "nW", "blocktype"):
            arr[name] = np.zeros(maxblocks, np.int32)
        for name in ("ampmax_in", "ampmax_out", "global_ampmax"):
            arr[name] = np.zeros(maxblocks, np.float32)
        arr["local_ampmax"] = np.zeros((maxblocks, ch), np.float32)
        arr["nonzero_in"] = np.zeros((maxblocks, ch), np.int32)
        arr["nonzero_out"] = np.zeros((maxblocks, ch), np.int32)
        arr["fit_posts"] = np.zeros((maxblocks, ch, 65), np.int32)
        arr["enc_posts"] = np.zeros((maxblocks, ch, 65), np.int32)
        for name in _CAP_F_N:
            if name in fields:
                arr[name] = np.zeros((maxblocks, ch, Nmax), np.float32)
        for name in _CAP_F_n:
            if name in fields:
                arr[name] = np.zeros((maxblocks, ch, Nmax // 2), np.float32)
        for name in _CAP_I_n:
            if name in fields:
                arr[name] = np.zeros((maxblocks, ch, Nmax // 2), np.int32)
        for k, v in arr.items():
            setattr(cap, k, v.ctypes.data)
        return cap, arr

    def encode_capture(self, pcm, maxblocks=None,
                       fields=("pcm", "windowed", "fft", "mdct_raw", "logfft", "logmdct", "noise", "tone",
                               "logmask", "mdct_m1", "ilogmask", "iwork_out"), timeline=False):
        """pcm: [ch][nsamples] float32.  One-shot: the handle is consumed."""
        pcm = np.ascontiguousarray(pcm, np.float32).reshape(self.channels, -1)
        ns = pcm.shape[1]
        if maxblocks is None:
            maxblocks = ns // (self.bs[0] // 2) + 8
        cap, arr = self._mkcap(maxblocks, fields)
        nbytes = C.c_long(0)
        tl = None
        if timeline:
            tl_cap = self.bs[1] // 2 + ns + 4 * self.bs[1]
            tl = np.zeros((self.channels, tl_cap), np.float32)
            self.L.ref_set_timeline(tl.ctypes.data, tl_cap)
        nb = self.L.ref_encode_capture(self.h, pcm, ns, C.byref(cap), C.byref(nbytes))
        k = min(nb, maxblocks)
        out = {name: a[:k] for name, a in arr.items()}
        out["nblocks"] = nb
        out["bytes"] = nbytes.value
        if timeline:
            ln, eof = C.c_long(0), C.c_long(0)
            self.L.ref_get_timeline(C.byref(ln), C.byref(eof))
            out["timeline"] = tl[:, :ln.value].copy()      # v->pcm in absolute samples (preamble, input, EOF tail)
            out["eof"] = eof.value
        return out

    def decode_capture(self, maxblocks, pcm_cap, fields=("dec_coef", "dec_imdct")):
        cap, arr = self._mkcap(maxblocks, fields)
        pcm = np.zeros((self.channels, pcm_cap), np.float32)
        Wseq = np.zeros(maxblocks, np.int32)
        got = self.L.ref_decode_capture(self.h, C.byref(cap), pcm, pcm_cap, Wseq.ctypes.data)
        if got < 0:
            raise RuntimeError("reference decode failed")
        k = cap.nblocks
        out = {name: arr[name][:k] for name in fields}
        out["W"] = Wseq[:k]
        out["pcm"] = pcm[:, :got]
        return out

    def blockin_sequence(self, Wseq, imdct, pcm_cap):
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        imdct = np.ascontiguousarray(imdct, np.float32)
        Nmax = imdct.shape[-1]
        pcm = np.zeros((self.channels, pcm_cap), np.float32)
        got = self.L.ref_blockin_sequence(self.h, len(Wseq), Wseq, imdct, Nmax, pcm, pcm_cap)
        if got < 0:
            raise RuntimeError("ref_blockin_sequence failed")
        return pcm[:, :got]
