"""ctypes loader for oracle/libvb_oracle.so — our own plain-C restatement of the path.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline leg; never by the product package.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from vorbis_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libvb_oracle.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")


def build(force=False):
    subprocess.check_call(["make", "-s"] + (["-B"] if force else []) + ["-C", HERE, "libvb_oracle.so", "CC=gcc"])


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        L.vbo_create.restype = C.c_void_p
        L.vbo_create.argtypes = [C.POINTER(abi.Setup)]
        L.vbo_destroy.argtypes = [C.c_void_p]
        L.vbo_table.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
        L.vbo_mdct_forward.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p]
        L.vbo_mdct_backward.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p]
        L.vbo_apply_window.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, f32p]
        L.vbo_drft_forward.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p]
        L.vbo_noisemask.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p]
        L.vbo_tonemask.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p, f32p, f32p, f32p]
        L.vbo_offset_and_mix.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, f32p, f32p, f32p, f32p, f32p]
        L.vbo_phaseA.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(abi.PhaseAIO)]
        L.vbo_phaseA_streams.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(abi.PhaseAIO), C.c_void_p]
        L.vbo_ampmax_decay.restype = C.c_float
        L.vbo_ampmax_decay.argtypes = [C.c_void_p, C.c_float, C.c_int]
        L.vbo_couple_quantize_normalize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    f32p, i32p, i32p]
        L.vbo_synthesis.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i64p, f32p, i64p, f32p, C.c_int64]
        L.vbo_decouple.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p]
        L.vbo_floor1_fit.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, f32p, f32p, i32p, i32p]
        L.vbo_floor1_render.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, i32p, i32p, i32p, i32p]
        L.vbo_floor1_inverse2.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, i32p, i32p, f32p]
        L.vbo_decode_dsp.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i64p, f32p, i32p, i32p, i64p, f32p, C.c_int64]
        L.vbo_residue_partvals.argtypes = [C.c_void_p, C.c_int]
        L.vbo_residue_classify.argtypes = [C.c_void_p, C.c_int, C.c_int, i32p, i32p, i32p, C.c_int]
        L.vbo_envelope_search.argtypes = [C.c_void_p, C.c_int, f32p, C.c_int64, C.c_int, C.c_int, i32p, u8p]
        L.vbo_envelope_apply_marks.argtypes = [u8p, C.c_int, C.c_int, i32p]
        L.vbo_plan_blocks.argtypes = [C.c_void_p, C.c_int, i32p, C.c_int64, C.c_int, i64p, C.c_void_p, C.c_int,
                                      C.c_void_p, i32p]
        _lib = L
    return _lib


class Oracle:
    def __init__(self, setup):
        """setup: abi.SetupHolder"""
        self.L = lib()
        self.setup = setup
        self.h = self.L.vbo_create(C.byref(setup.c))
        self.channels = setup.channels
        self.bs = [setup.blocksize(0), setup.blocksize(1)]

    def close(self):
        if self.h:
            self.L.vbo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def table(self, W, which):
        N = self.bs[W]
        out = np.zeros(N // 4, np.int32) if which == 1 else np.zeros(2 * N, np.float32)
        k = self.L.vbo_table(self.h, W, which, out.ctypes.data, out.size)
        assert k > 0
        return out[:k].copy()

    def mdct_forward(self, W, x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1, self.bs[W])
        out = np.empty((x.shape[0], self.bs[W] // 2), np.float32)
        self.L.vbo_mdct_forward(self.h, W, x.shape[0], x, out)
        return out

    def mdct_backward(self, W, x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1, self.bs[W] // 2)
        out = np.empty((x.shape[0], self.bs[W]), np.float32)
        self.L.vbo_mdct_backward(self.h, W, x.shape[0], x, out)
        return out

    def apply_window(self, W, x, lW=None, nW=None):
        x = np.array(x, np.float32).reshape(-1, self.bs[W])
        lWa = None if lW is None else np.ascontiguousarray(lW, np.int32)
        nWa = None if nW is None else np.ascontiguousarray(nW, np.int32)
        self.L.vbo_apply_window(self.h, W, x.shape[0],
                                None if lWa is None else lWa.ctypes.data,
                                None if nWa is None else nWa.ctypes.data, x)
        return x

    def drft_forward(self, W, x):
        x = np.array(x, np.float32).reshape(-1, self.bs[W])
        self.L.vbo_drft_forward(self.h, W, x.shape[0], x)
        return x

    def noisemask(self, look, logmdct):
        x = np.ascontiguousarray(logmdct, np.float32)
        x = x.reshape(-1, x.shape[-1])
        out = np.empty_like(x)
        self.L.vbo_noisemask(self.h, look, x.shape[0], x, out)
        return out

    def tonemask(self, look, logfft, gmax, lmax):
        x = np.ascontiguousarray(logfft, np.float32)
        x = x.reshape(-1, x.shape[-1])
        out = np.empty_like(x)
        g = np.ascontiguousarray(np.broadcast_to(np.asarray(gmax, np.float32), (x.shape[0],)))
        l = np.ascontiguousarray(np.broadcast_to(np.asarray(lmax, np.float32), (x.shape[0],)))
        self.L.vbo_tonemask(self.h, look, x.shape[0], x, g, l, out)
        return out

    def offset_and_mix(self, look, sel, noise, tone, mdct, logmdct):
        noise = np.ascontiguousarray(noise, np.float32)
        noise = noise.reshape(-1, noise.shape[-1])
        tone = np.ascontiguousarray(tone, np.float32).reshape(noise.shape)
        mdct = np.array(mdct, np.float32).reshape(noise.shape)
        logmdct = np.ascontiguousarray(logmdct, np.float32).reshape(noise.shape)
        logmask = np.empty_like(noise)
        self.L.vbo_offset_and_mix(self.h, look, noise.shape[0], sel, noise, tone, mdct, logmdct, logmask)
        return logmask, mdct

    def phaseA(self, W, pcm, desc, taps=False, streams=None, ampmax0=None):
        """pcm [nb][ch][N]; desc structured array (abi.BLOCKDESC_DTYPE).
        streams=(nstreams, blocks_per_stream) selects the ampmax-chain mode."""
        ch, N = self.channels, self.bs[W]
        pcm = np.ascontiguousarray(pcm, np.float32).reshape(-1, ch, N)
        nb = pcm.shape[0]
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        out = {k: np.empty((nb, ch, N // 2), np.float32) for k in ("mdct", "logmdct", "logmask")}
        out["ampmax_out"] = np.empty(nb, np.float32)
        io = abi.PhaseAIO()
        io.pcm, io.desc = pcm.ctypes.data, desc.ctypes.data
        io.mdct, io.logmdct, io.logmask = (out[k].ctypes.data for k in ("mdct", "logmdct", "logmask"))
        io.ampmax_out = out["ampmax_out"].ctypes.data
        if taps:
            for k in ("noise", "tone", "logfft", "mdct_raw"):
                out[k] = np.empty((nb, ch, N // 2), np.float32)
                setattr(io, "tap_" + k, out[k].ctypes.data)
        if streams is None:
            self.L.vbo_phaseA(self.h, W, nb, C.byref(io))
        else:
            a0 = None if ampmax0 is None else np.ascontiguousarray(ampmax0, np.float32)
            self.L.vbo_phaseA_streams(self.h, W, streams[0], streams[1], C.byref(io),
                                      None if a0 is None else a0.ctypes.data)
        return out

    def ampmax_decay(self, amp, W):
        return float(self.L.vbo_ampmax_decay(self.h, float(amp), W))

    def couple_quantize_normalize(self, W, blocktype, blobno, mdct, iwork, nonzero):
        mdct = np.ascontiguousarray(mdct, np.float32)
        iwork = np.array(iwork, np.int32)
        nonzero = np.array(nonzero, np.int32)
        self.L.vbo_couple_quantize_normalize(self.h, W, blocktype, blobno, mdct.shape[0], mdct, iwork, nonzero)
        return iwork, nonzero

    def floor1_fit(self, W, logmdct, logmask, floor_sel=-1):
        """[rows][n] x2 -> (posts [rows][FLOOR1_STRIDE], fit_nonzero [rows])"""
        n = self.bs[W] // 2
        a = np.ascontiguousarray(logmdct, np.float32).reshape(-1, n)
        b = np.ascontiguousarray(logmask, np.float32).reshape(-1, n)
        posts = np.zeros((a.shape[0], abi.FLOOR1_STRIDE), np.int32)
        nz = np.zeros(a.shape[0], np.int32)
        self.L.vbo_floor1_fit(self.h, W, floor_sel, a.shape[0], a, b, posts, nz)
        return posts, nz

    def floor1_render(self, W, posts, fit_nonzero, floor_sel=-1):
        n = self.bs[W] // 2
        posts = np.array(posts, np.int32).reshape(-1, abi.FLOOR1_STRIDE)
        fz = np.ascontiguousarray(fit_nonzero, np.int32)
        ilog = np.zeros((posts.shape[0], n), np.int32)
        nz = np.zeros(posts.shape[0], np.int32)
        self.L.vbo_floor1_render(self.h, W, floor_sel, posts.shape[0], posts, fz, ilog, nz)
        return posts, ilog, nz

    def encode_dsp(self, W, pcm, desc, streams=None, ampmax0=None, blobno=7):
        """The chain of mapping0_forward (lib/mapping0.c:230-646) composed from the stage oracles:
        Phase A -> floor1_fit -> floor render -> couple/quantise/normalise with each block's own
        psy look (blocktype).  pcm [nb][ch][N] block layout."""
        ch, n = self.channels, self.bs[W] // 2
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        a = self.phaseA(W, pcm, desc, streams=streams, ampmax0=ampmax0)
        nb = desc.shape[0]
        posts, fz = self.floor1_fit(W, a["logmdct"], a["logmask"])
        posts, ilog, nz = self.floor1_render(W, posts, fz)
        iwork = ilog.reshape(nb, ch, n).copy()
        nonzero = nz.reshape(nb, ch).copy()
        for bt in (0, 1):
            sel = np.where(desc["blocktype"] == bt)[0]
            if len(sel):
                iw, z = self.couple_quantize_normalize(W, bt, blobno, a["mdct"][sel], iwork[sel], nonzero[sel])
                iwork[sel], nonzero[sel] = iw, z
        a.update(posts=posts.reshape(nb, ch, -1), iwork=iwork, nonzero=nonzero)
        return a

    def floor1_interpolate_fit(self, A, B, del_):
        """floor1_interpolate_fit (lib/floor1.c:731-757) on rows of posts (padding entries are 0 and stay 0)"""
        A = np.asarray(A, np.int64); B = np.asarray(B, np.int64)
        out = ((65536 - del_) * (A & 0x7fff) + del_ * (B & 0x7fff) + 32768) >> 16
        out |= np.where(((A & 0x8000) != 0) & ((B & 0x8000) != 0), 0x8000, 0)
        return out.astype(np.int32)

    def encode_dsp_managed(self, W, pcm, desc, streams=None, ampmax0=None):
        """Bitrate-managed mapping0_forward (lib/mapping0.c:507-573, 596-646) composed from the stage oracles:
        Phase A (mask select 1) -> middle fit; where it exists: masks 2 / 0 -> high / low fits; twelve interpolated
        curves (NULL where an end is NULL); then per curve k the floor render and couple/quantise/normalise with
        blob k's parameters.  Returns blob-major posts / nonzero / iwork like vb200_encode_dsp_managed."""
        ch, n = self.channels, self.bs[W] // 2
        NB, MID, S = abi.PACKETBLOBS, abi.PACKETBLOBS // 2, abi.FLOOR1_STRIDE
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        a = self.phaseA(W, pcm, desc, taps=True, streams=streams, ampmax0=ampmax0)
        nb = desc.shape[0]
        rows = nb * ch
        logmask = {1: a["logmask"]}
        for sel in (2, 0):
            lm = np.empty((nb, ch, n), np.float32)
            for bt in (0, 1):
                idx = np.where(desc["blocktype"] == bt)[0]
                if len(idx):
                    m, _ = self.offset_and_mix(bt + (2 if W else 0), sel, a["noise"][idx], a["tone"][idx],
                                               a["mdct"][idx], a["logmdct"][idx])
                    lm[idx] = m.reshape(len(idx), ch, n)
            logmask[sel] = lm
        posts = np.zeros((NB, rows, S), np.int32)
        present = np.zeros((NB, rows), np.int32)
        pm, fm = self.floor1_fit(W, a["logmdct"], logmask[1])
        ph, fh = self.floor1_fit(W, a["logmdct"], logmask[2])
        pl, fl = self.floor1_fit(W, a["logmdct"], logmask[0])
        mid = fm != 0
        lo = mid & (fl != 0)
        hi = mid & (fh != 0)
        posts[MID][mid] = pm[mid]; present[MID] = mid
        posts[0][lo] = pl[lo]; present[0] = lo
        posts[NB - 1][hi] = ph[hi]; present[NB - 1] = hi
        for k in range(1, MID):
            posts[k][lo] = self.floor1_interpolate_fit(posts[0][lo], posts[MID][lo], k * 65536 // MID)
            present[k] = lo
        for k in range(MID + 1, NB - 1):
            posts[k][hi] = self.floor1_interpolate_fit(posts[MID][hi], posts[NB - 1][hi], (k - MID) * 65536 // MID)
            present[k] = hi
        iwork = np.zeros((NB, nb, ch, n), np.int32)
        nonzero = np.zeros((NB, nb, ch), np.int32)
        out_posts = np.zeros((NB, nb, ch, S), np.int32)
        for k in range(NB):
            pk, ilog, nz = self.floor1_render(W, posts[k], present[k])
            iw = ilog.reshape(nb, ch, n).copy()
            z = nz.reshape(nb, ch).copy()
            for bt in (0, 1):
                idx = np.where(desc["blocktype"] == bt)[0]
                if len(idx):
                    iw2, z2 = self.couple_quantize_normalize(W, bt, k, a["mdct"][idx], iw[idx], z[idx])
                    iw[idx], z[idx] = iw2, z2
            iwork[k], nonzero[k], out_posts[k] = iw, z, pk.reshape(nb, ch, S)
        return {"posts": out_posts, "nonzero": nonzero, "iwork": iwork, "ampmax_out": a["ampmax_out"]}

    def residue_partvals(self, W):
        return int(self.L.vbo_residue_partvals(self.h, W))

    def residue_classify(self, W, iwork, nonzero, stride=None):
        ch, n = self.channels, self.bs[W] // 2
        iwork = np.ascontiguousarray(iwork, np.int32).reshape(-1, ch, n)
        nonzero = np.ascontiguousarray(nonzero, np.int32).reshape(-1, ch)
        stride = self.residue_partvals(W) if stride is None else stride
        classes = np.zeros((iwork.shape[0], ch, stride), np.int32)
        self.L.vbo_residue_classify(self.h, W, iwork.shape[0], iwork, nonzero, classes, stride)
        return classes

    def floor1_inverse2(self, W, posts, present, data, floor_sel=-1):
        n = self.bs[W] // 2
        posts = np.ascontiguousarray(posts, np.int32).reshape(-1, abi.FLOOR1_STRIDE)
        present = np.ascontiguousarray(present, np.int32).reshape(-1)
        data = np.array(data, np.float32).reshape(posts.shape[0], n)
        self.L.vbo_floor1_inverse2(self.h, W, floor_sel, posts.shape[0], posts, present, data)
        return data

    def decode_dsp(self, Wseq, coef_off, res, posts, present, pcm_off, pcm_stride):
        """de-couple + floor multiply + IMDCT + overlap-add (lib/mapping0.c:754-795, lib/block.c:767-823)"""
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        res = np.array(res, np.float32)
        posts = np.ascontiguousarray(posts, np.int32)
        present = np.ascontiguousarray(present, np.int32)
        pcm = np.zeros((ns, self.channels, pcm_stride), np.float32)
        self.L.vbo_decode_dsp(self.h, ns, nblk, Wseq, np.ascontiguousarray(coef_off, np.int64), res,
                              posts.reshape(-1), present.reshape(-1), np.ascontiguousarray(pcm_off, np.int64),
                              pcm, pcm_stride)
        return pcm

    def envelope_search(self, pcm, first_step, nsteps, state=None):
        """pcm planar float [streams][ch][stride]; returns (ret uint8 [streams][nsteps], state words)"""
        pcm = np.ascontiguousarray(pcm, np.float32)
        ns, ch, stride = pcm.shape
        assert ch == self.channels and 64 * (first_step + nsteps - 1) + 128 <= stride
        state = (np.zeros((ns, abi.ve_state_words(ch)), np.int32) if state is None
                 else np.array(state, np.int32).reshape(ns, abi.ve_state_words(ch)))
        ret = np.zeros((ns, nsteps), np.uint8)
        self.L.vbo_envelope_search(self.h, ns, pcm, stride, first_step, nsteps, state, ret)
        return ret, state

    def envelope_marks(self, ret, first_step=0, mark=None):
        """replay lib/envelope.c:254-264 for one stream's ret codes"""
        ret = np.ascontiguousarray(ret, np.uint8)
        if mark is None:
            mark = np.zeros(first_step + len(ret) + 2, np.int32)
        self.L.vbo_envelope_apply_marks(ret, first_step, len(ret), mark)
        return mark

    def plan_blocks(self, mark, nsteps, pcm_len, eof=None, max_blocks=None):
        """what vorbis_analysis_blockout decides per block (lib/block.c:534-689) from the timeline marks"""
        mark = np.ascontiguousarray(mark, np.int32)
        ns, stride = mark.shape
        pcm_len = np.ascontiguousarray(pcm_len, np.int64)
        eofp = None if eof is None else np.ascontiguousarray(eof, np.int64)
        if max_blocks is None:
            max_blocks = int(pcm_len.max()) // (self.bs[0] // 2) + 8
        plan = np.zeros((ns, max_blocks), abi.STREAM_BLOCK_DTYPE)
        nb = np.zeros(ns, np.int32)
        self.L.vbo_plan_blocks(self.h, ns, mark.reshape(-1), stride, int(nsteps), pcm_len,
                               None if eofp is None else eofp.ctypes.data, max_blocks, plan.ctypes.data, nb)
        return plan, nb

    def timeline_marks(self, timeline):
        """envelope marks of whole timelines [streams][ch][len]: (mark [streams][nsteps+4], nsteps)"""
        tl = np.ascontiguousarray(timeline, np.float32)
        nsteps = tl.shape[2] // 64 - 4
        ret, _ = self.envelope_search(tl, 0, nsteps)
        mark = np.zeros((tl.shape[0], nsteps + 4), np.int32)
        for s in range(tl.shape[0]):
            mark[s, :nsteps + 2] = self.envelope_marks(ret[s])
        return mark, nsteps

    def encode_stream(self, tl, pcm_len, eof=0, blobno=7):
        """The composition for ONE stream (what vorbis_analysis_blockout + mapping0_forward do per block):
        marks -> block plan -> every block in order through encode_dsp with the ampmax decay chain carried
        across block sizes (lib/block.c:626-628).  tl [ch][len] float32 timeline (see vb200_plan_blocks).
        Returns (plan[nblocks], [encode_dsp result per block])."""
        tl = np.ascontiguousarray(tl, np.float32)
        pcm_len = int(pcm_len)
        last = max(0, min(tl.shape[1] // 64 - 4, pcm_len // 64 - 4))   # steps the reference would have analysed
        mark = np.zeros((1, last + 4), np.int32)
        if last > 0:
            ret, _ = self.envelope_search(tl[None], 0, last)
            mark[0, :last + 2] = self.envelope_marks(ret[0])
        plan, nb = self.plan_blocks(mark, last, [pcm_len], [int(eof)])
        outs = []
        g, prev = -9999.0, -9999.0
        for k in range(int(nb[0])):
            b = plan[0, k]
            W = int(b["W"])
            N = self.bs[W]
            if prev > g:
                g = prev
            g = self.ampmax_decay(g, W)
            d = np.zeros(1, abi.BLOCKDESC_DTYPE)
            d["lW"], d["nW"], d["blocktype"], d["ampmax"] = b["lW"], b["nW"], b["blocktype"], g
            r = self.encode_dsp(W, tl[None, :, b["pos"]:b["pos"] + N], d, blobno=blobno)
            prev = float(r["ampmax_out"][0])
            outs.append(r)
        return plan[0, :int(nb[0])], outs

    def decouple(self, W, res):
        res = np.array(res, np.float32)
        self.L.vbo_decouple(self.h, W, res.shape[0], res)
        return res

    def synthesis(self, Wseq, coef_off, coef, pcm_off, pcm_stride):
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        coef_off = np.ascontiguousarray(coef_off, np.int64)
        pcm_off = np.ascontiguousarray(pcm_off, np.int64)
        coef = np.ascontiguousarray(coef, np.float32)
        pcm = np.zeros((ns, self.channels, pcm_stride), np.float32)
        self.L.vbo_synthesis(self.h, ns, nblk, Wseq, coef_off, coef, pcm_off, pcm, pcm_stride)
        return pcm
