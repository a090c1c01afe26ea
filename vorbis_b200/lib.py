"""ctypes binding of the product library libvorbis_b200.so (C ABI: include/vorbis_b200.h).

This module is plumbing for tests and bench.py: it only marshals numpy arrays / raw
device pointers into the C entry points.  There is NO CPU fallback: if the CUDA
library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os

import numpy as np

from . import abi

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libvorbis_b200.so")

PCM_F32_PLANAR = 1
PCM_S16_INTERLEAVED = 2
IWORK_S32 = 0
IWORK_S16 = 1

EXPORTS = [
    "vb200_ctx_create", "vb200_ctx_destroy", "vb200_device_count", "vb200_last_error",
    "vb200_ctx_table", "vb200_launch_count", "vb200_set_profiling", "vb200_phaseA_kernel_ms", "vb200_debug_phase_cycles",
    "vb200_encode_dsp_kernel_ms",
    "vb200_mdct_forward_dev", "vb200_mdct_forward", "vb200_mdct_backward_dev", "vb200_mdct_backward",
    "vb200_apply_window", "vb200_drft_forward",
    "vb200_noisemask", "vb200_tonemask", "vb200_offset_and_mix",
    "vb200_analysis_phaseA_dev", "vb200_analysis_phaseA", "vb200_analysis_phaseA_streams_dev",
    "vb200_analysis_phaseA_pcmstream_dev", "vb200_synthesis_s16_dev",
    "vb200_couple_quantize_normalize_dev", "vb200_couple_quantize_normalize",
    "vb200_synthesis_dev", "vb200_synthesis", "vb200_synthesis_halfrate", "vb200_decouple_dev", "vb200_decouple",
    "vb200_floor1_fit_dev", "vb200_floor1_fit", "vb200_floor1_render_dev", "vb200_floor1_render",
    "vb200_encode_dsp_dev", "vb200_encode_dsp", "vb200_encode_dsp_managed_dev", "vb200_encode_dsp_managed",
    "vb200_envelope_search_dev", "vb200_envelope_search", "vb200_envelope_search_var", "vb200_envelope_apply_marks",
    "vb200_floor1_inverse2_dev", "vb200_floor1_inverse2", "vb200_decode_dsp_dev", "vb200_decode_dsp",
    "vb200_decode_dsp_resume_dev", "vb200_decode_dsp_resume",
    "vb200_decode_entropy_setup", "vb200_decode_entropy_dev", "vb200_decode_entropy",
    "vb200_decode_packets_resume_dev", "vb200_decode_packets_resume",
    "vb200_decode_streams_carry_bytes", "vb200_decode_streams_carry_init", "vb200_decode_streams_packets_dev",
    "vb200_decode_streams_packets", "vb200_decode_streams_index_dev", "vb200_decode_streams_index",
    "vb200_decode_ranges_dev", "vb200_decode_ranges",
    "vb200_encode_entropy_setup", "vb200_encode_packet_bound", "vb200_encode_entropy_dev", "vb200_encode_entropy",
    "vb200_encode_packets", "vb200_encode_entropy_managed_dev", "vb200_encode_packets_managed",
    "vb200_residue_partvals", "vb200_residue_classify_dev", "vb200_residue_classify",
    "vb200_plan_blocks", "vb200_encode_streams_dev", "vb200_encode_streams",
    "vb200_encode_streams_managed_dev", "vb200_encode_streams_managed",
    "vb200_bitrate_setup", "vb200_bitrate_init", "vb200_bitrate_addblocks_dev", "vb200_bitrate_addblocks",
    "vb200_encode_streams_packets", "vb200_encode_streams_packets_managed",
    "vb200_encode_carry_bytes", "vb200_encode_carry_init", "vb200_encode_streams_packets_resume",
    "vb200_encode_streams_packets_managed_resume",
    "vb200_encode_pcm_carry_bytes", "vb200_encode_pcm_carry_init", "vb200_encode_pcm_packets",
    "vb200_encode_pcm_packets_managed", "vb200_encode_pcm_packets_dev", "vb200_encode_pcm_packets_managed_dev",
    "vb200_lpc_extrapolate",
    "vb200_ogg_demux_dev", "vb200_ogg_demux", "vb200_ogg_links_dev", "vb200_ogg_links", "vb200_vorbis_window",
    "vb200_vorbis_headers_parse", "vb200_vorbis_headers_free",
    "vb200_ogg_group_scratch_bytes", "vb200_ogg_group_dev", "vb200_ogg_group",
    "vb200_ogg_mux_dev", "vb200_ogg_mux", "vb200_ogg_ranges_dev", "vb200_ogg_ranges",
    "vb200_malloc_device", "vb200_free_device", "vb200_memcpy_h2d", "vb200_memcpy_d2h", "vb200_synchronize",
]

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
vp = C.c_void_p


class VB200Error(RuntimeError):
    pass


_lib = None


def load():
    """Load libvorbis_b200.so; raises if it has not been built (run __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VB200Error("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`"
                         % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.vb200_last_error.restype = C.c_char_p
    L.vb200_launch_count.restype = C.c_uint64
    L.vb200_launch_count.argtypes = [vp]
    L.vb200_set_profiling.argtypes = [vp, C.c_int]
    L.vb200_phaseA_kernel_ms.argtypes = [vp, C.POINTER(C.c_float * 3)]
    L.vb200_encode_dsp_kernel_ms.argtypes = [vp, C.POINTER(C.c_float * 6)]
    L.vb200_debug_phase_cycles.argtypes = [vp, C.POINTER(C.c_ulonglong * 16), C.c_int]
    L.vb200_ctx_create.argtypes = [C.POINTER(abi.Setup), C.c_int, C.POINTER(vp)]
    L.vb200_ctx_destroy.argtypes = [vp]
    L.vb200_ctx_table.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int]
    L.vb200_mdct_forward_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
    L.vb200_mdct_backward_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
    L.vb200_mdct_forward.argtypes = [vp, C.c_int, C.c_int, vp, vp]
    L.vb200_mdct_backward.argtypes = [vp, C.c_int, C.c_int, vp, vp]
    L.vb200_apply_window.argtypes = [vp, C.c_int, C.c_int, vp, vp, f32p]
    L.vb200_drft_forward.argtypes = [vp, C.c_int, C.c_int, f32p]
    L.vb200_noisemask.argtypes = [vp, C.c_int, C.c_int, f32p, f32p]
    L.vb200_tonemask.argtypes = [vp, C.c_int, C.c_int, f32p, f32p, f32p, f32p]
    L.vb200_offset_and_mix.argtypes = [vp, C.c_int, C.c_int, C.c_int, f32p, f32p, f32p, f32p, f32p]
    L.vb200_analysis_phaseA_dev.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.PhaseAIO), vp]
    L.vb200_analysis_phaseA.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.PhaseAIO)]
    L.vb200_analysis_phaseA_streams_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(abi.PhaseAIO), vp, vp]
    L.vb200_analysis_phaseA_pcmstream_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int64, C.c_int,
                                                      C.POINTER(abi.PhaseAIO), vp, vp]
    L.vb200_synthesis_s16_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_int64, vp]
    L.vb200_couple_quantize_normalize_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    L.vb200_couple_quantize_normalize.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.vb200_synthesis_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_int64, vp]
    L.vb200_synthesis.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int64, vp, vp, C.c_int64]
    L.vb200_synthesis_halfrate.argtypes = [vp, C.c_int, vp]
    L.vb200_decouple_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp]
    L.vb200_decouple.argtypes = [vp, C.c_int, C.c_int, vp]
    L.vb200_floor1_fit_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp]
    L.vb200_floor1_fit.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    L.vb200_floor1_render_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp]
    L.vb200_floor1_render.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    L.vb200_encode_dsp_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(abi.EncodeIO), vp]
    L.vb200_encode_dsp.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(abi.EncodeIO)]
    L.vb200_encode_dsp_managed.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(abi.EncodeIO)]
    L.vb200_encode_dsp_managed_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(abi.EncodeIO), vp]
    L.vb200_residue_partvals.argtypes = [vp, C.c_int]
    L.vb200_residue_classify_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp]
    L.vb200_residue_classify.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int]
    L.vb200_floor1_inverse2_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    L.vb200_floor1_inverse2.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.vb200_decode_dsp_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int64, vp]
    L.vb200_decode_dsp.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int64, vp, vp, vp, vp, C.c_int, C.c_int64]
    L.vb200_decode_dsp_resume_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int64,
                                              C.POINTER(abi.DecodeCarry), vp]
    L.vb200_decode_dsp_resume.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int64, vp, vp, vp, vp, C.c_int,
                                          C.c_int64, C.POINTER(abi.DecodeCarry)]
    L.vb200_decode_entropy_setup.argtypes = [vp, C.POINTER(abi.EntropySetup)]
    L.vb200_decode_entropy_dev.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.vb200_decode_entropy.argtypes = [vp, C.c_int, vp, vp, vp, vp, C.c_int64, vp, vp, C.c_int64, vp, vp]
    L.vb200_decode_packets_resume_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int,
                                                  C.c_int64, C.POINTER(abi.DecodeCarry), vp]
    L.vb200_decode_packets_resume.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int64, vp, vp, vp, C.c_int64, vp,
                                              vp, C.c_int, C.c_int64, C.POINTER(abi.DecodeCarry)]
    L.vb200_decode_streams_carry_bytes.argtypes = [vp]
    L.vb200_decode_streams_carry_init.argtypes = [vp, C.c_int, vp]
    L.vb200_decode_streams_packets_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, vp, C.c_int64, vp,
                                                   vp, vp]
    L.vb200_decode_streams_packets.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int64, vp, C.c_int, vp,
                                               C.c_int64, vp, vp]
    L.vb200_decode_streams_index_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
    L.vb200_decode_streams_index.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int64, vp, vp]
    L.vb200_decode_ranges_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, C.c_int, vp, C.c_int32, vp,
                                          vp]
    L.vb200_decode_ranges.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int64, C.c_int, vp, C.c_int, vp,
                                      C.c_int32, vp]
    L.vb200_encode_entropy_setup.argtypes = [vp, C.POINTER(abi.EncodeEntropySetup)]
    L.vb200_encode_packet_bound.argtypes = [vp, C.c_int]
    L.vb200_encode_entropy_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int64, vp, vp, vp]
    L.vb200_encode_entropy.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_int64]
    L.vb200_encode_packets.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(abi.EncodeIO), vp, vp, vp,
                                       C.c_int64]
    L.vb200_encode_entropy_managed_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_int64, vp, vp,
                                                   vp]
    L.vb200_encode_packets_managed.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(abi.EncodeIO), vp, vp, vp,
                                               C.c_int64]
    L.vb200_envelope_search_dev.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int64, C.c_int, C.c_int, vp, vp, vp]
    L.vb200_envelope_search.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int64, C.c_int, C.c_int, vp, vp]
    L.vb200_envelope_apply_marks.argtypes = [vp, C.c_int, C.c_int, vp]
    L.vb200_envelope_apply_marks.restype = None
    L.vb200_plan_blocks.argtypes = [vp, C.c_int, vp, C.c_int64, C.c_int, vp, vp, C.c_int, vp, vp]
    L.vb200_encode_streams.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.StreamsIO)]
    L.vb200_encode_streams_dev.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.StreamsIO), vp]
    L.vb200_encode_streams_managed.argtypes = [vp, C.c_int, C.POINTER(abi.StreamsIO)]
    L.vb200_encode_streams_managed_dev.argtypes = [vp, C.c_int, C.POINTER(abi.StreamsIO), vp]
    L.vb200_bitrate_setup.argtypes = [vp, C.POINTER(abi.BitrateInfo)]
    L.vb200_bitrate_init.argtypes = [vp, vp]
    L.vb200_bitrate_addblocks_dev.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.vb200_bitrate_addblocks.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
    L.vb200_encode_streams_packets.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.StreamsIO), vp, vp, C.c_int64]
    L.vb200_encode_streams_packets_managed.argtypes = [vp, C.c_int, C.POINTER(abi.StreamsIO), vp, vp, C.c_int64]
    L.vb200_encode_carry_bytes.argtypes = [vp, C.c_int]
    L.vb200_encode_carry_init.argtypes = [vp, C.c_int, C.c_int, vp]
    L.vb200_encode_streams_packets_resume.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.StreamsIO), vp, vp, vp,
                                                      C.c_int64]
    L.vb200_encode_streams_packets_managed_resume.argtypes = [vp, C.c_int, C.POINTER(abi.StreamsIO), vp, vp, vp,
                                                              C.c_int64]
    L.vb200_encode_pcm_carry_bytes.argtypes = [vp, C.c_int]
    L.vb200_encode_pcm_carry_init.argtypes = [vp, C.c_int, C.c_int, vp]
    L.vb200_encode_pcm_packets.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.PcmIO), vp, vp, vp, C.c_int64]
    L.vb200_encode_pcm_packets_managed.argtypes = [vp, C.c_int, C.POINTER(abi.PcmIO), vp, vp, vp, C.c_int64]
    L.vb200_encode_pcm_packets_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(abi.PcmIO), vp, vp, vp, vp,
                                               C.c_int64, vp, vp, vp]
    L.vb200_encode_pcm_packets_managed_dev.argtypes = [vp, C.c_int, C.c_int, C.POINTER(abi.PcmIO), vp, vp, vp, vp,
                                                       C.c_int64, vp, vp, vp]
    L.vb200_lpc_extrapolate.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int64, vp, C.c_int32, vp, vp, C.c_int64]
    L.vb200_ogg_demux_dev.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    L.vb200_ogg_demux.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp, vp]
    L.vb200_ogg_links_dev.argtypes = [C.c_int, vp, vp, vp, vp, C.c_int64, vp]
    L.vb200_ogg_links.argtypes = [C.c_int, vp, vp, vp, vp, C.c_int64]
    L.vb200_vorbis_window.argtypes = [C.c_int, vp]
    L.vb200_vorbis_headers_parse.argtypes = [vp, C.c_int32, vp, C.c_int32, vp, C.c_int32,
                                             C.POINTER(C.POINTER(abi.VorbisHeaders))]
    L.vb200_vorbis_headers_free.argtypes = [C.POINTER(abi.VorbisHeaders)]
    L.vb200_vorbis_headers_free.restype = None
    L.vb200_ogg_group_scratch_bytes.argtypes = [C.c_int, C.c_int]
    L.vb200_ogg_group_scratch_bytes.restype = C.c_size_t
    L.vb200_ogg_group_dev.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.vb200_ogg_group.argtypes = [C.c_int, vp, C.c_int64, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.vb200_ogg_mux_dev.argtypes = [C.c_int, vp, C.c_int64, vp, C.c_int, vp, vp, vp, vp, C.c_int64, vp, vp, vp]
    L.vb200_ogg_mux.argtypes = [C.c_int, vp, C.c_int64, vp, C.c_int, vp, vp, vp, vp, C.c_int64, vp, vp]
    L.vb200_ogg_ranges_dev.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, vp, C.c_int32, C.c_int64, vp, vp]
    L.vb200_ogg_ranges.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, vp, C.c_int32, C.c_int64, vp]
    L.vb200_malloc_device.argtypes = [vp, C.c_size_t, C.POINTER(vp)]
    L.vb200_free_device.argtypes = [vp, vp]
    L.vb200_memcpy_h2d.argtypes = [vp, vp, vp, C.c_size_t]
    L.vb200_memcpy_d2h.argtypes = [vp, vp, vp, C.c_size_t]
    L.vb200_synchronize.argtypes = [vp]
    _lib = L
    return L


def _ptr(a):
    """numpy array / int (device pointer) / None -> c_void_p value"""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return int(a)


class Context:
    """One vb200_ctx: device tables for a (channels, rate, quality) setup on one GPU."""

    def __init__(self, setup, device=0):
        self.L = load()
        self.setup = setup
        self.channels = setup.channels
        self.bs = [setup.blocksize(0), setup.blocksize(1)]
        h = vp()
        self._chk(self.L.vb200_ctx_create(C.byref(setup.c), device, C.byref(h)))
        self.h = h
        self.halfrate = 0

    @classmethod
    def wrap(cls, handle, channels, blocksizes):
        """a Context on a vb200_ctx created elsewhere (e.g. by the decode driver), which keeps owning it"""
        self = cls.__new__(cls)
        self.L = load()
        self.setup = None
        self.h = vp(handle)
        self.halfrate = 0
        self.channels, self.bs = channels, list(blocksizes)
        return self

    def close(self):
        if getattr(self, "h", None) and self.setup is not None:
            self.L.vb200_ctx_destroy(self.h)
        self.h = None

    def _chk(self, rc):
        if rc != 0:
            raise VB200Error("vb200 error %d: %s" % (rc, (self.L.vb200_last_error() or b"").decode()))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def launch_count(self):
        return int(self.L.vb200_launch_count(self.h))

    def set_profiling(self, on=True):
        self._chk(self.L.vb200_set_profiling(self.h, 1 if on else 0))

    def phaseA_kernel_ms(self):
        ms = (C.c_float * 3)()
        self._chk(self.L.vb200_phaseA_kernel_ms(self.h, C.byref(ms)))
        return [float(x) for x in ms]

    def encode_dsp_kernel_ms(self):
        ms = (C.c_float * 6)()
        self._chk(self.L.vb200_encode_dsp_kernel_ms(self.h, C.byref(ms)))
        return list(ms)

    def debug_phase_cycles(self, reset=True):
        out = (C.c_ulonglong * 16)()
        self._chk(self.L.vb200_debug_phase_cycles(self.h, C.byref(out), 1 if reset else 0))
        return [int(x) for x in out]

    def table(self, W, which):
        N = self.bs[W]
        out = np.zeros(N // 4, np.int32) if which == 1 else np.zeros(2 * N, np.float32)
        k = self.L.vb200_ctx_table(self.h, W, which, out.ctypes.data, out.size)
        if k <= 0:
            raise VB200Error("vb200_ctx_table failed")
        return out[:k].copy()

    # ---- transforms: host buffers -------------------------------------------
    def mdct_forward(self, W, x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1, self.bs[W])
        out = np.empty((x.shape[0], self.bs[W] // 2), np.float32)
        self._chk(self.L.vb200_mdct_forward(self.h, W, x.shape[0], _ptr(x), _ptr(out)))
        return out

    def mdct_backward(self, W, x):
        """in half-rate mode the transform of size blocksizes[W]/2"""
        N = self.bs[W] >> self.halfrate
        x = np.ascontiguousarray(x, np.float32).reshape(-1, N // 2)
        out = np.empty((x.shape[0], N), np.float32)
        self._chk(self.L.vb200_mdct_backward(self.h, W, x.shape[0], _ptr(x), _ptr(out)))
        return out

    def apply_window(self, W, x, lW=None, nW=None):
        x = np.array(x, np.float32).reshape(-1, self.bs[W])
        lWa = None if lW is None else np.ascontiguousarray(lW, np.int32)
        nWa = None if nW is None else np.ascontiguousarray(nW, np.int32)
        self._chk(self.L.vb200_apply_window(self.h, W, x.shape[0], _ptr(lWa), _ptr(nWa), x))
        return x

    def drft_forward(self, W, x):
        x = np.array(x, np.float32).reshape(-1, self.bs[W])
        self._chk(self.L.vb200_drft_forward(self.h, W, x.shape[0], x))
        return x

    # ---- transforms: device pointers ----------------------------------------
    def mdct_forward_dev(self, W, nvec, d_in, d_out, stream=None):
        self._chk(self.L.vb200_mdct_forward_dev(self.h, W, nvec, _ptr(d_in), _ptr(d_out), _ptr(stream)))

    def mdct_backward_dev(self, W, nvec, d_in, d_out, stream=None):
        self._chk(self.L.vb200_mdct_backward_dev(self.h, W, nvec, _ptr(d_in), _ptr(d_out), _ptr(stream)))

    # ---- psy stages -----------------------------------------------------------
    def noisemask(self, look, logmdct):
        x = np.ascontiguousarray(logmdct, np.float32)
        x = x.reshape(-1, x.shape[-1])
        out = np.empty_like(x)
        self._chk(self.L.vb200_noisemask(self.h, look, x.shape[0], x, out))
        return out

    def tonemask(self, look, logfft, gmax, lmax):
        x = np.ascontiguousarray(logfft, np.float32)
        x = x.reshape(-1, x.shape[-1])
        out = np.empty_like(x)
        g = np.ascontiguousarray(np.broadcast_to(np.asarray(gmax, np.float32), (x.shape[0],)))
        l = np.ascontiguousarray(np.broadcast_to(np.asarray(lmax, np.float32), (x.shape[0],)))
        self._chk(self.L.vb200_tonemask(self.h, look, x.shape[0], x, g, l, out))
        return out

    def offset_and_mix(self, look, sel, noise, tone, mdct, logmdct):
        noise = np.ascontiguousarray(noise, np.float32)
        noise = noise.reshape(-1, noise.shape[-1])
        tone = np.ascontiguousarray(tone, np.float32).reshape(noise.shape)
        mdct = np.array(mdct, np.float32).reshape(noise.shape)
        logmdct = np.ascontiguousarray(logmdct, np.float32).reshape(noise.shape)
        logmask = np.empty_like(noise)
        self._chk(self.L.vb200_offset_and_mix(self.h, look, noise.shape[0], sel, noise, tone, mdct,
                                              logmdct, logmask))
        return logmask, mdct

    # ---- Phase A ---------------------------------------------------------------
    def phaseA(self, W, pcm, desc, taps=False):
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
        self._chk(self.L.vb200_analysis_phaseA(self.h, W, nb, C.byref(io)))
        return out

    def phaseA_dev(self, W, nblocks, io, stream=None, streams=None, d_ampmax0=None):
        """io: abi.PhaseAIO holding DEVICE pointers."""
        if streams is None:
            self._chk(self.L.vb200_analysis_phaseA_dev(self.h, W, nblocks, C.byref(io), _ptr(stream)))
        else:
            self._chk(self.L.vb200_analysis_phaseA_streams_dev(self.h, W, streams[0], streams[1], C.byref(io),
                                                               _ptr(d_ampmax0), _ptr(stream)))

    def phaseA_pcmstream_dev(self, W, nstreams, bps, d_pcm, fmt, stream_stride, hop, io, d_ampmax0=None, stream=None):
        self._chk(self.L.vb200_analysis_phaseA_pcmstream_dev(self.h, W, nstreams, bps, _ptr(d_pcm), fmt, stream_stride,
                                                             hop, C.byref(io), _ptr(d_ampmax0), _ptr(stream)))

    def synthesis_s16_dev(self, nstreams, nblk, d_Wseq, d_coef_off, d_coef, d_pcm_off, d_pcm16, pcm_stride, stream=None):
        self._chk(self.L.vb200_synthesis_s16_dev(self.h, nstreams, nblk, _ptr(d_Wseq), _ptr(d_coef_off), _ptr(d_coef),
                                                 _ptr(d_pcm_off), _ptr(d_pcm16), pcm_stride, _ptr(stream)))

    # ---- Phase B ---------------------------------------------------------------
    def couple_quantize_normalize(self, W, blocktype, blobno, mdct, iwork, nonzero):
        mdct = np.ascontiguousarray(mdct, np.float32)
        iwork = np.array(iwork, np.int32)
        nonzero = np.array(nonzero, np.int32)
        self._chk(self.L.vb200_couple_quantize_normalize(self.h, W, blocktype, blobno, mdct.shape[0],
                                                         _ptr(mdct), _ptr(iwork), _ptr(nonzero)))
        return iwork, nonzero

    def couple_quantize_normalize_dev(self, W, blocktype, blobno, nblocks, d_mdct, d_iwork, d_nonzero, stream=None):
        self._chk(self.L.vb200_couple_quantize_normalize_dev(self.h, W, blocktype, blobno, nblocks,
                                                             _ptr(d_mdct), _ptr(d_iwork), _ptr(d_nonzero),
                                                             _ptr(stream)))

    # ---- floor 1 (lib/floor1.c:576 floor1_fit, :765 floor1_encode minus the bit packing) -------
    def floor1_fit(self, W, logmdct, logmask, floor_sel=-1):
        """logmdct, logmask [rows][n] -> (posts [rows][FLOOR1_STRIDE] int32, fit_nonzero [rows])"""
        n = self.bs[W] // 2
        a = np.ascontiguousarray(logmdct, np.float32).reshape(-1, n)
        b = np.ascontiguousarray(logmask, np.float32).reshape(-1, n)
        posts = np.zeros((a.shape[0], abi.FLOOR1_STRIDE), np.int32)
        nz = np.zeros(a.shape[0], np.int32)
        self._chk(self.L.vb200_floor1_fit(self.h, W, floor_sel, a.shape[0], _ptr(a), _ptr(b), _ptr(posts), _ptr(nz)))
        return posts, nz

    def floor1_render(self, W, posts, fit_nonzero, floor_sel=-1):
        """posts from floor1_fit -> (posts as floor1_encode leaves them, ilogmask [rows][n], nonzero)"""
        n = self.bs[W] // 2
        posts = np.array(posts, np.int32).reshape(-1, abi.FLOOR1_STRIDE)
        fz = np.ascontiguousarray(fit_nonzero, np.int32)
        ilog = np.zeros((posts.shape[0], n), np.int32)
        nz = np.zeros(posts.shape[0], np.int32)
        self._chk(self.L.vb200_floor1_render(self.h, W, floor_sel, posts.shape[0], _ptr(posts), _ptr(fz),
                                             _ptr(ilog), _ptr(nz)))
        return posts, ilog, nz

    def floor1_fit_dev(self, W, nrows, d_logmdct, d_logmask, d_posts, d_fit_nonzero, floor_sel=-1, stream=None):
        self._chk(self.L.vb200_floor1_fit_dev(self.h, W, floor_sel, nrows, _ptr(d_logmdct), _ptr(d_logmask),
                                              _ptr(d_posts), _ptr(d_fit_nonzero), _ptr(stream)))

    def floor1_render_dev(self, W, nrows, d_posts, d_fit_nonzero, d_ilogmask, d_nonzero, floor_sel=-1, stream=None):
        self._chk(self.L.vb200_floor1_render_dev(self.h, W, floor_sel, nrows, _ptr(d_posts), _ptr(d_fit_nonzero),
                                                 _ptr(d_ilogmask), _ptr(d_nonzero), _ptr(stream)))

    # ---- whole streams: envelope marks -> block plan -> both block sizes, ampmax chain across sizes ----
    def plan_blocks(self, mark, nsteps, pcm_len, eof=None, max_blocks=None):
        """mark [streams][stride] int32 (timeline steps), pcm_len/eof [streams] int64 -> (plan, nblocks)"""
        mark = np.ascontiguousarray(mark, np.int32)
        ns, stride = mark.shape
        pcm_len = np.ascontiguousarray(pcm_len, np.int64)
        eofp = None if eof is None else np.ascontiguousarray(eof, np.int64)
        if max_blocks is None:
            max_blocks = int(pcm_len.max()) // (self.bs[0] // 2) + 8
        plan = np.zeros((ns, max_blocks), abi.STREAM_BLOCK_DTYPE)
        nb = np.zeros(ns, np.int32)
        self._chk(self.L.vb200_plan_blocks(self.h, ns, mark.ctypes.data, stride, int(nsteps), pcm_len.ctypes.data,
                                        None if eofp is None else eofp.ctypes.data, max_blocks, plan.ctypes.data,
                                        nb.ctypes.data))
        return plan, nb

    def encode_streams(self, pcm, pcm_len, eof=None, fmt=PCM_F32_PLANAR, max_blocks=None, cap=None, blobno=7):
        """pcm: timeline buffers, PCM_F32_PLANAR [streams][ch][stride] float32 or PCM_S16_INTERLEAVED
        [streams][stride][ch] int16.  Returns plan, nblocks and per block size W the batch outputs."""
        return self._encode_streams(pcm, pcm_len, eof, fmt, max_blocks, cap, blobno, None)

    def encode_streams_managed(self, pcm, pcm_len, eof=None, fmt=PCM_F32_PLANAR, max_blocks=None, cap=None):
        """Bitrate-managed vb200_encode_streams_managed: inputs and result as encode_streams, with the per-size
        posts / nonzero / iwork shaped [15][count][ch][...] (curve k = blob k); ampmax_out [count]."""
        return self._encode_streams(pcm, pcm_len, eof, fmt, max_blocks, cap, 0, abi.PACKETBLOBS)

    def _streams_io(self, pcm, pcm_len, eof, fmt, max_blocks, cap):
        """the inputs of the whole-stream encode calls as an abi.StreamsIO, max_blocks and cap defaulting to what the
        timelines can hold: (io, plan, nblocks, the arrays io points into, to be kept alive until the call returns)"""
        ch = self.channels
        if fmt == PCM_F32_PLANAR:
            pcm = np.ascontiguousarray(pcm, np.float32)
            ns, stride = pcm.shape[0], pcm.shape[2]
            assert pcm.shape[1] == ch
        else:
            pcm = np.ascontiguousarray(pcm, np.int16)
            ns, stride = pcm.shape[0], pcm.shape[1]
            assert pcm.shape[2] == ch
        pcm_len = np.ascontiguousarray(pcm_len, np.int64)
        eofp = None if eof is None else np.ascontiguousarray(eof, np.int64)
        if max_blocks is None:
            max_blocks = stride // (self.bs[0] // 2) + 8
        if cap is None:
            cap = [ns * max_blocks, ns * (stride // (self.bs[1] // 2) + 8)]
        io = abi.StreamsIO()
        io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = pcm.ctypes.data, fmt, max_blocks, stride
        io.pcm_len = pcm_len.ctypes.data
        io.eof = None if eofp is None else eofp.ctypes.data
        plan = np.zeros((ns, max_blocks), abi.STREAM_BLOCK_DTYPE)
        nb = np.zeros(ns, np.int32)
        io.plan, io.nblocks = plan.ctypes.data, nb.ctypes.data
        io.cap[0], io.cap[1] = int(cap[0]), int(cap[1])
        return io, plan, nb, (pcm, pcm_len, eofp)

    def _encode_streams(self, pcm, pcm_len, eof, fmt, max_blocks, cap, blobno, curves):
        ch = self.channels
        io, plan, nb, keep = self._streams_io(pcm, pcm_len, eof, fmt, max_blocks, cap)
        out = {}
        lead = () if curves is None else (curves,)
        for w in range(2):
            n, cw = self.bs[w] // 2, io.cap[w]
            out[w] = {"posts": np.zeros(lead + (cw, ch, abi.FLOOR1_STRIDE), np.int32),
                      "nonzero": np.zeros(lead + (cw, ch), np.int32),
                      "iwork": np.zeros(lead + (cw, ch, n), np.int32), "ampmax_out": np.zeros(cw, np.float32)}
            io.posts[w], io.nonzero[w] = out[w]["posts"].ctypes.data, out[w]["nonzero"].ctypes.data
            io.iwork[w], io.ampmax_out[w] = out[w]["iwork"].ctypes.data, out[w]["ampmax_out"].ctypes.data
        ns = plan.shape[0]
        if curves is None:
            self._chk(self.L.vb200_encode_streams(self.h, ns, blobno, C.byref(io)))
        else:
            self._chk(self.L.vb200_encode_streams_managed(self.h, ns, C.byref(io)))
        for w in range(2):
            cnt = io.count[w]
            out[w] = {k: (v[:cnt] if k == "ampmax_out" or curves is None else v[:, :cnt]) for k, v in out[w].items()}
        return {"plan": plan, "nblocks": nb, "count": [io.count[0], io.count[1]], 0: out[0], 1: out[1]}

    # ---- whole per-block encode DSP (Phase A -> floor1 -> Phase B) in one call ---------------
    def _encode_io(self, W, pcm, desc, nstreams, fmt, hop, ampmax0, independent):
        """the inputs of the block-level encode calls as an abi.EncodeIO: (io, nstreams, blocks per stream, the arrays
        io points into, to be kept alive until the call returns)"""
        ch, N = self.channels, self.bs[W]
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        nb = desc.shape[0]
        if nstreams is None:
            nstreams = nb
            if independent is None:
                independent = True
        bps = nb // nstreams
        assert bps * nstreams == nb
        io = abi.EncodeIO()
        if fmt == 0:
            pcm = np.ascontiguousarray(pcm, np.float32).reshape(nb, ch, N)
        elif fmt == PCM_F32_PLANAR:
            pcm = np.ascontiguousarray(pcm, np.float32)
            assert pcm.shape[:2] == (nstreams, ch)
            io.stream_stride = pcm.shape[2]
        else:
            pcm = np.ascontiguousarray(pcm, np.int16)
            assert pcm.shape[0] == nstreams and pcm.shape[2] == ch
            io.stream_stride = pcm.shape[1]
        io.pcm, io.pcm_fmt, io.hop = pcm.ctypes.data, fmt, hop
        io.desc = desc.ctypes.data
        io.independent = 1 if independent else 0
        if ampmax0 is not None:
            ampmax0 = np.ascontiguousarray(ampmax0, np.float32)
            io.ampmax0 = ampmax0.ctypes.data
        return io, nstreams, bps, (pcm, desc, ampmax0)

    def encode_dsp(self, W, pcm, desc, nstreams=None, fmt=0, hop=0, ampmax0=None, independent=None, blobno=7,
                   floats=False, iwork_s16=False, classes=False):
        """Host buffers.  fmt 0: pcm [nblocks][ch][N] float; PCM_F32_PLANAR: [streams][ch][stride] float;
        PCM_S16_INTERLEAVED: [streams][stride][ch] int16.  nstreams None = every block its own stream.
        independent None = True when the blocks are not grouped in streams."""
        ch, n = self.channels, self.bs[W] // 2
        io, nstreams, bps, keep = self._encode_io(W, pcm, desc, nstreams, fmt, hop, ampmax0, independent)
        nb = nstreams * bps
        out = {"posts": np.zeros((nb, ch, abi.FLOOR1_STRIDE), np.int32), "nonzero": np.zeros((nb, ch), np.int32),
               "iwork": np.zeros((nb, ch, n), np.int16 if iwork_s16 else np.int32),
               "ampmax_out": np.zeros(nb, np.float32)}
        if iwork_s16:
            io.iwork_fmt = IWORK_S16
            out["overflow"] = np.full(nb, -1, np.int32)
        if classes:
            io.class_stride = self.residue_partvals(W)
            out["classes"] = np.full((nb, ch, int(io.class_stride)), -1, np.int32)
        if floats:
            for k in ("mdct", "logmdct", "logmask"):
                out[k] = np.zeros((nb, ch, n), np.float32)
        for k, v in out.items():
            setattr(io, k, v.ctypes.data)
        self._chk(self.L.vb200_encode_dsp(self.h, W, nstreams, bps, blobno, C.byref(io)))
        return out

    def encode_dsp_managed(self, W, pcm, desc, nstreams=None, fmt=0, hop=0, ampmax0=None, independent=None):
        """Bitrate-managed mode (vb200_encode_dsp_managed): the 15 curves of every block.  Inputs as encode_dsp;
        returns posts [15][nb][ch][FLOOR1_STRIDE], nonzero [15][nb][ch], iwork [15][nb][ch][n], ampmax_out [nb]."""
        ch, n = self.channels, self.bs[W] // 2
        io, nstreams, bps, keep = self._encode_io(W, pcm, desc, nstreams, fmt, hop, ampmax0, independent)
        nb = nstreams * bps
        NB = abi.PACKETBLOBS
        out = {"posts": np.full((NB, nb, ch, abi.FLOOR1_STRIDE), -1, np.int32), "nonzero": np.full((NB, nb, ch), -1, np.int32),
               "iwork": np.full((NB, nb, ch, n), -1, np.int32), "ampmax_out": np.zeros(nb, np.float32)}
        for k, v in out.items():
            setattr(io, k, v.ctypes.data)
        self._chk(self.L.vb200_encode_dsp_managed(self.h, W, nstreams, bps, C.byref(io)))
        return out

    def encode_dsp_dev(self, W, nstreams, bps, io, blobno=7, stream=None):
        """io: abi.EncodeIO holding DEVICE pointers."""
        self._chk(self.L.vb200_encode_dsp_dev(self.h, W, nstreams, bps, blobno, C.byref(io), _ptr(stream)))

    # ---- residue partition classification (lib/res0.c:412-532) --------------------------------
    def residue_partvals(self, W):
        return int(self.L.vb200_residue_partvals(self.h, W))

    def residue_classify(self, W, iwork, nonzero, stride=None):
        ch, n = self.channels, self.bs[W] // 2
        iwork = np.ascontiguousarray(iwork, np.int32).reshape(-1, ch, n)
        nonzero = np.ascontiguousarray(nonzero, np.int32).reshape(-1, ch)
        stride = self.residue_partvals(W) if stride is None else stride
        classes = np.full((iwork.shape[0], ch, stride), -1, np.int32)
        self._chk(self.L.vb200_residue_classify(self.h, W, iwork.shape[0], _ptr(iwork), _ptr(nonzero), _ptr(classes),
                                                stride))
        return classes

    def residue_classify_dev(self, W, nblocks, d_iwork, d_nonzero, d_classes, stride, stream=None):
        self._chk(self.L.vb200_residue_classify_dev(self.h, W, nblocks, _ptr(d_iwork), _ptr(d_nonzero), _ptr(d_classes),
                                                    stride, _ptr(stream)))

    # ---- decode: floor multiply and the whole decode DSP in one call ----------------------------
    def floor1_inverse2(self, W, posts, present, data, floor_sel=-1):
        """floor1_inverse2 (lib/floor1.c:1041): rows [block][channel] of n floats, multiplied in place"""
        n = self.bs[W] // 2
        posts = np.ascontiguousarray(posts, np.int32).reshape(-1, abi.FLOOR1_STRIDE)
        present = np.ascontiguousarray(present, np.int32).reshape(-1)
        data = np.array(data, np.float32).reshape(posts.shape[0], n)
        self._chk(self.L.vb200_floor1_inverse2(self.h, W, floor_sel, posts.shape[0], _ptr(posts), _ptr(present),
                                               _ptr(data)))
        return data

    def decode_dsp(self, Wseq, coef_off, res, posts, present, pcm_off, pcm_stride, s16=False):
        """de-couple + floor multiply + IMDCT + overlap-add in one call; layout as synthesis()"""
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        res = np.array(res, np.float32)
        posts = np.ascontiguousarray(posts, np.int32)
        present = np.ascontiguousarray(present, np.int32)
        coef_off = np.ascontiguousarray(coef_off, np.int64)
        pcm_off = np.ascontiguousarray(pcm_off, np.int64)
        pcm = (np.zeros((ns, pcm_stride, self.channels), np.int16) if s16
               else np.zeros((ns, self.channels, pcm_stride), np.float32))
        self._chk(self.L.vb200_decode_dsp(self.h, ns, nblk, _ptr(Wseq), _ptr(coef_off), _ptr(res), res.size,
                                          _ptr(posts), _ptr(present), _ptr(pcm_off), _ptr(pcm), 1 if s16 else 0,
                                          pcm_stride))
        return pcm

    def new_decode_carry(self, nstreams):
        """the overlap state of nstreams fresh decoders for decode_dsp_resume: (tail, W)"""
        return (np.zeros((nstreams, self.channels, self.bs[1] // 2), np.float32),
                np.full((nstreams, self.channels), -1, np.int32))

    def decode_dsp_resume(self, Wseq, coef_off, res, posts, present, pcm_off, pcm_stride, carry, count=None,
                          s16=False):
        """vb200_decode_dsp_resume: decode_dsp that continues each stream from carry = (tail, W) (new_decode_carry)
        and leaves the overlap of its last decoded block there, in place.  count [nstreams]: blocks per stream
        (None = all).  Offsets from synthesis_layout(..., carry_W=carry[1], count=count)."""
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        tail, W = carry
        assert tail.dtype == np.float32 and W.dtype == np.int32 and tail.flags.c_contiguous and W.flags.c_contiguous
        assert tail.shape == (ns, self.channels, self.bs[1] // 2) and W.shape == (ns, self.channels)
        res = np.array(res, np.float32)
        posts = np.ascontiguousarray(posts, np.int32)
        present = np.ascontiguousarray(present, np.int32)
        coef_off = np.ascontiguousarray(coef_off, np.int64)
        pcm_off = np.ascontiguousarray(pcm_off, np.int64)
        count = None if count is None else np.ascontiguousarray(count, np.int32)
        pcm = (np.zeros((ns, pcm_stride, self.channels), np.int16) if s16
               else np.zeros((ns, self.channels, pcm_stride), np.float32))
        k = abi.DecodeCarry(tail.ctypes.data, W.ctypes.data)
        self._chk(self.L.vb200_decode_dsp_resume(self.h, ns, nblk, _ptr(count), _ptr(Wseq), _ptr(coef_off), _ptr(res),
                                                 res.size, _ptr(posts), _ptr(present), _ptr(pcm_off), _ptr(pcm),
                                                 1 if s16 else 0, pcm_stride, C.byref(k)))
        return pcm

    def decode_dsp_resume_dev(self, nstreams, nblk, d_count, d_Wseq, d_coef_off, d_res, d_posts, d_present, d_pcm_off,
                              d_pcm, pcm_s16, pcm_stride, d_tail, d_W, stream=None):
        k = abi.DecodeCarry(_ptr(d_tail), _ptr(d_W))
        self._chk(self.L.vb200_decode_dsp_resume_dev(self.h, nstreams, nblk, _ptr(d_count), _ptr(d_Wseq),
                                                     _ptr(d_coef_off), _ptr(d_res), _ptr(d_posts), _ptr(d_present),
                                                     _ptr(d_pcm_off), _ptr(d_pcm), pcm_s16, pcm_stride, C.byref(k),
                                                     _ptr(stream)))

    # ---- decode from the packets: the entropy decoders on the device ---------------------------------
    def decode_entropy_setup(self, es):
        """vb200_decode_entropy_setup with an abi.EntropySetup"""
        self._chk(self.L.vb200_decode_entropy_setup(self.h, C.byref(es)))

    def decode_entropy(self, Wseq, pkt_off, pkt_bytes, data, coef_off, res_len):
        """vb200_decode_entropy: (res [res_len], posts [nblocks][ch][FLOOR1_STRIDE], present [nblocks][ch])"""
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        nb = len(Wseq)
        pkt_off = np.ascontiguousarray(pkt_off, np.int64)
        pkt_bytes = np.ascontiguousarray(pkt_bytes, np.int32)
        data = np.ascontiguousarray(data, np.uint8)
        coef_off = np.ascontiguousarray(coef_off, np.int64)
        res = np.zeros(max(res_len, 1), np.float32)
        posts = np.zeros((nb, self.channels, abi.FLOOR1_STRIDE), np.int32)
        present = np.zeros((nb, self.channels), np.int32)
        self._chk(self.L.vb200_decode_entropy(self.h, nb, _ptr(Wseq), _ptr(pkt_off), _ptr(pkt_bytes), _ptr(data),
                                              data.size, _ptr(coef_off), _ptr(res), res_len, _ptr(posts),
                                              _ptr(present)))
        return res, posts, present

    def decode_packets_resume(self, Wseq, coef_off, res_len, pkt_off, pkt_bytes, data, pcm_off, pcm_stride, carry,
                              count=None, s16=False):
        """vb200_decode_packets_resume: decode_dsp_resume from the packets (pkt_off, pkt_bytes [nstreams][nblk] into
        data); carry = (tail, W) as for decode_dsp_resume, updated in place"""
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        tail, W = carry
        assert tail.dtype == np.float32 and W.dtype == np.int32 and tail.flags.c_contiguous and W.flags.c_contiguous
        coef_off = np.ascontiguousarray(coef_off, np.int64)
        pcm_off = np.ascontiguousarray(pcm_off, np.int64)
        pkt_off = np.ascontiguousarray(pkt_off, np.int64)
        pkt_bytes = np.ascontiguousarray(pkt_bytes, np.int32)
        data = np.ascontiguousarray(data, np.uint8)
        count = None if count is None else np.ascontiguousarray(count, np.int32)
        pcm = (np.zeros((ns, pcm_stride, self.channels), np.int16) if s16
               else np.zeros((ns, self.channels, pcm_stride), np.float32))
        k = abi.DecodeCarry(tail.ctypes.data, W.ctypes.data)
        self._chk(self.L.vb200_decode_packets_resume(self.h, ns, nblk, _ptr(count), _ptr(Wseq), _ptr(coef_off),
                                                     res_len, _ptr(pkt_off), _ptr(pkt_bytes), _ptr(data), data.size,
                                                     _ptr(pcm_off), _ptr(pcm), 1 if s16 else 0, pcm_stride,
                                                     C.byref(k)))
        return pcm

    def decode_packets_resume_dev(self, nstreams, nblk, d_count, d_Wseq, d_coef_off, d_res, d_pkt_off, d_pkt_bytes,
                                  d_data, d_pcm_off, d_pcm, pcm_s16, pcm_stride, d_tail, d_W, stream=None):
        k = abi.DecodeCarry(_ptr(d_tail), _ptr(d_W))
        self._chk(self.L.vb200_decode_packets_resume_dev(self.h, nstreams, nblk, _ptr(d_count), _ptr(d_Wseq),
                                                         _ptr(d_coef_off), _ptr(d_res), _ptr(d_pkt_off),
                                                         _ptr(d_pkt_bytes), _ptr(d_data), _ptr(d_pcm_off),
                                                         _ptr(d_pcm), pcm_s16, pcm_stride, C.byref(k),
                                                         _ptr(stream)))

    # ---- whole streams from packets ----------------------------------------------------------------
    def decode_streams_carry(self, nstreams):
        """fresh decoder carries for decode_streams_packets, in device memory (a DecodeStreamsCarry)"""
        nbytes = self.L.vb200_decode_streams_carry_bytes(self.h)
        self._chk(min(nbytes, 0))
        carry = DecodeStreamsCarry(self, nstreams, nbytes)
        self.decode_streams_carry_init(carry)
        return carry

    def decode_streams_carry_init(self, carry, stream=None):
        """vb200_decode_streams_carry_init (vorbis_synthesis_restart) on every carry, or on stream `stream`'s only"""
        if stream is None:
            self._chk(self.L.vb200_decode_streams_carry_init(self.h, carry.nstreams, carry.ptr))
        else:
            assert 0 <= stream < carry.nstreams
            self._chk(self.L.vb200_decode_streams_carry_init(self.h, 1, carry.ptr + stream * carry.nbytes))

    def decode_streams_packets(self, npkt, info, data, carry, s16=False, pcm_cap=None, check=True):
        """vb200_decode_streams_packets: npkt [nstreams], info PACKET_INFO_DTYPE [nstreams][max_packets], data uint8;
        carry from decode_streams_carry, advanced in place.  pcm_cap (elements) defaults to the bound
        sum(npkt) * (blocksizes[1]/2 >> halfrate) * ch.  Returns {"pcm_base", "out" (DECODED_PACKET_DTYPE, shaped as
        info), "pcm": per stream float [ch][n_s] or int16 [n_s][ch], "rc"}; check: raise on an error"""
        npkt = np.ascontiguousarray(npkt, np.int32)
        info = np.ascontiguousarray(info, abi.PACKET_INFO_DTYPE)
        data = np.ascontiguousarray(data, np.uint8)
        ns, mp = info.shape
        ch = self.channels
        if pcm_cap is None:
            pcm_cap = int(npkt.sum()) * ((self.bs[1] // 2) >> self.halfrate) * ch
        pcm = np.zeros(max(pcm_cap, 1), np.int16 if s16 else np.float32)
        base = np.zeros(ns + 1, np.int64)
        out = np.zeros((ns, mp), abi.DECODED_PACKET_DTYPE)
        rc = self.L.vb200_decode_streams_packets(self.h, ns, mp, _ptr(npkt), _ptr(info), _ptr(data), data.size,
                                                 carry.ptr, 1 if s16 else 0, _ptr(pcm), pcm_cap, _ptr(base), _ptr(out))
        if check:
            self._chk(rc)
        res = {"pcm_base": base, "out": out, "rc": rc}
        if rc == 0:
            res["pcm"] = [pcm[base[s] * ch:base[s + 1] * ch].reshape(-1, ch) if s16
                          else pcm[base[s] * ch:base[s + 1] * ch].reshape(ch, -1) for s in range(ns)]
        return res

    def decode_streams_packets_dev(self, nstreams, max_packets, d_npkt, d_info, d_data, d_carry, pcm_s16, d_pcm,
                                   pcm_cap, d_pcm_base, d_out, stream=None):
        self._chk(self.L.vb200_decode_streams_packets_dev(self.h, nstreams, max_packets, _ptr(d_npkt), _ptr(d_info),
                                                          _ptr(d_data), _ptr(d_carry), pcm_s16, _ptr(d_pcm), pcm_cap,
                                                          _ptr(d_pcm_base), _ptr(d_out), _ptr(stream)))

    # ---- sample ranges from packets ---------------------------------------------------------------
    def decode_streams_index(self, npkt, info, data, check=True):
        """vb200_decode_streams_index: the bookkeeping of a fresh-carry decode_streams_packets call without decoding.
        Returns {"length" int64 [nstreams], "out" (DECODED_PACKET_DTYPE, shaped as info), "rc"}"""
        npkt = np.ascontiguousarray(npkt, np.int32)
        info = np.ascontiguousarray(info, abi.PACKET_INFO_DTYPE)
        data = np.ascontiguousarray(data, np.uint8)
        ns, mp = info.shape
        length = np.zeros(ns, np.int64)
        out = np.zeros((ns, mp), abi.DECODED_PACKET_DTYPE)
        rc = self.L.vb200_decode_streams_index(self.h, ns, mp, _ptr(npkt), _ptr(info), _ptr(data), data.size,
                                               _ptr(length), _ptr(out))
        if check:
            self._chk(rc)
        return {"length": length, "out": out, "rc": rc}

    def decode_streams_index_dev(self, nstreams, max_packets, d_npkt, d_info, d_data, d_length, d_out, stream=None):
        self._chk(self.L.vb200_decode_streams_index_dev(self.h, nstreams, max_packets, _ptr(d_npkt), _ptr(d_info),
                                                        _ptr(d_data), _ptr(d_length), _ptr(d_out), _ptr(stream)))

    def decode_ranges(self, npkt, info, data, req, out_stride, s16=False, check=True):
        """vb200_decode_ranges: req PCM_RANGE_DTYPE [nreq] (or (start, stream, length) rows).  Returns {"pcm": float
        [nreq][ch][out_stride] or int16 [nreq][out_stride][ch], "got" int32 [nreq], "rc"}"""
        npkt = np.ascontiguousarray(npkt, np.int32)
        info = np.ascontiguousarray(info, abi.PACKET_INFO_DTYPE)
        data = np.ascontiguousarray(data, np.uint8)
        if not (isinstance(req, np.ndarray) and req.dtype == abi.PCM_RANGE_DTYPE):
            req = np.array([tuple(r) for r in req], abi.PCM_RANGE_DTYPE)
        req = np.ascontiguousarray(req)
        ns, mp = info.shape
        nreq, ch = len(req), self.channels
        pcm = np.zeros((nreq, out_stride, ch) if s16 else (nreq, ch, out_stride), np.int16 if s16 else np.float32)
        got = np.zeros(nreq, np.int32)
        rc = self.L.vb200_decode_ranges(self.h, ns, mp, _ptr(npkt), _ptr(info), _ptr(data), data.size, nreq,
                                        _ptr(req), 1 if s16 else 0, _ptr(pcm), out_stride, _ptr(got))
        if check:
            self._chk(rc)
        return {"pcm": pcm, "got": got, "rc": rc}

    def decode_ranges_dev(self, nstreams, max_packets, d_npkt, d_info, d_data, nreq, d_req, pcm_s16, d_pcm,
                          out_stride, d_got, stream=None):
        self._chk(self.L.vb200_decode_ranges_dev(self.h, nstreams, max_packets, _ptr(d_npkt), _ptr(d_info),
                                                 _ptr(d_data), nreq, _ptr(d_req), pcm_s16, _ptr(d_pcm), out_stride,
                                                 _ptr(d_got), _ptr(stream)))

    def ogg_ranges(self, files, req, out_stride, pkt_cap, s16=False, check=True):
        """vb200_ogg_ranges on a list of Ogg rows (bytes or uint8 arrays) laid back to back: req PCM_RANGE_DTYPE [nreq]
        (or (start, row, length) rows).  Returns {"pcm": float [nreq][ch][out_stride] or int16
        [nreq][out_stride][ch], "got" int32 [nreq], "row_off" int64 [nrows+1], "rc"}"""
        arrs = [np.frombuffer(bytes(f), np.uint8) for f in files]
        row_off = np.zeros(len(arrs) + 1, np.int64)
        row_off[1:] = np.cumsum([len(a) for a in arrs])
        buf = np.ascontiguousarray(np.concatenate(arrs) if arrs else np.zeros(1, np.uint8))
        if not (isinstance(req, np.ndarray) and req.dtype == abi.PCM_RANGE_DTYPE):
            req = np.array([tuple(r) for r in req], abi.PCM_RANGE_DTYPE)
        req = np.ascontiguousarray(req)
        nreq, ch = len(req), self.channels
        pcm = np.zeros((nreq, out_stride, ch) if s16 else (nreq, ch, out_stride), np.int16 if s16 else np.float32)
        got = np.zeros(nreq, np.int32)
        rc = self.L.vb200_ogg_ranges(self.h, len(arrs), _ptr(buf), _ptr(row_off), nreq, _ptr(req), 1 if s16 else 0,
                                     _ptr(pcm), out_stride, pkt_cap, _ptr(got))
        if check:
            self._chk(rc)
        return {"pcm": pcm, "got": got, "row_off": row_off, "rc": rc}

    def ogg_ranges_dev(self, nrows, d_bytes, d_row_off, nreq, d_req, pcm_s16, d_pcm, out_stride, pkt_cap, d_got,
                       stream=None):
        self._chk(self.L.vb200_ogg_ranges_dev(self.h, nrows, _ptr(d_bytes), _ptr(d_row_off), nreq, _ptr(d_req),
                                              pcm_s16, _ptr(d_pcm), out_stride, pkt_cap, _ptr(d_got), _ptr(stream)))

    # ---- encode: the entropy coding of mapping0_forward on the device -----------------------------
    def encode_entropy_setup(self, es):
        """vb200_encode_entropy_setup with an abi.EncodeEntropySetup"""
        self._chk(self.L.vb200_encode_entropy_setup(self.h, C.byref(es)))

    def packet_bound(self, W):
        b = self.L.vb200_encode_packet_bound(self.h, W)
        if b < 0:
            self._chk(b)
        return b

    @staticmethod
    def _packets(out, nb):
        off, bits, data = out["pkt_off"], out["pkt_bits"], out["data"]
        out["packets"] = [bytes(data[off[i]:off[i] + (bits[i] + 7) // 8]) for i in range(nb)]
        return out

    def encode_entropy(self, W, desc, posts, nonzero, iwork, data_cap=None, check=True):
        """vb200_encode_entropy on vb200_encode_dsp's outputs: {"packets": [bytes], "pkt_bits", "pkt_off", "data"}
        (and "rc" when check is False, in which case an error does not raise)"""
        ch, n = self.channels, self.bs[W] // 2
        desc = np.ascontiguousarray(desc, abi.BLOCKDESC_DTYPE)
        nb = desc.shape[0]
        posts = np.ascontiguousarray(posts, np.int32).reshape(nb, ch, abi.FLOOR1_STRIDE)
        nonzero = np.ascontiguousarray(nonzero, np.int32).reshape(nb, ch)
        iwork = np.ascontiguousarray(iwork, np.int32).reshape(nb, ch, n)
        cap = nb * self.packet_bound(W) if data_cap is None else data_cap
        out = {"pkt_off": np.zeros(nb, np.int64), "pkt_bits": np.zeros(nb, np.int32),
               "data": np.zeros(max(cap, 1), np.uint8)}
        rc = self.L.vb200_encode_entropy(self.h, W, nb, _ptr(desc), _ptr(posts), _ptr(nonzero), _ptr(iwork),
                                         _ptr(out["pkt_off"]), _ptr(out["pkt_bits"]), _ptr(out["data"]), cap)
        if not check:
            out["rc"] = rc
            return out
        self._chk(rc)
        return self._packets(out, nb)

    def encode_entropy_dev(self, W, nblocks, d_desc, d_posts, d_nonzero, d_iwork, pkt_stride, d_pkt_bits, d_data,
                           stream=None, check=True):
        rc = self.L.vb200_encode_entropy_dev(self.h, W, nblocks, _ptr(d_desc), _ptr(d_posts), _ptr(d_nonzero),
                                             _ptr(d_iwork), pkt_stride, _ptr(d_pkt_bits), _ptr(d_data), _ptr(stream))
        if check:
            self._chk(rc)
        return rc

    def encode_packets(self, W, pcm, desc, nstreams=None, fmt=0, hop=0, ampmax0=None, independent=None, blobno=7,
                       data_cap=None):
        """vb200_encode_packets: PCM as for encode_dsp in, {"packets", "pkt_bits", "pkt_off", "data", "ampmax_out"}
        out"""
        io, nstreams, bps, keep = self._encode_io(W, pcm, desc, nstreams, fmt, hop, ampmax0, independent)
        nb = nstreams * bps
        cap = nb * self.packet_bound(W) if data_cap is None else data_cap
        out = {"pkt_off": np.zeros(nb, np.int64), "pkt_bits": np.zeros(nb, np.int32),
               "data": np.zeros(max(cap, 1), np.uint8), "ampmax_out": np.zeros(nb, np.float32)}
        io.ampmax_out = out["ampmax_out"].ctypes.data
        self._chk(self.L.vb200_encode_packets(self.h, W, nstreams, bps, blobno, C.byref(io), _ptr(out["pkt_off"]),
                                              _ptr(out["pkt_bits"]), _ptr(out["data"]), cap))
        return self._packets(out, nb)

    def encode_entropy_managed_dev(self, W, nblocks, blob_blocks, d_desc, d_posts, d_nonzero, d_iwork, pkt_stride,
                                   d_pkt_bits, d_data, stream=None, check=True):
        """vb200_encode_entropy_managed_dev: all 15 packets of every block, packet (k, b) at d_data +
        (k*nblocks + b)*pkt_stride; returns the status"""
        rc = self.L.vb200_encode_entropy_managed_dev(self.h, W, nblocks, blob_blocks, _ptr(d_desc), _ptr(d_posts),
                                                     _ptr(d_nonzero), _ptr(d_iwork), pkt_stride, _ptr(d_pkt_bits),
                                                     _ptr(d_data), _ptr(stream))
        if check:
            self._chk(rc)
        return rc

    def encode_packets_managed(self, W, pcm, desc, nstreams=None, fmt=0, hop=0, ampmax0=None, independent=None,
                               data_cap=None, check=True):
        """vb200_encode_packets_managed: PCM as for encode_dsp_managed in; {"packets": [15][nb] bytes, "pkt_bits"
        [15][nb], "pkt_off" [15][nb], "data", "ampmax_out"} out (and "rc" when check is False, in which case an error
        does not raise and "packets" is absent)"""
        NB = abi.PACKETBLOBS
        io, nstreams, bps, keep = self._encode_io(W, pcm, desc, nstreams, fmt, hop, ampmax0, independent)
        nb = nstreams * bps
        cap = NB * nb * self.packet_bound(W) if data_cap is None else data_cap
        out = {"pkt_off": np.zeros((NB, nb), np.int64), "pkt_bits": np.zeros((NB, nb), np.int32),
               "data": np.zeros(max(cap, 1), np.uint8), "ampmax_out": np.zeros(nb, np.float32)}
        io.ampmax_out = out["ampmax_out"].ctypes.data
        rc = self.L.vb200_encode_packets_managed(self.h, W, nstreams, bps, C.byref(io), _ptr(out["pkt_off"]),
                                                 _ptr(out["pkt_bits"]), _ptr(out["data"]), cap)
        if not check:
            out["rc"] = rc
            return out
        self._chk(rc)
        off, bits, data = out["pkt_off"], out["pkt_bits"], out["data"]
        out["packets"] = [[bytes(data[off[k, i]:off[k, i] + (bits[k, i] + 7) // 8]) for i in range(nb)]
                          for k in range(NB)]
        return out

    # ---- the bitrate manager on the device and whole streams to packets ------------------------------------
    def bitrate_setup(self, info):
        """vb200_bitrate_setup with an abi.BitrateInfo"""
        self._chk(self.L.vb200_bitrate_setup(self.h, C.byref(info)))

    def bitrate_init(self, nstreams=1):
        """vorbis_bitrate_init's state for nstreams streams (abi.BITRATE_STATE_DTYPE [nstreams])"""
        st = np.zeros(nstreams, abi.BITRATE_STATE_DTYPE)
        for i in range(nstreams):
            self._chk(self.L.vb200_bitrate_init(self.h, st[i:].ctypes.data))
        return st

    def bitrate_addblocks(self, count, W, pkt_bits, state, choice=None, nbytes=None, check=True):
        """vb200_bitrate_addblocks: count [ns], W [ns][max_blocks], pkt_bits [ns][max_blocks][15]; state
        (BITRATE_STATE_DTYPE [ns]) advanced in place.  Returns (choice, bytes) [ns][max_blocks] (entries past count as
        passed in), or the status when check is False."""
        W = np.ascontiguousarray(W, np.int32)
        ns, mb = W.shape
        count = np.ascontiguousarray(count, np.int32)
        pkt_bits = np.ascontiguousarray(pkt_bits, np.int32).reshape(ns, mb, abi.PACKETBLOBS)
        choice = np.zeros((ns, mb), np.int32) if choice is None else choice
        nbytes = np.zeros((ns, mb), np.int32) if nbytes is None else nbytes
        rc = self.L.vb200_bitrate_addblocks(self.h, ns, mb, _ptr(count), _ptr(W), _ptr(pkt_bits), _ptr(state),
                                            _ptr(choice), _ptr(nbytes))
        if not check:
            return rc
        self._chk(rc)
        return choice, nbytes

    def bitrate_addblocks_dev(self, nstreams, max_blocks, d_count, d_W, d_pkt_bits, d_state, d_choice, d_bytes,
                              stream=None, check=True):
        rc = self.L.vb200_bitrate_addblocks_dev(self.h, nstreams, max_blocks, _ptr(d_count), _ptr(d_W),
                                                _ptr(d_pkt_bits), _ptr(d_state), _ptr(d_choice), _ptr(d_bytes),
                                                _ptr(stream))
        if check:
            self._chk(rc)
        return rc

    def encode_carry_init(self, nstreams, mark_steps=0):
        """vb200_encode_carry_init: fresh carries, uint8 [nstreams][vb200_encode_carry_bytes] (the managed form wants
        them made after bitrate_setup); encode_carry_head(carry) reads their public heads"""
        nbytes = self.L.vb200_encode_carry_bytes(self.h, mark_steps)
        self._chk(min(nbytes, 0))
        carry = np.zeros((nstreams, nbytes), np.uint8)
        self._chk(self.L.vb200_encode_carry_init(self.h, nstreams, mark_steps, _ptr(carry)))
        return carry

    @staticmethod
    def encode_carry_head(carry):
        """the vb200_encode_carry heads of carries made by encode_carry_init (ENCODE_CARRY_HEAD_DTYPE [nstreams], a copy)"""
        hs = abi.ENCODE_CARRY_HEAD_DTYPE.itemsize
        return np.ascontiguousarray(carry[:, :hs]).view(abi.ENCODE_CARRY_HEAD_DTYPE)[:, 0]

    def encode_streams_packets_resume(self, pcm, pcm_len, carry, eof=None, managed=False, **kw):
        """vb200_encode_streams_packets[_managed]_resume: as encode_streams_packets, stream s's buffer starting at its
        carry's base; carry (from encode_carry_init) is advanced in place when the call succeeds"""
        return self.encode_streams_packets(pcm, pcm_len, eof, managed=managed, carry=carry, **kw)

    def encode_streams_packets(self, pcm, pcm_len, eof=None, fmt=PCM_F32_PLANAR, max_blocks=None, cap=None, blobno=7,
                               managed=False, data_cap=None, check=True, carry=None):
        """vb200_encode_streams_packets[_managed] on timeline buffers as for encode_streams: {"plan", "nblocks",
        "count", "info" (PACKET_INFO_DTYPE [ns][max_blocks]), "data", "packets": per stream [bytes]} (and "rc" when
        check is False, in which case an error does not raise and "packets" is absent).  carry: the _resume forms"""
        io, plan, nb, keep = self._streams_io(pcm, pcm_len, eof, fmt, max_blocks, cap)
        ns, max_blocks = plan.shape
        info = np.zeros((ns, max_blocks), abi.PACKET_INFO_DTYPE)
        if data_cap is None:
            data_cap = ns * max_blocks * max(self.packet_bound(0), self.packet_bound(1))
        data = np.zeros(max(data_cap, 1), np.uint8)
        if carry is not None:
            assert carry.dtype == np.uint8 and carry.flags.c_contiguous and carry.shape[0] == ns
            if managed:
                rc = self.L.vb200_encode_streams_packets_managed_resume(self.h, ns, C.byref(io), _ptr(carry), _ptr(info),
                                                                        _ptr(data), data_cap)
            else:
                rc = self.L.vb200_encode_streams_packets_resume(self.h, ns, blobno, C.byref(io), _ptr(carry), _ptr(info),
                                                                _ptr(data), data_cap)
        elif managed:
            rc = self.L.vb200_encode_streams_packets_managed(self.h, ns, C.byref(io), _ptr(info), _ptr(data), data_cap)
        else:
            rc = self.L.vb200_encode_streams_packets(self.h, ns, blobno, C.byref(io), _ptr(info), _ptr(data), data_cap)
        return self._stream_packets(rc, check, io, plan, nb, info, data)

    def _stream_packets(self, rc, check, io, plan, nb, info, data):
        """the result of the calls that write stream-ordered packets: stream i's packets split out of data by its
        first nb[i] info records ("rc" in place of "packets" when check is False)"""
        out = {"plan": plan, "nblocks": nb, "count": [io.count[0], io.count[1]], "info": info, "data": data}
        if not check:
            out["rc"] = rc
            return out
        self._chk(rc)
        out["packets"] = [[bytes(data[r["offset"]:r["offset"] + r["bytes"]]) for r in info[i, :nb[i]]]
                          for i in range(len(nb))]
        return out

    def encode_pcm_carry_init(self, nstreams, mark_steps=0):
        """vb200_encode_pcm_carry_init: fresh raw-PCM carries, uint8 [nstreams][vb200_encode_pcm_carry_bytes] (the
        managed form wants them made after bitrate_setup); encode_pcm_carry_head(carry) reads their public heads"""
        nbytes = self.L.vb200_encode_pcm_carry_bytes(self.h, mark_steps)
        self._chk(min(nbytes, 0))
        carry = np.zeros((nstreams, nbytes), np.uint8)
        self._chk(self.L.vb200_encode_pcm_carry_init(self.h, nstreams, mark_steps, _ptr(carry)))
        return carry

    @staticmethod
    def encode_pcm_carry_head(carry):
        """the vb200_pcm_carry heads of carries made by encode_pcm_carry_init (PCM_CARRY_HEAD_DTYPE [nstreams], a copy)"""
        hs = abi.PCM_CARRY_HEAD_DTYPE.itemsize
        return np.ascontiguousarray(carry[:, :hs]).view(abi.PCM_CARRY_HEAD_DTYPE)[:, 0]

    def encode_pcm_packets(self, pcm, pcm_len, carry, end=None, managed=False, max_blocks=None, cap=None, blobno=7,
                           data_cap=None, check=True):
        """vb200_encode_pcm_packets[_managed]: pcm float32 [ns][ch][stride] (VB200_PCM_F32_PLANAR) or int16
        [ns][stride][ch] (VB200_PCM_S16_INTERLEAVED), stream s's input from its carry's raw_base; pcm_len [ns] the kept
        plus the new samples; end [ns] (nonzero: vorbis_analysis_wrote(v, 0)) or None.  carry (from
        encode_pcm_carry_init) is advanced in place when the call succeeds.  Returns as encode_streams_packets."""
        ch, bs0, bs1 = self.channels, self.bs[0], self.bs[1]
        if pcm.dtype == np.int16:
            fmt, pcm = PCM_S16_INTERLEAVED, np.ascontiguousarray(pcm)
            ns, stride = pcm.shape[0], pcm.shape[1]
            assert pcm.shape[2] == ch
        else:
            fmt, pcm = PCM_F32_PLANAR, np.ascontiguousarray(pcm, np.float32)
            ns, stride = pcm.shape[0], pcm.shape[2]
            assert pcm.shape[1] == ch
        assert carry.dtype == np.uint8 and carry.flags.c_contiguous and carry.shape[0] == ns
        pcm_len = np.ascontiguousarray(pcm_len, np.int64)
        endp = None if end is None else np.ascontiguousarray(end, np.int32)
        span = stride + 4 * bs1                       # the timeline adds the preamble and the tail to the input
        if max_blocks is None:
            max_blocks = span // (bs0 // 2) + 8
        if cap is None:
            cap = [ns * max_blocks, ns * (span // (bs1 // 2) + 8)]
        io = abi.PcmIO()
        io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = pcm.ctypes.data, fmt, max_blocks, stride
        io.pcm_len = pcm_len.ctypes.data
        io.end = None if endp is None else endp.ctypes.data
        plan = np.zeros((ns, max_blocks), abi.STREAM_BLOCK_DTYPE)
        nb = np.zeros(ns, np.int32)
        io.plan, io.nblocks = plan.ctypes.data, nb.ctypes.data
        io.cap[0], io.cap[1] = int(cap[0]), int(cap[1])
        info = np.zeros((ns, max_blocks), abi.PACKET_INFO_DTYPE)
        if data_cap is None:
            data_cap = ns * max_blocks * max(self.packet_bound(0), self.packet_bound(1))
        data = np.zeros(max(data_cap, 1), np.uint8)
        if managed:
            rc = self.L.vb200_encode_pcm_packets_managed(self.h, ns, C.byref(io), _ptr(carry), _ptr(info), _ptr(data),
                                                         data_cap)
        else:
            rc = self.L.vb200_encode_pcm_packets(self.h, ns, blobno, C.byref(io), _ptr(carry), _ptr(info), _ptr(data),
                                                 data_cap)
        return self._stream_packets(rc, check, io, plan, nb, info, data)

    def encode_pcm_packets_dev(self, nstreams, d_pcm, pcm_fmt, stream_stride, d_pcm_len, d_carry, d_plan, d_nblocks,
                               max_blocks, cap, d_info, d_data, data_cap, d_status, d_result, d_end=None, d_first=None,
                               mark_steps=0, managed=False, blobno=7, stream=None, check=True):
        """vb200_encode_pcm_packets[_managed]_dev: d_ arguments are device addresses (ints, e.g. data_ptr());
        the call's outcome is in d_status and d_result (abi.ENCODE_RESULT_DTYPE).  Returns the synchronous status."""
        io = abi.PcmIO()
        io.pcm, io.pcm_fmt, io.max_blocks, io.stream_stride = _ptr(d_pcm), pcm_fmt, max_blocks, stream_stride
        io.pcm_len, io.end, io.plan, io.nblocks = _ptr(d_pcm_len), _ptr(d_end), _ptr(d_plan), _ptr(d_nblocks)
        io.cap[0], io.cap[1] = int(cap[0]), int(cap[1])
        args = (_ptr(d_first), _ptr(d_carry), _ptr(d_info), _ptr(d_data), data_cap, _ptr(d_status), _ptr(d_result),
                _ptr(stream))
        if managed:
            rc = self.L.vb200_encode_pcm_packets_managed_dev(self.h, nstreams, mark_steps, C.byref(io), *args)
        else:
            rc = self.L.vb200_encode_pcm_packets_dev(self.h, nstreams, blobno, mark_steps, C.byref(io), *args)
        if check:
            self._chk(rc)
        return rc

    def lpc_extrapolate(self, data, n, order, count, check=True):
        """vb200_lpc_extrapolate: data float32 [rows][stride], n [rows]; returns (coeff float32 [rows][order], out
        float32 [rows][count]), or the status when check is False"""
        data = np.ascontiguousarray(data, np.float32)
        n = np.ascontiguousarray(n, np.int32)
        rows = data.shape[0]
        coeff = np.zeros((rows, order), np.float32)
        out = np.zeros((rows, max(count, 1)), np.float32)
        rc = self.L.vb200_lpc_extrapolate(self.h, rows, order, _ptr(data), data.shape[1], _ptr(n), count, _ptr(coeff),
                                          _ptr(out), out.shape[1])
        if not check:
            return rc
        self._chk(rc)
        return coeff, out[:, :count]

    # ---- envelope / block-switch detector (lib/envelope.c) --------------------------------------
    def envelope_search(self, pcm, first_step, nsteps, state=None, fmt=PCM_F32_PLANAR):
        """Host buffers.  pcm: float [streams][ch][stride] (PCM_F32_PLANAR) or int16 [streams][stride][ch].
        Returns (ret uint8 [streams][nsteps], state int32 [streams][ve_state_words])."""
        ch = self.channels
        if fmt == PCM_F32_PLANAR:
            pcm = np.ascontiguousarray(pcm, np.float32)
            ns, stride = pcm.shape[0], pcm.shape[2]
            assert pcm.shape[1] == ch
        else:
            pcm = np.ascontiguousarray(pcm, np.int16)
            ns, stride = pcm.shape[0], pcm.shape[1]
            assert pcm.shape[2] == ch
        state = (np.zeros((ns, abi.ve_state_words(ch)), np.int32) if state is None
                 else np.array(state, np.int32).reshape(ns, abi.ve_state_words(ch)))
        ret = np.zeros((ns, nsteps), np.uint8)
        self._chk(self.L.vb200_envelope_search(self.h, ns, _ptr(pcm), fmt, stride, first_step, nsteps,
                                               _ptr(state), _ptr(ret)))
        return ret, state

    def envelope_search_dev(self, nstreams, d_pcm, fmt, stride, first_step, nsteps, d_state, d_ret, stream=None):
        self._chk(self.L.vb200_envelope_search_dev(self.h, nstreams, _ptr(d_pcm), fmt, stride, first_step, nsteps,
                                                   _ptr(d_state), _ptr(d_ret), _ptr(stream)))

    def envelope_marks(self, ret, first_step=0, mark=None):
        """replay lib/envelope.c:254-264 for one stream's trigger bits (plain C helper, no GPU)"""
        ret = np.ascontiguousarray(ret, np.uint8)
        if mark is None:
            mark = np.zeros(first_step + len(ret) + 2, np.int32)
        self.L.vb200_envelope_apply_marks(_ptr(ret), first_step, len(ret), _ptr(mark))
        return mark

    # ---- decode ------------------------------------------------------------------
    def decouple(self, W, res):
        res = np.array(res, np.float32)
        self._chk(self.L.vb200_decouple(self.h, W, res.shape[0], _ptr(res)))
        return res

    def synthesis(self, Wseq, coef_off, coef, pcm_off, pcm_stride):
        Wseq = np.ascontiguousarray(Wseq, np.int32)
        ns, nblk = Wseq.shape
        coef_off = np.ascontiguousarray(coef_off, np.int64)
        pcm_off = np.ascontiguousarray(pcm_off, np.int64)
        coef = np.ascontiguousarray(coef, np.float32)
        pcm = np.zeros((ns, self.channels, pcm_stride), np.float32)
        self._chk(self.L.vb200_synthesis(self.h, ns, nblk, _ptr(Wseq), _ptr(coef_off), _ptr(coef), coef.size,
                                         _ptr(pcm_off), _ptr(pcm), pcm_stride))
        return pcm

    def synthesis_halfrate(self, flag, windows=None):
        """vb200_synthesis_halfrate: half-rate decode on (flag true) or off for the decode entry points.
        windows: the half windows of blocksizes[w]/2 (SetupHolder.halfrate_windows()); None = closed form.
        Use synthesis_layout(..., halfrate=True) for the offsets while it is on."""
        keep, ptrs = abi.halfrate_window_ptrs(windows)
        self._chk(self.L.vb200_synthesis_halfrate(self.h, 1 if flag else 0, ptrs))
        self.halfrate = 1 if flag else 0

    def synthesis_dev(self, nstreams, nblk, d_Wseq, d_coef_off, d_coef, d_pcm_off, d_pcm, pcm_stride, stream=None):
        self._chk(self.L.vb200_synthesis_dev(self.h, nstreams, nblk, _ptr(d_Wseq), _ptr(d_coef_off), _ptr(d_coef),
                                             _ptr(d_pcm_off), _ptr(d_pcm), pcm_stride, _ptr(stream)))


class DecodeStreamsCarry:
    """nstreams carries of vb200_decode_streams_packets in device memory (vb200_malloc_device), freed with close()"""

    def __init__(self, ctx, nstreams, nbytes):
        self.ctx, self.nstreams, self.nbytes = ctx, nstreams, nbytes
        p = vp()
        ctx._chk(ctx.L.vb200_malloc_device(ctx.h, nstreams * nbytes, C.byref(p)))
        self.ptr = p.value

    def read(self):
        """a host copy, uint8 [nstreams][nbytes]"""
        a = np.zeros((self.nstreams, self.nbytes), np.uint8)
        self.ctx._chk(self.ctx.L.vb200_memcpy_d2h(self.ctx.h, a.ctypes.data, self.ptr, a.nbytes))
        return a

    def write(self, a):
        a = np.ascontiguousarray(a, np.uint8)
        assert a.shape == (self.nstreams, self.nbytes)
        self.ctx._chk(self.ctx.L.vb200_memcpy_h2d(self.ctx.h, self.ptr, a.ctypes.data, a.nbytes))

    def close(self):
        if self.ptr and self.ctx.h:
            self.ctx.L.vb200_free_device(self.ctx.h, self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def synthesis_layout(Wseq, bs, channels, halfrate=False, carry_W=None, count=None):
    """Offsets for vb200_synthesis: Wseq [nstreams][nblk] -> (coef_off, pcm_off, coef_len, pcm_len)
    with every stream's spectra packed back to back (block-major, channel-minor).  halfrate: the spectra
    keep this layout, the finished samples are counted at half rate ((bs[lW]/4 + bs[W]/4) >> 1 per block,
    lib/block.c:840-842).
    For vb200_decode_dsp_resume: carry_W [nstreams] or [nstreams][ch] = the carried block flags (-1 = none):
    where one is >= 0, block 0 finishes samples as well; count [nstreams]: blocks past count[s] get no spectra
    and finish nothing."""
    Wseq = np.asarray(Wseq, np.int32)
    ns, nblk = Wseq.shape
    N = np.where(Wseq == 1, bs[1], bs[0]).astype(np.int64)
    if count is not None:
        N = np.where(np.arange(nblk)[None, :] < np.asarray(count).reshape(ns, 1), N, 0)
    per_block = channels * (N // 2)
    coef_off = np.zeros((ns, nblk), np.int64)
    flat = per_block.reshape(-1)
    coef_off.reshape(-1)[1:] = np.cumsum(flat)[:-1]
    fin = np.zeros((ns, nblk), np.int64)
    fin[:, 1:] = np.where(N[:, 1:] > 0, N[:, :-1] // 4 + N[:, 1:] // 4, 0) >> (1 if halfrate else 0)
    if carry_W is not None:
        cw = np.asarray(carry_W).reshape(ns, -1)
        assert (cw == cw[:, :1]).all(), "the carried W of a stream differs between its channels"
        cw = cw[:, 0]
        fin[:, 0] = np.where((cw >= 0) & (N[:, 0] > 0), np.where(cw == 1, bs[1], bs[0]) // 4 + N[:, 0] // 4, 0) >> (
            1 if halfrate else 0)
    pcm_off = np.cumsum(fin, axis=1) - fin      # finished samples before block k's contribution
    # block k's finished samples start where block k-1's ended
    pcm_off = np.concatenate([np.zeros((ns, 1), np.int64), np.cumsum(fin, axis=1)[:, :-1]], axis=1)
    pcm_len = int(np.cumsum(fin, axis=1)[:, -1].max())
    return coef_off, pcm_off, int(flat.sum()), pcm_len


# ---- Ogg Vorbis files in ----------------------------------------------------------------------------
def _check(L, rc):
    if rc != 0:
        raise VB200Error("vb200 error %d: %s" % (rc, (L.vb200_last_error() or b"").decode()))


def ogg_demux(files, max_packets=None, check=True):
    """vb200_ogg_demux on a list of Ogg files (bytes or uint8 arrays), on the current CUDA device.  Returns {"data"
    uint8 (every file's packets inside its own byte range, zeros elsewhere), "file_off" int64 [n+1], "info"
    PACKET_INFO_DTYPE [n][max_packets], "npkt" int32 [n], "streams" OGG_STREAM_DTYPE [n], "rc"}.  max_packets
    defaults to the most packets any of the files can hold: a page of 27 + k bytes or more ends at most k packets."""
    L = load()
    arrs = [np.frombuffer(bytes(f), np.uint8) for f in files]
    n = len(arrs)
    file_off = np.zeros(n + 1, np.int64)
    file_off[1:] = np.cumsum([len(a) for a in arrs])
    buf = np.ascontiguousarray(np.concatenate(arrs) if n else np.zeros(0, np.uint8))
    if max_packets is None:
        max_packets = max([1] + [len(a) * 255 // 282 + 1 for a in arrs])
    info = np.zeros((n, max_packets), abi.PACKET_INFO_DTYPE)
    npkt = np.zeros(n, np.int32)
    data = np.zeros(max(len(buf), 1), np.uint8)
    streams = np.zeros(n, abi.OGG_STREAM_DTYPE)
    rc = L.vb200_ogg_demux(n, _ptr(buf), _ptr(file_off), max_packets, _ptr(info), _ptr(npkt), _ptr(data),
                           _ptr(streams))
    if check:
        _check(L, rc)
    return {"data": data[:len(buf)], "file_off": file_off, "info": info, "npkt": npkt, "streams": streams, "rc": rc}


def ogg_demux_dev(nfiles, d_bytes, d_file_off, max_packets, d_info, d_npkt, d_data, d_streams, stream=None):
    """vb200_ogg_demux_dev: device pointers (ints, e.g. torch tensors' data_ptr()), asynchronous on `stream`"""
    L = load()
    _check(L, L.vb200_ogg_demux_dev(nfiles, _ptr(d_bytes), _ptr(d_file_off), max_packets, _ptr(d_info), _ptr(d_npkt),
                                    _ptr(d_data), _ptr(d_streams), _ptr(stream)))


def ogg_links(files, link_cap=None, check=True):
    """vb200_ogg_links on a list of Ogg files (bytes or uint8 arrays), on the current CUDA device.  Returns {"file_off"
    int64 [n+1] (the files back to back), "link_first" int64 [n+1], "link_off" int64 [total+1] (zeros when link_cap
    is below the total), "rc"}.  link_cap defaults to what the table needs (a sizing call first).  link_off with
    link_first[n] is the file_off and nfiles of ogg_demux's rows: ogg_demux([bytes of each link]) is the same call."""
    L = load()
    arrs = [np.frombuffer(bytes(f), np.uint8) for f in files]
    n = len(arrs)
    file_off = np.zeros(n + 1, np.int64)
    file_off[1:] = np.cumsum([len(a) for a in arrs])
    buf = np.ascontiguousarray(np.concatenate(arrs) if n else np.zeros(1, np.uint8))
    link_first = np.zeros(n + 1, np.int64)
    if link_cap is None:
        rc = L.vb200_ogg_links(n, _ptr(buf), _ptr(file_off), _ptr(link_first), None, 0)
        link_cap = int(link_first[n]) if n else 0
        if rc != 0 and link_cap == 0:
            _check(L, rc)
    link_off = np.zeros(link_cap + 1, np.int64)
    rc = L.vb200_ogg_links(n, _ptr(buf), _ptr(file_off), _ptr(link_first), _ptr(link_off), link_cap)
    if check:
        _check(L, rc)
    total = int(link_first[n])
    return {"file_off": file_off, "link_first": link_first,
            "link_off": link_off[:total + 1] if total <= link_cap else np.zeros(total + 1, np.int64), "rc": rc}


def ogg_links_dev(nfiles, d_bytes, d_file_off, d_link_first, d_link_off, link_cap, stream=None):
    """vb200_ogg_links_dev: device pointers (ints, e.g. torch tensors' data_ptr()), asynchronous on `stream`"""
    L = load()
    _check(L, L.vb200_ogg_links_dev(nfiles, _ptr(d_bytes), _ptr(d_file_off), _ptr(d_link_first), _ptr(d_link_off),
                                    link_cap, _ptr(stream)))


def vorbis_window(n):
    """vb200_vorbis_window: the reference's tabulated rising half window of an n-sample block, float32 [n/2]"""
    L = load()
    out = np.zeros(max(n // 2, 1), np.float32)
    _check(L, L.vb200_vorbis_window(n, _ptr(out)))
    return out[:n // 2]


# ---- the header packets to a decode context, and files grouped by setup ---------------------------------------
class VorbisHeaders:
    """vb200_vorbis_headers_parse of three header packets (bytes).  .info: channels, rate, the three bitrates and
    blocksizes; .c / .entropy: the vb200_setup and vb200_entropy_setup it holds (views into it); .context(device)
    a Context with the entropy setup registered.  Raises VB200Error with .code where the parse refuses the headers."""

    def __init__(self, id_, comment, setup):
        self.L = load()
        self._p = C.POINTER(abi.VorbisHeaders)()
        bufs = [np.frombuffer(bytes(b) + b"\0", np.uint8) for b in (id_, comment, setup)]
        rc = self.L.vb200_vorbis_headers_parse(_ptr(bufs[0]), len(id_), _ptr(bufs[1]), len(comment), _ptr(bufs[2]),
                                               len(setup), C.byref(self._p))
        if rc != 0:
            self._p = None
            e = VB200Error("vb200_vorbis_headers_parse: %d" % rc)
            e.code = rc
            raise e
        h = self._p.contents
        self.h = h
        self.c = h.setup
        self.entropy = h.entropy
        self.channels = int(h.channels)
        self.rate = int(h.rate)
        self.blocksizes = [int(h.blocksizes[0]), int(h.blocksizes[1])]
        self.bitrates = (int(h.bitrate_upper), int(h.bitrate_nominal), int(h.bitrate_lower))

    def blocksize(self, W):
        return self.blocksizes[W]

    def context(self, device=0):
        """a Context on these headers' setup, with the entropy setup registered; it keeps this object alive"""
        ctx = Context(self, device)
        ctx.decode_entropy_setup(self.entropy)
        return ctx

    def __del__(self):
        if getattr(self, "_p", None):
            self.L.vb200_vorbis_headers_free(self._p)
            self._p = None


def vorbis_headers(id_, comment, setup):
    """vb200_vorbis_headers_parse: a VorbisHeaders (see there)"""
    return VorbisHeaders(id_, comment, setup)


def ogg_group(res, check=True):
    """vb200_ogg_group on the outputs of ogg_demux (a dict as it returns).  Returns {"status", "order", "npkt",
    "info" (permuted), "groups" FILE_GROUP_DTYPE [ngroups], "rc"}"""
    L = load()
    st = np.ascontiguousarray(res["streams"])
    info = np.ascontiguousarray(res["info"])
    n, mp = info.shape
    npkt = np.ascontiguousarray(res["npkt"], np.int32)
    data = np.ascontiguousarray(res["data"], np.uint8)
    status, order, npkt_out = (np.zeros(n, np.int32) for _ in range(3))
    info_out = np.zeros_like(info)
    groups = np.zeros(max(n, 1), abi.FILE_GROUP_DTYPE)
    ng = np.zeros(1, np.int32)
    rc = L.vb200_ogg_group(n, _ptr(data), data.size, _ptr(st), mp, _ptr(npkt), _ptr(info), _ptr(status), _ptr(order),
                           _ptr(npkt_out), _ptr(info_out), _ptr(groups), _ptr(ng))
    if check:
        _check(L, rc)
    return {"status": status, "order": order, "npkt": npkt_out, "info": info_out, "groups": groups[:int(ng[0])],
            "rc": rc}


def ogg_group_scratch_bytes(nfiles, max_packets):
    return int(load().vb200_ogg_group_scratch_bytes(nfiles, max_packets))


def ogg_group_dev(nfiles, d_data, d_streams, max_packets, d_npkt, d_info, d_status, d_order, d_npkt_out, d_info_out,
                  d_groups, d_ngroups, d_scratch, scratch_bytes, stream=None):
    """vb200_ogg_group_dev: device pointers (ints, e.g. torch tensors' data_ptr()), asynchronous on `stream`"""
    L = load()
    _check(L, L.vb200_ogg_group_dev(nfiles, _ptr(d_data), _ptr(d_streams), max_packets, _ptr(d_npkt), _ptr(d_info),
                                    _ptr(d_status), _ptr(d_order), _ptr(d_npkt_out), _ptr(d_info_out),
                                    _ptr(d_groups), _ptr(d_ngroups), _ptr(d_scratch), scratch_bytes, _ptr(stream)))


# ---- Ogg Vorbis files out -----------------------------------------------------------------------------------
def ogg_mux(packets, granules, eos=None, headers=None, serials=None, carries=None, hdr_granules=(0, 0, 0),
            out_cap=None, check=True):
    """vb200_ogg_mux on host lists, on the current CUDA device.  Per stream s: packets[s] (bytes; the carry's kept
    packets first), granules[s] and eos[s] (default: e_o_s on the last packet), headers[s] (the three header packets,
    needed for fresh carries), and either carries (OGG_MUX_CARRY_DTYPE [n], not modified) or serials (fresh carries).
    Returns {"pages": per stream the bytes of this call's pages (the whole file for a fresh carry and an e_o_s packet),
    "carry" (the new carries; the same as given unless rc is 0), "status", "out_off", "rc"}.  out_cap defaults to
    what the pages need (a sizing call first)."""
    L = load()
    n = len(packets)
    if carries is None:
        carries = np.zeros(n, abi.OGG_MUX_CARRY_DTYPE)
        carries["serial"] = serials
    carry = np.ascontiguousarray(carries, abi.OGG_MUX_CARRY_DTYPE).copy()
    if eos is None:
        eos = [[k == len(p) - 1 for k in range(len(p))] for p in packets]
    max_packets = max([1] + [len(p) for p in packets])
    npkt = np.array([len(p) for p in packets], np.int32)
    info = np.zeros((n, max_packets), abi.PACKET_INFO_DTYPE)
    hdr = np.zeros((n, 3), abi.PACKET_INFO_DTYPE) if headers is not None else None
    blobs, at = [], 0
    for s in range(n):
        if headers is not None:
            for k, h in enumerate(headers[s]):
                hdr[s, k] = (at, hdr_granules[k], len(h), 0, k, 0)
                blobs.append(bytes(h))
                at += len(h)
        for k, p in enumerate(packets[s]):
            info[s, k] = (at, granules[s][k], len(p), 1 if eos[s][k] else 0, 0, 0)
            blobs.append(bytes(p))
            at += len(p)
    data = np.frombuffer(b"".join(blobs) + b"\0", np.uint8)
    out_off = np.zeros(n + 1, np.int64)
    status = np.zeros(max(n, 1), np.int32)

    def call(out, cap, c):
        return L.vb200_ogg_mux(n, _ptr(data), at, _ptr(hdr), max_packets, _ptr(npkt), _ptr(info), _ptr(c), _ptr(out),
                               cap, _ptr(out_off), _ptr(status))
    if out_cap is None:
        call(None, 0, carry.copy())
        out_cap = int(out_off[n])
    out = np.zeros(max(out_cap, 1), np.uint8)
    rc = call(out, out_cap, carry)
    if check:
        _check(L, rc)
    fits = int(out_off[n]) <= out_cap
    pages = [out[out_off[s]:out_off[s + 1]].tobytes() if fits else b"" for s in range(n)]
    return {"pages": pages, "carry": carry, "status": status[:n], "out_off": out_off, "rc": rc}


def ogg_mux_dev(nstreams, d_data, data_bytes, d_hdr, max_packets, d_npkt, d_info, d_carry, d_out, out_cap, d_out_off,
                d_status, stream=None):
    """vb200_ogg_mux_dev: device pointers (ints, e.g. torch tensors' data_ptr()), asynchronous on `stream`"""
    L = load()
    _check(L, L.vb200_ogg_mux_dev(nstreams, _ptr(d_data), data_bytes, _ptr(d_hdr), max_packets, _ptr(d_npkt),
                                  _ptr(d_info), _ptr(d_carry), _ptr(d_out), out_cap, _ptr(d_out_off), _ptr(d_status),
                                  _ptr(stream)))
