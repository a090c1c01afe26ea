"""ctypes mirrors of the plain-C structs in include/vorbis_b200.h.

These are shared by the loader of the product library (libvorbis_b200.so), by the
test-only loaders of the CPU oracle (oracle/libvb_oracle.so) and of the compiled
reference (oracle/_ref/libvorbis_ref.so), and by the golden-fixture reader.
Field order and types must match the header exactly.
"""
import ctypes as C
import numpy as np

P_BANDS = 17
P_LEVELS = 8
P_NOISECURVES = 3
EHMER_MAX = 56
COMPAND_LEVELS = 40
PACKETBLOBS = 15
MAX_COUPLING = 256
MAX_CHANNELS = 255
MAX_SUBMAPS = 4
VE_BANDS = 7
VE_FILTER_WORDS = 36


def ve_state_words(ch):
    return 1 + VE_FILTER_WORDS * VE_BANDS * ch

FLOOR1_STRIDE = 65

c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)
c_int64_p = C.POINTER(C.c_int64)


class PsySetup(C.Structure):
    _fields_ = [
        ("n", C.c_int32),
        ("blockflag", C.c_int32),
        ("ath_adjatt", C.c_float),
        ("ath_maxatt", C.c_float),
        ("tone_masteratt", C.c_float * P_NOISECURVES),
        ("tone_abs_limit", C.c_float),
        ("noisemaxsupp", C.c_float),
        ("noisewindowfixed", C.c_int32),
        ("noisecompand", C.c_float * COMPAND_LEVELS),
        ("max_curve_dB", C.c_float),
        ("normal_p", C.c_int32),
        ("normal_start", C.c_int32),
        ("normal_partition", C.c_int32),
        ("normal_thresh", C.c_double),
        ("firstoc", C.c_int32),
        ("shiftoc", C.c_int32),
        ("eighth_octave_lines", C.c_int32),
        ("total_octave_lines", C.c_int32),
        ("m_val", C.c_float),
        ("ath", c_float_p),
        ("octave", c_int32_p),
        ("bark", c_int32_p),
        ("tonecurves", c_float_p),
        ("noiseoffset", c_float_p),
    ]


VIF_POSIT = 63


class Floor1Setup(C.Structure):
    _fields_ = [
        ("posts", C.c_int32),
        ("postlist", C.c_int32 * (VIF_POSIT + 2)),
        ("mult", C.c_int32),
        ("n", C.c_int32),
        ("maxover", C.c_float), ("maxunder", C.c_float), ("maxerr", C.c_float),
        ("twofitweight", C.c_float), ("twofitatten", C.c_float),
    ]


class ResidueSetup(C.Structure):
    _fields_ = [
        ("type", C.c_int32), ("begin", C.c_int32), ("end", C.c_int32), ("grouping", C.c_int32),
        ("partitions", C.c_int32), ("classmetric1", C.c_int32 * 64), ("classmetric2", C.c_int32 * 64),
    ]


class Setup(C.Structure):
    _fields_ = [
        ("channels", C.c_int32),
        ("rate", C.c_int32),
        ("blocksizes", C.c_int32 * 2),
        ("n_psy", C.c_int32),
        ("psy", PsySetup * 4),
        ("ampmax_att_per_sec", C.c_float),
        ("coupling_pointlimit", (C.c_int32 * PACKETBLOBS) * 2),
        ("coupling_prepointamp", C.c_int32 * PACKETBLOBS),
        ("coupling_postpointamp", C.c_int32 * PACKETBLOBS),
        ("sliding_lowpass", (C.c_int32 * PACKETBLOBS) * 2),
        ("coupling_steps", C.c_int32 * 2),
        ("coupling_mag", (C.c_int32 * MAX_COUPLING) * 2),
        ("coupling_ang", (C.c_int32 * MAX_COUPLING) * 2),
        ("window", c_float_p * 2),
        ("submaps", C.c_int32 * 2),
        ("chmux", (C.c_uint8 * (MAX_CHANNELS + 1)) * 2),
        ("floor1", (Floor1Setup * MAX_SUBMAPS) * 2),
        ("preecho_thresh", C.c_float * VE_BANDS),
        ("postecho_thresh", C.c_float * VE_BANDS),
        ("stretch_penalty", C.c_float),
        ("preecho_minenergy", C.c_float),
        ("residue", (ResidueSetup * MAX_SUBMAPS) * 2),
    ]


class BlockDesc(C.Structure):
    _fields_ = [
        ("lW", C.c_int32),
        ("nW", C.c_int32),
        ("blocktype", C.c_int32),
        ("ampmax", C.c_float),
    ]


BLOCKDESC_DTYPE = np.dtype(
    [("lW", np.int32), ("nW", np.int32), ("blocktype", np.int32), ("ampmax", np.float32)]
)
assert BLOCKDESC_DTYPE.itemsize == C.sizeof(BlockDesc)


STREAM_BLOCK_DTYPE = np.dtype([("pos", "<i4"), ("slot", "<i4"), ("W", "<i4"), ("lW", "<i4"), ("nW", "<i4"),
                               ("blocktype", "<i4")])      # vb200_stream_block


class PhaseAIO(C.Structure):
    _fields_ = [
        ("pcm", C.c_void_p),
        ("desc", C.c_void_p),
        ("mdct", C.c_void_p),
        ("logmdct", C.c_void_p),
        ("logmask", C.c_void_p),
        ("ampmax_out", C.c_void_p),
        ("tap_noise", C.c_void_p),
        ("tap_tone", C.c_void_p),
        ("tap_logfft", C.c_void_p),
        ("tap_mdct_raw", C.c_void_p),
    ]

class EncodeIO(C.Structure):
    """vb200_encode_io (include/vorbis_b200.h)"""
    _fields_ = [
        ("pcm", C.c_void_p),
        ("pcm_fmt", C.c_int32),
        ("hop", C.c_int32),
        ("stream_stride", C.c_int64),
        ("desc", C.c_void_p),
        ("ampmax0", C.c_void_p),
        ("independent", C.c_int32),
        ("iwork_fmt", C.c_int32),
        ("posts", C.c_void_p),
        ("nonzero", C.c_void_p),
        ("iwork", C.c_void_p),
        ("ampmax_out", C.c_void_p),
        ("mdct", C.c_void_p),
        ("logmdct", C.c_void_p),
        ("logmask", C.c_void_p),
        ("overflow", C.c_void_p),
        ("classes", C.c_void_p),
        ("class_stride", C.c_int64),
    ]


class StreamsIO(C.Structure):
    """vb200_streams_io (include/vorbis_b200.h)"""
    _fields_ = [
        ("pcm", C.c_void_p),
        ("pcm_fmt", C.c_int32),
        ("max_blocks", C.c_int32),
        ("stream_stride", C.c_int64),
        ("pcm_len", C.c_void_p),
        ("eof", C.c_void_p),
        ("plan", C.c_void_p),
        ("nblocks", C.c_void_p),
        ("cap", C.c_int32 * 2),
        ("count", C.c_int32 * 2),
        ("posts", C.c_void_p * 2),
        ("nonzero", C.c_void_p * 2),
        ("iwork", C.c_void_p * 2),
        ("ampmax_out", C.c_void_p * 2),
    ]


class PcmIO(C.Structure):
    """vb200_pcm_io (include/vorbis_b200.h)"""
    _fields_ = [
        ("pcm", C.c_void_p),
        ("pcm_fmt", C.c_int32),
        ("max_blocks", C.c_int32),
        ("stream_stride", C.c_int64),
        ("pcm_len", C.c_void_p),
        ("end", C.c_void_p),
        ("plan", C.c_void_p),
        ("nblocks", C.c_void_p),
        ("cap", C.c_int32 * 2),
        ("count", C.c_int32 * 2),
    ]


class BitrateInfo(C.Structure):
    """vb200_bitrate_info (include/vorbis_b200.h): bitrate_manager_info, lib/bitrate.h:41-50"""
    _fields_ = [
        ("avg_rate", C.c_int64),
        ("min_rate", C.c_int64),
        ("max_rate", C.c_int64),
        ("reservoir_bits", C.c_int64),
        ("reservoir_bias", C.c_double),
        ("slew_damp", C.c_double),
    ]


BITRATE_STATE_DTYPE = np.dtype([("avg_reservoir", "<i8"), ("minmax_reservoir", "<i8"), ("avgfloat", "<f8"),
                                ("choice", "<i4"), ("pad", "<i4")])           # vb200_bitrate_state
PACKET_INFO_DTYPE = np.dtype([("offset", "<i8"), ("granulepos", "<i8"), ("bytes", "<i4"), ("e_o_s", "<i4"),
                              ("packetno", "<i4"), ("choice", "<i4")])         # vb200_packet_info
assert C.sizeof(BitrateInfo) == 48 and BITRATE_STATE_DTYPE.itemsize == 32 and PACKET_INFO_DTYPE.itemsize == 32
# vb200_encode_carry: the public head of every stream's carry ([nstreams][vb200_encode_carry_bytes] bytes)
ENCODE_CARRY_HEAD_DTYPE = np.dtype([("base", "<i8"), ("granulepos", "<i8"), ("packetno", "<i4"), ("done", "<i4")])
assert ENCODE_CARRY_HEAD_DTYPE.itemsize == 24
# vb200_pcm_carry: the public head of every raw-PCM carry ([nstreams][vb200_encode_pcm_carry_bytes] bytes)
PCM_CARRY_HEAD_DTYPE = np.dtype([("enc", ENCODE_CARRY_HEAD_DTYPE), ("raw_base", "<i8"), ("written", "<i8"),
                                 ("ended", "<i4"), ("drained", "<i4")])
assert PCM_CARRY_HEAD_DTYPE.itemsize == 48
# vb200_encode_result: what a _dev packet call reports on the device
ENCODE_RESULT_DTYPE = np.dtype([("bytes", "<i8"), ("count", "<i4", (2,)), ("rc", "<i4"), ("pad", "<i4")])
assert ENCODE_RESULT_DTYPE.itemsize == 24
# vb200_decoded_packet: what vb200_decode_streams_packets reports for every packet it was given
DECODED_PACKET_DTYPE = np.dtype([("pcm_offset", "<i8"), ("granulepos", "<i8"), ("samples", "<i4"), ("status", "<i4")])
assert DECODED_PACKET_DTYPE.itemsize == 24
# vb200_pcm_range: one request of vb200_decode_ranges, samples [start, start + length) of stream `stream`
PCM_RANGE_DTYPE = np.dtype([("start", "<i8"), ("stream", "<i4"), ("length", "<i4")])
assert PCM_RANGE_DTYPE.itemsize == 16
# vb200_ogg_stream: what vb200_ogg_demux reports per file
OGG_STREAM_DTYPE = np.dtype([("status", "<i4"), ("serial", "<u4"), ("pages", "<i4"), ("dropped", "<i4"),
                             ("holes", "<i4"), ("foreign", "<i4"), ("chained", "<i4"), ("pad", "<i4"),
                             ("hdr_offset", "<i8", (3,)), ("hdr_bytes", "<i4", (3,)), ("pad2", "<i4")])
assert OGG_STREAM_DTYPE.itemsize == 72 and OGG_STREAM_DTYPE.fields["hdr_offset"][1] == 32


class Codebook(C.Structure):
    """vb200_codebook (include/vorbis_b200.h)"""
    _fields_ = [
        ("dim", C.c_int32),
        ("used", C.c_int32),
        ("length", C.c_void_p),
        ("bits", C.c_void_p),
        ("entry", C.c_void_p),
        ("value", C.c_void_p),
    ]


class FloorDecode(C.Structure):
    """vb200_floor_decode"""
    _fields_ = [
        ("type", C.c_int32),
        ("partitions", C.c_int32),
        ("partitionclass", C.c_int32 * 31),
        ("class_dim", C.c_int32 * 16),
        ("class_subs", C.c_int32 * 16),
        ("class_book", C.c_int32 * 16),
        ("class_subbook", (C.c_int32 * 8) * 16),
    ]


class ResidueDecode(C.Structure):
    """vb200_residue_decode"""
    _fields_ = [
        ("type", C.c_int32),
        ("begin", C.c_int32),
        ("end", C.c_int32),
        ("grouping", C.c_int32),
        ("partitions", C.c_int32),
        ("partvals", C.c_int32),
        ("groupbook", C.c_int32),
        ("stagebook", (C.c_int32 * 8) * 64),
    ]


class EntropySetup(C.Structure):
    """vb200_entropy_setup"""
    _fields_ = [
        ("nbooks", C.c_int32),
        ("books", C.POINTER(Codebook)),
        ("modebits", C.c_int32),
        ("floor", (FloorDecode * MAX_SUBMAPS) * 2),
        ("residue", (ResidueDecode * MAX_SUBMAPS) * 2),
    ]


class VorbisHeaders(C.Structure):
    """vb200_vorbis_headers: what vb200_vorbis_headers_parse returns"""
    _fields_ = [
        ("channels", C.c_int32), ("rate", C.c_int32), ("bitrate_upper", C.c_int32), ("bitrate_nominal", C.c_int32),
        ("bitrate_lower", C.c_int32), ("blocksizes", C.c_int32 * 2), ("pad", C.c_int32),
        ("setup", Setup),
        ("entropy", EntropySetup),
    ]


assert VorbisHeaders.setup.offset == 32 and VorbisHeaders.entropy.offset == 32 + C.sizeof(Setup)
# vb200_file_group: one group of vb200_ogg_group
FILE_GROUP_DTYPE = np.dtype([("first", "<i4"), ("files", "<i4"), ("rep", "<i4")])
assert FILE_GROUP_DTYPE.itemsize == 12
# vb200_ogg_mux_carry: one stream's page state between vb200_ogg_mux calls
OGG_MUX_CARRY_DTYPE = np.dtype([("serial", "<u4"), ("pageno", "<u4"), ("state", "<i4"), ("kept", "<i4"),
                                ("kept_segs", "<i4"), ("pad", "<i4")])
assert OGG_MUX_CARRY_DTYPE.itemsize == 24 and OGG_MUX_CARRY_DTYPE.fields["kept_segs"][1] == 16


class EncCodebook(C.Structure):
    """vb200_enc_codebook"""
    _fields_ = [
        ("dim", C.c_int32),
        ("entries", C.c_int32),
        ("length", C.c_void_p),
        ("codeword", C.c_void_p),
        ("minval", C.c_int32),
        ("delta", C.c_int32),
        ("quantvals", C.c_int32),
    ]


class EncodeEntropySetup(C.Structure):
    """struct vb200_encode_entropy_setup"""
    _fields_ = [
        ("nbooks", C.c_int32),
        ("books", C.POINTER(EncCodebook)),
        ("modebits", C.c_int32),
        ("floor", (FloorDecode * MAX_SUBMAPS) * 2),
        ("residue", (ResidueDecode * MAX_SUBMAPS) * 2),
    ]


class DecodeCarry(C.Structure):
    """vb200_decode_carry (include/vorbis_b200.h): tail [nstreams][ch][blocksizes[1]/2] float32, W [nstreams][ch]
    int32 (-1 = nothing decoded yet)"""
    _fields_ = [
        ("tail", C.c_void_p),
        ("W", C.c_void_p),
    ]


_PSY_SCALARS = [
    "n", "blockflag", "ath_adjatt", "ath_maxatt", "tone_abs_limit", "noisemaxsupp",
    "noisewindowfixed", "max_curve_dB", "normal_p", "normal_start", "normal_partition",
    "normal_thresh", "firstoc", "shiftoc", "eighth_octave_lines", "total_octave_lines", "m_val",
]


def _sc(v):
    """scalar out of a 0-d / 1-element numpy array (npz round trip)"""
    return np.asarray(v).reshape(-1)[0].item()


def _np_ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


def halfrate_window_ptrs(windows):
    """the `const float *const window[2]` argument of vb200_synthesis_halfrate (and of the oracle's counterpart):
    returns (what must stay alive during the call, pointer).  windows None: (None, NULL) = closed form."""
    if windows is None:
        return None, None
    arrs = [np.ascontiguousarray(w, np.float32) for w in windows]
    ptrs = (c_float_p * 2)(*[_np_ptr(a, C.c_float) for a in arrs])
    return (arrs, ptrs), C.cast(ptrs, C.c_void_p)


class SetupHolder:
    """Owns numpy copies of every table a `Setup` points to (so the ctypes struct
    stays valid), and converts to / from a flat dict of arrays (npz fixtures)."""

    def __init__(self, arrays):
        self.arrays = {k: np.ascontiguousarray(v) for k, v in arrays.items()}
        self.c = Setup()
        a = self.arrays
        s = self.c
        s.channels = int(_sc(a["channels"]))
        s.rate = int(_sc(a["rate"]))
        s.blocksizes[0], s.blocksizes[1] = [int(x) for x in a["blocksizes"]]
        s.n_psy = int(_sc(a["n_psy"]))
        s.ampmax_att_per_sec = float(_sc(a["ampmax_att_per_sec"]))
        for w in range(2):
            for k in range(PACKETBLOBS):
                s.coupling_pointlimit[w][k] = int(a["coupling_pointlimit"][w][k])
                s.sliding_lowpass[w][k] = int(a["sliding_lowpass"][w][k])
            s.coupling_steps[w] = int(a["coupling_steps"][w])
            for k in range(int(a["coupling_steps"][w])):
                s.coupling_mag[w][k] = int(a["coupling_mag"][w][k])
                s.coupling_ang[w][k] = int(a["coupling_ang"][w][k])
        for k in range(PACKETBLOBS):
            s.coupling_prepointamp[k] = int(a["coupling_prepointamp"][k])
            s.coupling_postpointamp[k] = int(a["coupling_postpointamp"][k])
        for w in range(2):
            key = "window%d" % w
            if key in a and a[key].size:
                a[key] = np.ascontiguousarray(a[key], dtype=np.float32)
                s.window[w] = _np_ptr(a[key], C.c_float)
        for w in range(2):
            key = "halfrate_window%d" % w
            if key in a:
                a[key] = np.ascontiguousarray(a[key], dtype=np.float32)
        if "chmux" in a:
            cm = np.asarray(a["chmux"]).astype(np.int64)
            for w in range(2):
                s.submaps[w] = int(a["submaps"][w])
                for k in range(cm.shape[1]):
                    s.chmux[w][k] = int(cm[w][k])
        for w in range(2):
            for sm in range(MAX_SUBMAPS):
                s.residue[w][sm].type = -1
                pre = "residue_%d_%d_" % (w, sm)
                if pre + "type" not in a:
                    continue
                rs = s.residue[w][sm]
                for nm in ("type", "begin", "end", "grouping", "partitions"):
                    setattr(rs, nm, int(_sc(a[pre + nm])))
                for k in range(64):
                    rs.classmetric1[k] = int(a[pre + "classmetric1"][k])
                    rs.classmetric2[k] = int(a[pre + "classmetric2"][k])
        if "env_preecho_thresh" in a:
            for k in range(VE_BANDS):
                s.preecho_thresh[k] = float(a["env_preecho_thresh"][k])
                s.postecho_thresh[k] = float(a["env_postecho_thresh"][k])
            s.stretch_penalty = float(_sc(a["env_stretch_penalty"]))
            s.preecho_minenergy = float(_sc(a["env_preecho_minenergy"]))
        for w in range(2):
            for sm in range(MAX_SUBMAPS):
                key = "floor1_%d_%d_postlist" % (w, sm)
                if key not in a:
                    continue
                f = s.floor1[w][sm]
                pl = np.asarray(a[key]).astype(np.int64)
                f.posts = len(pl)
                for k, v in enumerate(pl):
                    f.postlist[k] = int(v)
                pre = "floor1_%d_%d_" % (w, sm)
                f.mult = int(_sc(a[pre + "mult"]))
                f.n = int(_sc(a[pre + "n"]))
                for nm in ("maxover", "maxunder", "maxerr", "twofitweight", "twofitatten"):
                    setattr(f, nm, float(_sc(a[pre + nm])))
        for i in range(s.n_psy):
            p = s.psy[i]
            pre = "psy%d_" % i
            for name in _PSY_SCALARS:
                v = _sc(a[pre + name])
                setattr(p, name, float(v) if name in ("ath_adjatt", "ath_maxatt", "tone_abs_limit",
                                                      "noisemaxsupp", "max_curve_dB", "normal_thresh",
                                                      "m_val") else int(v))
            for j in range(P_NOISECURVES):
                p.tone_masteratt[j] = float(a[pre + "tone_masteratt"][j])
            for j in range(COMPAND_LEVELS):
                p.noisecompand[j] = float(a[pre + "noisecompand"][j])
            for name, ct, dt in (("ath", C.c_float, np.float32), ("octave", C.c_int32, np.int32),
                                 ("bark", C.c_int32, np.int32), ("tonecurves", C.c_float, np.float32),
                                 ("noiseoffset", C.c_float, np.float32)):
                a[pre + name] = np.ascontiguousarray(a[pre + name], dtype=dt)
                setattr(p, name, _np_ptr(a[pre + name], ct))

    # ---- conveniences -------------------------------------------------------
    @property
    def channels(self):
        return int(self.c.channels)

    @property
    def rate(self):
        return int(self.c.rate)

    def blocksize(self, W):
        return int(self.c.blocksizes[W])

    def psy_n(self, look):
        return int(self.c.psy[look].n)

    def floor_of(self, W, channel):
        return int(self.c.chmux[W][channel])

    def floor_posts(self, W, sel=0):
        return int(self.c.floor1[W][sel].posts)

    def halfrate_windows(self):
        """[w0, w1] the half windows of the block sizes blocksizes[w]/2 (blocksizes[w]/4 floats each, what
        _vorbis_window_get(b->window[w]-1) returns) where the arrays hold them (keys halfrate_window0/1),
        else None; the window argument of vb200_synthesis_halfrate"""
        if "halfrate_window0" not in self.arrays:
            return None
        return [self.arrays["halfrate_window%d" % w] for w in range(2)]

    def save(self, path):
        np.savez_compressed(path, **self.arrays)

    @classmethod
    def load(cls, path):
        with np.load(path) as z:
            return cls({k: z[k] for k in z.files})

    @classmethod
    def from_struct(cls, s):
        """Deep-copy a C `Setup` (e.g. filled by ref_get_setup) into numpy arrays."""
        a = {
            "channels": np.int32(s.channels), "rate": np.int32(s.rate),
            "blocksizes": np.array([s.blocksizes[0], s.blocksizes[1]], np.int32),
            "n_psy": np.int32(s.n_psy),
            "ampmax_att_per_sec": np.float32(s.ampmax_att_per_sec),
            "coupling_pointlimit": np.array([[s.coupling_pointlimit[w][k] for k in range(PACKETBLOBS)]
                                             for w in range(2)], np.int32),
            "coupling_prepointamp": np.array(list(s.coupling_prepointamp), np.int32),
            "coupling_postpointamp": np.array(list(s.coupling_postpointamp), np.int32),
            "sliding_lowpass": np.array([[s.sliding_lowpass[w][k] for k in range(PACKETBLOBS)]
                                         for w in range(2)], np.int32),
            "coupling_steps": np.array(list(s.coupling_steps), np.int32),
        }
        ms = max(1, max(s.coupling_steps))
        a["coupling_mag"] = np.array([[s.coupling_mag[w][k] for k in range(ms)] for w in range(2)], np.int32)
        a["coupling_ang"] = np.array([[s.coupling_ang[w][k] for k in range(ms)] for w in range(2)], np.int32)
        for w in range(2):
            if s.window[w]:
                a["window%d" % w] = np.ctypeslib.as_array(s.window[w], shape=(s.blocksizes[w] // 2,)).copy()
        for w in range(2):
            for sm in range(MAX_SUBMAPS):
                rs = s.residue[w][sm]
                if rs.type < 0 or rs.grouping <= 0:
                    continue
                pre = "residue_%d_%d_" % (w, sm)
                for nm in ("type", "begin", "end", "grouping", "partitions"):
                    a[pre + nm] = np.int32(getattr(rs, nm))
                a[pre + "classmetric1"] = np.array(list(rs.classmetric1), np.int32)
                a[pre + "classmetric2"] = np.array(list(rs.classmetric2), np.int32)
        a["env_preecho_thresh"] = np.array(list(s.preecho_thresh), np.float32)
        a["env_postecho_thresh"] = np.array(list(s.postecho_thresh), np.float32)
        a["env_stretch_penalty"] = np.float32(s.stretch_penalty)
        a["env_preecho_minenergy"] = np.float32(s.preecho_minenergy)
        a["submaps"] = np.array(list(s.submaps), np.int32)
        a["chmux"] = np.array([[s.chmux[w][k] for k in range(max(1, s.channels))] for w in range(2)], np.int32)
        for w in range(2):
            for sm in range(MAX_SUBMAPS):
                f = s.floor1[w][sm]
                if f.posts <= 0:
                    continue
                pre = "floor1_%d_%d_" % (w, sm)
                a[pre + "postlist"] = np.array([f.postlist[k] for k in range(f.posts)], np.int32)
                a[pre + "mult"] = np.int32(f.mult)
                a[pre + "n"] = np.int32(f.n)
                for nm in ("maxover", "maxunder", "maxerr", "twofitweight", "twofitatten"):
                    a[pre + nm] = np.float64(getattr(f, nm))
        for i in range(s.n_psy):
            p = s.psy[i]
            pre = "psy%d_" % i
            n = p.n
            for name in _PSY_SCALARS:
                v = getattr(p, name)
                a[pre + name] = np.float64(v) if isinstance(v, float) else np.int32(v)
            a[pre + "tone_masteratt"] = np.array(list(p.tone_masteratt), np.float32)
            a[pre + "noisecompand"] = np.array(list(p.noisecompand), np.float32)
            a[pre + "ath"] = np.ctypeslib.as_array(p.ath, shape=(n,)).copy()
            a[pre + "octave"] = np.ctypeslib.as_array(p.octave, shape=(n,)).copy()
            a[pre + "bark"] = np.ctypeslib.as_array(p.bark, shape=(n,)).copy()
            a[pre + "tonecurves"] = np.ctypeslib.as_array(
                p.tonecurves, shape=(P_BANDS * P_LEVELS * (EHMER_MAX + 2),)).copy()
            a[pre + "noiseoffset"] = np.ctypeslib.as_array(p.noiseoffset, shape=(P_NOISECURVES * n,)).copy()
        return cls(a)
