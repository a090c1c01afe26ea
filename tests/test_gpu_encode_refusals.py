"""The argument checks of the encode entry points, each made in its un-managed and its bitrate-managed form: the
status and the message that vb200_last_error() gives for it.  Every call is refused before any device work, so the
inputs are host arrays even for the _dev forms."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyref
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

VB200_EINVAL = -131                                       # include/vorbis_b200.h
MANAGED_INFO = abi.BitrateInfo(128000, -1, -1, 192000, 0.1, 1.5)


@pytest.fixture
def ctx(cuda_ok):
    from oracle import encode_packets as ep
    if not (pyref.available() and ep.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    d = ep.Driver(2, 44100, 0.5)
    assert d.on_device
    yield d.ctx
    d.close()


def _refused(ctx, rc, what):
    assert rc == VB200_EINVAL
    msg = (ctx.L.vb200_last_error() or b"").decode()
    assert what in msg, msg


def _block_io(ctx, nb, keep, outputs=True):
    """an encode io of nb blocks of the long size, one stream each (host arrays kept alive in keep)"""
    W, ch = 1, ctx.channels
    n = ctx.bs[W] // 2
    arrs = {"pcm": np.zeros((nb, ch, ctx.bs[W]), np.float32), "desc": np.zeros(nb, abi.BLOCKDESC_DTYPE),
            "ampmax_out": np.zeros(nb, np.float32)}
    arrs["desc"]["lW"] = arrs["desc"]["nW"] = 1
    if outputs:
        arrs.update(posts=np.zeros((abi.PACKETBLOBS, nb, ch, abi.FLOOR1_STRIDE), np.int32),
                    nonzero=np.zeros((abi.PACKETBLOBS, nb, ch), np.int32),
                    iwork=np.zeros((abi.PACKETBLOBS, nb, ch, n), np.int32))
    keep.extend(arrs.values())
    io = abi.EncodeIO()
    io.independent = 1
    for k, v in arrs.items():
        setattr(io, k, v.ctypes.data)
    return io


def _streams_io(ctx, keep, outputs=True):
    """a streams io of one stream with both sizes' capacity (host arrays kept alive in keep)"""
    ch, stride, mb = ctx.channels, 4 * ctx.bs[1], 64
    arrs = {"pcm": np.zeros((1, ch, stride), np.float32), "pcm_len": np.full(1, stride, np.int64),
            "plan": np.zeros((1, mb), abi.STREAM_BLOCK_DTYPE), "nblocks": np.zeros(1, np.int32)}
    io = abi.StreamsIO()
    io.pcm_fmt, io.max_blocks, io.stream_stride = lib.PCM_F32_PLANAR, mb, stride
    for w in range(2):
        io.cap[w] = mb
        if outputs:
            n = ctx.bs[w] // 2
            o = [np.zeros((abi.PACKETBLOBS, mb, ch, abi.FLOOR1_STRIDE), np.int32),
                 np.zeros((abi.PACKETBLOBS, mb, ch), np.int32), np.zeros((abi.PACKETBLOBS, mb, ch, n), np.int32),
                 np.zeros(mb, np.float32)]
            keep.extend(o)
            io.posts[w], io.nonzero[w], io.iwork[w], io.ampmax_out[w] = (a.ctypes.data for a in o)
    keep.extend(arrs.values())
    for k, v in arrs.items():
        setattr(io, k, v.ctypes.data)
    return io


def test_block_packets(ctx):
    """vb200_encode_packets[_managed] stage their own outputs and refuse an io that gives posts"""
    keep = []
    io = _block_io(ctx, 2, keep, outputs=False)
    io.posts = keep[0].ctypes.data
    info = [np.zeros(2 * abi.PACKETBLOBS, t) for t in (np.int64, np.int32, np.uint8)]
    ptrs = [a.ctypes.data for a in info]
    _refused(ctx, ctx.L.vb200_encode_packets(ctx.h, 1, 2, 1, 7, C.byref(io), *ptrs, info[2].size),
             "encode_packets: posts / nonzero / iwork / classes / overflow / spectra must be NULL")
    _refused(ctx, ctx.L.vb200_encode_packets_managed(ctx.h, 1, 2, 1, C.byref(io), *ptrs, info[2].size),
             "encode_packets_managed: posts / nonzero / iwork / classes / overflow / spectra must be NULL")
    io.posts = None
    _refused(ctx, ctx.L.vb200_encode_packets(ctx.h, 1, 2, 1, abi.PACKETBLOBS, C.byref(io), *ptrs, info[2].size),
             "blobno")


def test_block_chain(ctx):
    """the managed chain writes int32 residue and does not classify; the un-managed one refuses a bad blobno"""
    keep = []
    io = _block_io(ctx, 2, keep)
    overflow = np.zeros(2, np.int32)
    classes = np.zeros((2, ctx.channels, 64), np.int32)
    io.iwork_fmt, io.overflow = lib.IWORK_S16, overflow.ctypes.data
    _refused(ctx, ctx.L.vb200_encode_dsp_managed(ctx.h, 1, 2, 1, C.byref(io)), "managed mode writes int32 residue")
    _refused(ctx, ctx.L.vb200_encode_dsp_managed_dev(ctx.h, 1, 2, 1, C.byref(io), None),
             "managed mode writes int32 residue")
    io.iwork_fmt, io.overflow = lib.IWORK_S32, None
    io.classes, io.class_stride = classes.ctypes.data, classes.shape[2]
    _refused(ctx, ctx.L.vb200_encode_dsp_managed(ctx.h, 1, 2, 1, C.byref(io)), "managed mode does not classify")
    _refused(ctx, ctx.L.vb200_encode_dsp_managed_dev(ctx.h, 1, 2, 1, C.byref(io), None),
             "managed mode does not classify")
    io.classes = None
    _refused(ctx, ctx.L.vb200_encode_dsp(ctx.h, 1, 2, 1, -1, C.byref(io)), "blobno")


def test_streams_dev(ctx):
    """the device streams calls: a bad blobno (un-managed), and cap > 0 without that size's outputs"""
    keep = []
    io = _streams_io(ctx, keep)
    _refused(ctx, ctx.L.vb200_encode_streams_dev(ctx.h, 1, abi.PACKETBLOBS, C.byref(io), None), "blobno")
    io.iwork[1] = None
    _refused(ctx, ctx.L.vb200_encode_streams_dev(ctx.h, 1, 7, C.byref(io), None),
             "encode_streams: outputs of a size with capacity > 0")
    _refused(ctx, ctx.L.vb200_encode_streams_managed_dev(ctx.h, 1, C.byref(io), None),
             "encode_streams: outputs of a size with capacity > 0")


def test_streams_host(ctx):
    """the host streams calls, with and without packets: a null pcm, and outputs the packet calls stage themselves"""
    ctx.bitrate_setup(MANAGED_INFO)
    keep = []
    io = _streams_io(ctx, keep)
    io.pcm = None
    _refused(ctx, ctx.L.vb200_encode_streams(ctx.h, 1, 7, C.byref(io)), "encode_streams: pcm, pcm_len, plan, nblocks")
    _refused(ctx, ctx.L.vb200_encode_streams_managed(ctx.h, 1, C.byref(io)),
             "encode_streams: pcm, pcm_len, plan, nblocks")
    info = np.zeros(io.max_blocks, abi.PACKET_INFO_DTYPE)
    data = np.zeros(1 << 16, np.uint8)
    pk = (info.ctypes.data, data.ctypes.data, data.size)
    io = _streams_io(ctx, keep, outputs=False)
    io.pcm = None
    _refused(ctx, ctx.L.vb200_encode_streams_packets(ctx.h, 1, 7, C.byref(io), *pk),
             "encode_streams_packets: pcm, pcm_len, plan, nblocks")
    _refused(ctx, ctx.L.vb200_encode_streams_packets_managed(ctx.h, 1, C.byref(io), *pk),
             "encode_streams_packets: pcm, pcm_len, plan, nblocks")
    io = _streams_io(ctx, keep, outputs=False)
    io.posts[1] = data.ctypes.data
    _refused(ctx, ctx.L.vb200_encode_streams_packets(ctx.h, 1, 7, C.byref(io), *pk),
             "encode_streams_packets: posts / nonzero / iwork / ampmax_out must be NULL")
    _refused(ctx, ctx.L.vb200_encode_streams_packets_managed(ctx.h, 1, C.byref(io), *pk),
             "encode_streams_packets: posts / nonzero / iwork / ampmax_out must be NULL")


def test_entropy_dev(ctx):
    """both device entropy coders refuse a pkt_stride below the packet bound or not a multiple of 4; the managed one
    refuses curves closer together than the blocks they hold"""
    bound = ctx.packet_bound(1)
    for stride in (bound - 4, bound + 2):
        _refused(ctx, ctx.L.vb200_encode_entropy_dev(ctx.h, 1, 1, None, None, None, None, stride, None, None, None),
                 "pkt_stride: a multiple of 4, >= the packet bound")
        _refused(ctx, ctx.L.vb200_encode_entropy_managed_dev(ctx.h, 1, 1, 1, None, None, None, None, stride, None, None,
                                                             None),
                 "pkt_stride: a multiple of 4, >= the packet bound")
    _refused(ctx, ctx.L.vb200_encode_entropy_managed_dev(ctx.h, 1, 2, 1, None, None, None, None, bound, None, None,
                                                         None),
             "blob_blocks < nblocks")
