"""vb200_decode_entropy_setup and vb200_encode_entropy_setup check one floor / residue description in one order.  Each
single-fault edit of a stock stream's setup (44.1 kHz stereo, q 0.5) is made twice: to the decoder's setup
(vb200md_entropy_new) and to the encoder's (vb200ms_entropy_setup_build).  Both calls refuse it with the same status
and the same vb200_last_error() text, apart from the coder's name.  After every refusal the registered tables still
decode the stream to the reference's staging and encode its blocks to the stock encoder's packets."""
import ctypes as C

import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode, decode_packets as dp, headers as H, pyref
from test_gpu_encode_packets import _capture, _desc
from vorbis_b200 import abi

pytestmark = pytest.mark.gpu

CH, RATE, Q = 2, 44100, 0.5
EINVAL, EIMPL = -131, -130
INT32_MAX = 2 ** 31 - 1


def _floor(e):
    return e.floor[1][0]


def _res(e):
    return e.residue[1][0]


def _class(e):
    """a class with class_subs > 0 that the long block's first floor uses"""
    f = _floor(e)
    return next(c for c in (f.partitionclass[i] for i in range(f.partitions)) if f.class_subs[c] > 0)


def _stage(e):
    r = _res(e)
    return next((c, s) for c in range(r.partitions) for s in range(8) if r.stagebook[c][s] >= 0)


def _set_stage(e, b):
    c, s = _stage(e)
    _res(e).stagebook[c][s] = b


# (id, status, message: one text with {verb} = decode / encode, or a (decoder, encoder) pair, edit of the setup)
CASES = [
    ("nbooks", EINVAL, ("entropy setup", "encode entropy setup"), lambda e: setattr(e, "nbooks", -1)),
    ("modebits", EINVAL, "modebits", lambda e: setattr(e, "modebits", 9)),
    ("floor_type", EIMPL, "only floor type 1 {verb}s on the device", lambda e: setattr(_floor(e), "type", 0)),
    ("floor_partitions", EINVAL, "floor partitions", lambda e: setattr(_floor(e), "partitions", 32)),
    ("floor_partition_class", EINVAL, "floor partition class",
     lambda e: _floor(e).partitionclass.__setitem__(0, 16)),
    ("floor_class_dim", EINVAL, "floor class dim / subs",
     lambda e: _floor(e).class_dim.__setitem__(_class(e), 9)),
    ("floor_class_dim_int32_max", EINVAL, "floor class dim / subs",
     lambda e: _floor(e).class_dim.__setitem__(_class(e), INT32_MAX)),
    ("floor_class_subs", EINVAL, "floor class dim / subs",
     lambda e: _floor(e).class_subs.__setitem__(_class(e), 4)),
    ("floor_posts", EINVAL, "floor partitions do not give the floor's posts",
     lambda e: setattr(_floor(e), "partitions", _floor(e).partitions - 1)),
    ("floor_class_book", EINVAL, "floor class book",
     lambda e: _floor(e).class_book.__setitem__(_class(e), e.nbooks)),
    ("floor_subclass_book", EINVAL, "floor subclass book",
     lambda e: _floor(e).class_subbook[_class(e)].__setitem__(0, e.nbooks)),
    ("residue_type0", EIMPL, "residue type 0 does not {verb} on the device", lambda e: setattr(_res(e), "type", 0)),
    ("residue_type", EINVAL, "residue type", lambda e: setattr(_res(e), "type", 3)),
    ("residue_begin", EINVAL, "residue begin / end / grouping do not fit the block",
     lambda e: (setattr(_res(e), "begin", 1 << 20), setattr(_res(e), "end", 1 << 20))),
    ("residue_groupbook", EINVAL, "residue partitions / groupbook", lambda e: setattr(_res(e), "groupbook", e.nbooks)),
    ("residue_partvals", EINVAL, "residue partvals != partitions ^ dim(groupbook)",
     lambda e: setattr(_res(e), "partvals", _res(e).partvals + 1)),
    ("residue_stage_book", EINVAL, "residue stage book", lambda e: _set_stage(e, e.nbooks)),
]


@pytest.fixture(scope="module")
def coders(cuda_ok):
    """the stock stream's decoder (its setup from vb200md_entropy_new registered, a copy of that setup, the packets
    and the reference's staging of them) and encoder (its setup registered, a copy, blocks and the stock packets)"""
    from oracle import encode_packets as ep
    if not (H.available() and decode.available() and dp.available() and pyref.available() and ep.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    pcm = probe_signal(CH, RATE, 0.5, seed=21)
    p = decode.encode(CH, RATE, Q, pcm)
    hdr = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:3, :2]]
    L = H._lib()
    rc, why = C.c_int(0), C.c_int(0)
    rh = L.rh_open(hdr[0], len(hdr[0]), hdr[1], len(hdr[1]), hdr[2], len(hdr[2]), C.byref(rc), C.byref(why))
    assert rh and rc.value == 0 and why.value == 0
    dec = dp.Driver(p)
    enc = ep.Driver(CH, RATE, Q)
    try:
        assert dec.on_device and enc.on_device
        pkts = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.audio[:40, :2]]
        W = dp.ref_headers(p, pkts)
        staging = dp.ref_staging(p, pkts, W, dec.bs, dec.channels)
        cap, want = _capture(CH, RATE, Q, pcm)
        sel = np.nonzero(cap["W"] == 1)[0][:8]
        blocks = np.ascontiguousarray(cap["pcm"][sel][:, :, :enc.ctx.bs[1]])
        mask = np.zeros(len(cap["W"]), bool)
        mask[sel] = True
        es_enc, books = enc.setup_copy()
        yield {"dec": dec, "es_dec": abi.EntropySetup.from_buffer_copy(L.rh_entropy(rh).contents), "pkts": pkts,
               "W": W, "staging": staging, "enc": enc, "es_enc": es_enc, "books": books, "blocks": blocks,
               "desc": _desc(cap, mask), "packets": [want[i] for i in sel]}
    finally:
        dec.close()
        enc.close()
        L.rh_close(rh)


def _refusal(ctx, call, es, edit):
    e = type(es).from_buffer_copy(es)
    edit(e)
    rc = call(ctx.h, C.byref(e))
    return rc, (ctx.L.vb200_last_error() or b"").decode()


@pytest.mark.parametrize("name,status,msg,edit", CASES, ids=[c[0] for c in CASES])
def test_both_coders_refuse_and_keep_their_tables(coders, name, status, msg, edit):
    k = coders
    dec, enc = k["dec"].ctx, k["enc"].ctx
    for i, (ctx, call, es, verb) in enumerate(((dec, dec.L.vb200_decode_entropy_setup, k["es_dec"], "decode"),
                                               (enc, enc.L.vb200_encode_entropy_setup, k["es_enc"], "encode"))):
        want = msg[i] if isinstance(msg, tuple) else msg.format(verb=verb)
        assert _refusal(ctx, call, es, edit) == (status, want), verb
    got = dp.dev_staging(dec, k["pkts"], k["W"], k["dec"].bs, k["dec"].channels)
    for a, b in zip(k["staging"], got):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "decode after a refused " + name
    assert enc.encode_packets(1, k["blocks"], k["desc"])["packets"] == k["packets"], "encode after a refused " + name
