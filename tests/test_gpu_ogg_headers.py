"""Ogg Vorbis files decoded with nothing but this library: vb200_ogg_demux -> vb200_ogg_group -> the group's header
packets copied back -> vb200_vorbis_headers_parse -> a context -> vb200_decode_streams_packets / vb200_decode_ranges.
- a mixed corpus: the four stock setups of test_gpu_ogg.py and the tests/vorbis_gen.py INSIDE setups, three files each
  with its own comment header, interleaved in a seeded order under the three pagings; every file's PCM (float and
  int16, and half rate where blocksizes[0] > 64) equals the stock decoder's bit for bit.  No libvorbis-derived context
  is made: the stock decoder is only the yardstick;
- vb200_ogg_group against a Python reference built from the oracle demux: setup headers that differ in one bit,
  identical setups under different identification headers (rate, channels), a damaged comment header, a file without
  Vorbis and one whose header packets are cut short; files whose tables max_packets cut (VB200_EINVAL) grouped with
  the rest; and a build of the library whose hash keeps two bits, so that collisions decide every group;
- the _dev form equals the host form, and a call is five kernel launches at 1 and at 1000 files (torch.profiler, in a
  process of its own);
- a context from the headers stages the damaged packets of two INSIDE setups exactly as the libvorbis-derived
  driver's context does."""
import struct

import numpy as np
import pytest

from oracle import decode
from oracle import decode_packets as dp
from oracle import decode_streams as ds
from oracle import ogg
from test_gpu_ogg import CASES, PAGINGS, _decode_as_stock, _stock, launched_kernels
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
EBADHEADER, ENOTVORBIS, EINVAL = -133, -132, -131


def _need():
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def comment_packet(tags, vendor=b"vb200 test"):
    out = b"\x03vorbis" + struct.pack("<I", len(vendor)) + vendor + struct.pack("<I", len(tags))
    for t in tags:
        out += struct.pack("<I", len(t)) + t
    return out + b"\x01"


def with_packets(p, ident=None, comment=None, setup=None):
    """p (decode.Packets) with header packets replaced"""
    pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
    for k, new in enumerate((ident, comment, setup)):
        if new is not None:
            pk[k] = new
    meta = p.meta.copy()
    meta[:, 1] = [len(x) for x in pk]
    meta[:, 0] = np.concatenate([[0], np.cumsum(meta[:-1, 1])])
    return decode.Packets(np.frombuffer(b"".join(pk), np.uint8).copy(), meta)


def comment_ok(b):
    """_vorbis_unpack_comment with the packet type and magic, on whole bytes"""
    n = len(b)
    if b[:7] != b"\x03vorbis":
        return False
    at = 7

    def i32(a):
        return struct.unpack("<i", b[a:a + 4])[0] if a + 4 <= n else None
    v = i32(at)
    if v is None or v < 0 or v > n - 8 or at + 4 + v > n:
        return False
    at += 4 + v
    c = i32(at)
    if c is None or c < 0 or c > (n - at - 4) >> 2:
        return False
    at += 4
    for _ in range(c):
        ln = i32(at)
        if ln is None or ln < 0 or ln > n - at - 4:
            return False
        at += 4 + ln
    return at < n and b[at] & 1 == 1


def group_reference(files, max_packets):
    """status, order, groups of vb200_ogg_group from oracle.ogg.demux"""
    rs = [ogg.demux(f, max_packets) for f in files]
    status = []
    for r in rs:
        s = r["status"]
        if s in (0, EINVAL) and not comment_ok(r["hdr_data"][1]):
            s = EBADHEADER
        status.append(s)
    reps = {}
    members = {}
    for f, r in enumerate(rs):
        if status[f] not in (0, EINVAL):
            continue
        key = (r["hdr_data"][0], r["hdr_data"][2])
        reps.setdefault(key, f)
        members.setdefault(reps[key], []).append(f)
    order, groups = [], []
    for rep in sorted(members):
        groups.append((len(order), len(members[rep]), rep))
        order += members[rep]
    order += [f for f in range(len(files)) if status[f] not in (0, EINVAL)]
    return np.array(status), np.array(order), groups


def _check_group(res, g, files, what):
    status, order, groups = group_reference(files, res["info"].shape[1])
    assert (g["status"] == status).all(), "%s: status %s, want %s" % (what, g["status"], status)
    assert (g["order"] == order).all(), "%s: order %s, want %s" % (what, g["order"], order)
    assert [tuple(int(x) for x in row) for row in g["groups"]] == groups, "%s: groups" % what
    for p, f in enumerate(order):
        n = int(res["npkt"][f])
        assert g["npkt"][p] == n
        assert g["info"][p, :n].tobytes() == res["info"][f, :n].tobytes(), "%s: rows of position %d" % (what, p)


def _hdr_bytes(data, st, k):
    return bytes(data[int(st["hdr_offset"][k]):int(st["hdr_offset"][k] + st["hdr_bytes"][k])])


def _mixed_corpus():
    import vorbis_gen as G
    from test_generated_setups_oracle import corpus
    src = [_stock(*c) for c in CASES] + [corpus(name)[2] for name in G.INSIDE]
    rng = np.random.default_rng(20261017)
    files = []
    for si, p in enumerate(src):
        for j in range(3):
            q = with_packets(p, comment=comment_packet([b"TITLE=setup %d copy %d" % (si, j)] * (j + 1)))
            files.append((si, b"".join(ogg.file_of(q, rng, **PAGINGS[j]))))
    perm = rng.permutation(len(files))
    return [files[i] for i in perm], len(src)


def test_mixed_corpus_end_to_end(cuda_ok):
    _need()
    files, nsetups = _mixed_corpus()
    blobs = [b for _, b in files]
    res = lib.ogg_demux(blobs)
    assert (res["streams"]["status"] == 0).all()
    g = lib.ogg_group(res)
    _check_group(res, g, blobs, "mixed")
    assert len(g["groups"]) == nsetups
    mp = res["info"].shape[1]
    for first, nf, rep in g["groups"].tolist():
        assert len({files[int(f)][0] for f in g["order"][first:first + nf]}) == 1, "a group mixes setups"
        st = res["streams"][rep]
        h = lib.vorbis_headers(*[_hdr_bytes(res["data"], st, k) for k in range(3)])
        ctx = h.context()
        sub = {"data": res["data"], "npkt": g["npkt"][first:first + nf], "info": g["info"][first:first + nf],
               "streams": res["streams"][g["order"][first:first + nf]]}
        assert sub["info"].shape[1] == mp
        what = "group of file %d" % rep
        _decode_as_stock(ctx, sub, list(range(nf)), h.channels, what)
        if ctx.bs[0] > 64:
            ctx.synthesis_halfrate(True, [lib.vorbis_window(ctx.bs[0] // 2), lib.vorbis_window(ctx.bs[1] // 2)])
            _decode_as_stock(ctx, sub, list(range(nf)), h.channels, what + " half rate", half=True)
        ctx.close()


def _group_cases():
    p = _stock(*CASES[0])
    hdr = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:3, :2]]
    setup_bit = bytearray(hdr[2])
    setup_bit[len(setup_bit) // 2] ^= 0x04                 # one bit of the setup header
    rate = bytearray(hdr[0])
    rate[12:16] = struct.pack("<I", 48000)
    chans = bytearray(hdr[0])
    chans[11] = 1
    rng = np.random.default_rng(7)

    def f(**kw):
        return b"".join(ogg.file_of(with_packets(p, **kw), rng, max_segs=255))
    bad_comment = comment_packet([b"A=1"])[:-1] + b"\x00"  # end-of-packet bit clear
    pages = ogg.file_of(p, rng, max_segs=255)
    return [("plain", f()), ("tags", f(comment=comment_packet([b"X=1"]))), ("setup bit", f(setup=bytes(setup_bit))),
            ("rate", f(ident=bytes(rate))), ("channels", f(ident=bytes(chans))), ("bad comment", f(comment=bad_comment)),
            ("setup bit again", f(setup=bytes(setup_bit), comment=comment_packet([]))),
            ("no vorbis", b"".join([ogg.page(2, 0, 9, 0, [30], b"\x01notvrb" + bytes(23))])),
            ("headers cut", b"".join(pages[:1])), ("plain again", f())]


def test_group_against_reference(cuda_ok):
    _need()
    cases = _group_cases()
    files = [b for _, b in cases]
    res = lib.ogg_demux(files)
    g = lib.ogg_group(res)
    _check_group(res, g, files, "cases")
    st = dict(zip([w for w, _ in cases], g["status"].tolist()))
    assert st["bad comment"] == EBADHEADER and st["no vorbis"] == ENOTVORBIS and st["headers cut"] == EBADHEADER
    grp = {int(f): int(rep) for first, n, rep in g["groups"].tolist() for f in g["order"][first:first + n]}
    assert grp[1] == 0 and grp[9] == 0 and grp[6] == 2 and grp[3] == 3 and grp[4] == 4
    assert len(g["groups"]) == 4


def _dev_call(files, mp, profiled=False):
    """vb200_ogg_group_dev on the demux of files: (host form's result, device outputs, kernel names or None)"""
    import torch
    dev = torch.device("cuda", 0)
    nfiles = len(files)
    res = lib.ogg_demux(files, max_packets=mp)
    host = lib.ogg_group(res)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)  # noqa: E731
    d_data, d_st, d_npkt, d_info = t(res["data"]), t(res["streams"]), t(res["npkt"]), t(res["info"])
    d_status, d_order, d_npkt_out = (torch.zeros(nfiles, dtype=torch.int32, device=dev) for _ in range(3))
    d_info_out = torch.zeros_like(d_info)
    d_groups = torch.zeros(nfiles * abi.FILE_GROUP_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d_ng = torch.zeros(1, dtype=torch.int32, device=dev)
    sb = lib.ogg_group_scratch_bytes(nfiles, mp)
    d_scr = torch.zeros(sb, dtype=torch.uint8, device=dev)
    args = (nfiles, d_data.data_ptr(), d_st.data_ptr(), mp, d_npkt.data_ptr(), d_info.data_ptr(), d_status.data_ptr(),
            d_order.data_ptr(), d_npkt_out.data_ptr(), d_info_out.data_ptr(), d_groups.data_ptr(), d_ng.data_ptr(),
            d_scr.data_ptr(), sb)
    torch.cuda.synchronize()
    kernels = None

    def call():
        lib.ogg_group_dev(*args)
        torch.cuda.synchronize()
    if profiled:
        kernels = launched_kernels(call)
    else:
        call()
    ng = int(d_ng.item())
    out = {"status": d_status.cpu().numpy(), "order": d_order.cpu().numpy(), "npkt": d_npkt_out.cpu().numpy(),
           "groups": d_groups.cpu().numpy()[:ng * abi.FILE_GROUP_DTYPE.itemsize].view(abi.FILE_GROUP_DTYPE),
           "info": d_info_out.cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(nfiles, mp)}
    return res, host, out, kernels


def _files_of(nfiles):
    base = [b for _, b in _group_cases()]
    return [base[i % len(base)] for i in range(nfiles)]


def test_dev_form(cuda_ok):
    _need()
    for nfiles in (1, 1000):
        files = _files_of(nfiles)
        res, host, dev, _ = _dev_call(files, 200)
        _check_group(res, host, files, "%d files" % nfiles)
        for k in ("status", "order", "npkt", "groups"):
            assert dev[k].tobytes() == host[k].tobytes(), "%d files: %s" % (nfiles, k)
        for p in range(nfiles):
            n = dev["npkt"][p]
            assert dev["info"][p, :n].tobytes() == host["info"][p, :n].tobytes(), "%d files: rows %d" % (nfiles, p)
    L = lib.load()
    assert L.vb200_ogg_group_dev(1, None, None, 1, None, None, None, None, None, None, None, None, None, 0,
                                 None) == -131


def test_launches(cuda_ok):
    """five kernels at 1 and at 1000 files, counted with torch.profiler in a process of its own (a profiler session
    of another test in the same process can lose the kernel records of a later one)"""
    _need()
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_ogg_headers as T; "
            "print(json.dumps([T._dev_call(T._files_of(n), 200, profiled=True)[3] for n in (1, 1000)]))"
            % (here, os.path.dirname(here)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=here)
    assert r.returncode == 0, r.stderr[-3000:]
    for kernels in json.loads(r.stdout.strip().splitlines()[-1]):
        assert len(kernels) == 5 and all("k_ogg_group" in k for k in kernels), kernels


@pytest.mark.parametrize("name", ["s256_512_3ch", "s128_128_3ch_4sub"])
def test_context_matches_driver(cuda_ok, name):
    _need()
    import vorbis_gen as G
    from test_generated_setups_oracle import ALL, corpus, headers_of
    d, pk, p = corpus(name)
    drv = dp.Driver(p)
    try:
        assert drv.on_device
        ctx = lib.vorbis_headers(*headers_of(p)).context()
        for pkts, what in ((pk, "clean"), (G.damaged(pk, 2000 + ALL.index(name), G.header_bits(d)), "damaged")):
            W = dp.ref_headers(p, pkts)
            a = dp.dev_staging(drv.ctx, pkts, W, drv.bs, drv.channels)
            b = dp.dev_staging(ctx, pkts, W, ctx.bs, ctx.channels)
            for x, y, k in zip(a, b, ("residue", "posts", "present")):
                assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                                      y.view(np.uint32) if y.dtype == np.float32 else y), "%s %s: %s" % (name, what, k)
        ctx.close()
    finally:
        drv.close()


def test_cut_tables_are_grouped(cuda_ok):
    """max_packets below the files' packet counts: VB200_EINVAL files keep their status and join their groups, and the
    group's slice decodes the first max_packets packets of each as the stock decoder does"""
    _need()
    files, nsetups = _mixed_corpus()
    blobs = [b for _, b in files][:12] + [b for _, b in _group_cases()]
    mp = 12
    res = lib.ogg_demux(blobs, max_packets=mp)
    assert (res["streams"]["status"] == EINVAL).sum() >= 12
    g = lib.ogg_group(res)
    _check_group(res, g, blobs, "max_packets %d" % mp)
    assert (g["status"] == EINVAL).sum() >= 12
    grouped = sum(int(n) for _, n, _ in g["groups"].tolist())
    assert grouped == int(((g["status"] == 0) | (g["status"] == EINVAL)).sum())
    first, nf, rep = g["groups"].tolist()[0]
    st = res["streams"][rep]
    h = lib.vorbis_headers(*[_hdr_bytes(res["data"], st, k) for k in range(3)])
    ctx = h.context()
    sub = {"data": res["data"], "npkt": g["npkt"][first:first + nf], "info": g["info"][first:first + nf],
           "streams": res["streams"][g["order"][first:first + nf]]}
    assert (sub["npkt"] == mp).all()
    _decode_as_stock(ctx, sub, list(range(nf)), h.channels, "cut tables")
    ctx.close()


def test_hash_collisions(cuda_ok, tmp_path):
    """the library built with VB200_OGG_GROUP_HASH_MASK = 3: nearly every pair of files shares a hash, so the byte
    comparison and the ordered scan over lower files decide each group; the result equals the reference"""
    _need()
    import ctypes as C
    import os
    import subprocess
    import __graft_entry__ as E
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = str(tmp_path / "libvorbis_b200_hash2.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + E.NVCC_FLAGS + ["-DVB200_OGG_GROUP_HASH_MASK=3ULL", "-I", os.path.join(root, "include"),
                                                   "-I", os.path.join(root, "vorbis_b200", "csrc"),
                                                   os.path.join(root, "vorbis_b200", "csrc", "vb200.cu"), "-o", so])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.vb200_ogg_group.argtypes = [C.c_int, vp, C.c_int64, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    files, _ = _mixed_corpus()
    blobs = [b for _, b in files] + [b for _, b in _group_cases()]
    for mp in (None, 12):
        res = lib.ogg_demux(blobs, max_packets=mp)
        info = np.ascontiguousarray(res["info"])
        n, m = info.shape
        st, npkt, data = res["streams"], np.ascontiguousarray(res["npkt"]), np.ascontiguousarray(res["data"])
        status, order, npkt_out = (np.zeros(n, np.int32) for _ in range(3))
        info_out = np.zeros_like(info)
        groups = np.zeros(n, abi.FILE_GROUP_DTYPE)
        ng = np.zeros(1, np.int32)
        p = lambda a: a.ctypes.data  # noqa: E731
        assert L.vb200_ogg_group(n, p(data), data.size, p(st), m, p(npkt), p(info), p(status), p(order),
                                 p(npkt_out), p(info_out), p(groups), p(ng)) == 0
        g = {"status": status, "order": order, "npkt": npkt_out, "info": info_out, "groups": groups[:int(ng[0])]}
        _check_group(res, g, blobs, "hash mask 3, max_packets %s" % mp)
        assert len(g["groups"]) > 4
