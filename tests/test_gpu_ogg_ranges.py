"""Sample ranges straight from Ogg files on the device (vb200_ogg_ranges[_dev]):
- stock streams of four setups (44.1 kHz stereo, mono 22 kHz, 6 channels, 512/4096) muxed under three seeded pagings,
  cut in mid-stream (first granulepos far above zero), interleaved with another serial's pages, written by
  vb200_ogg_mux, and the links of a chained file: got and rows equal vb200_decode_ranges on the vb200_ogg_demux tables
  of the same rows bit for bit, float and int16, full and half rate, for seeded requests (starts at 0, at page
  granulepos +- blocksizes[1]/2, near and past the end; lengths 0..out_stride);
- files under seeded random damage (tests/test_gpu_ogg_edges.py's mutations) equal oracle/ogg_ranges.py: got, and
  the samples of its kept blocks decoded by vb200_decode_streams_packets; nothing lands outside a request's row;
- a small pkt_cap gives VB200_EINVAL and a zero row;
- the _dev form on link_off rows equals the host form, launches three kernels after the memset at 1 and 600 requests,
  and refuses null pointers."""
import numpy as np
import pytest

from oracle import ogg
from oracle import ogg_ranges as orr
from test_gpu_decode_streams import drivers  # noqa: F401  (drivers: a fixture)
from test_gpu_ogg import CASES, _ctx, _damaged, _files, _need, _stock
from test_gpu_ogg_edges import _mutate
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
PKT_CAP = 1 << 20
EINVAL = -131


def _rows(p, seed):
    """the rows of one stock stream: three pagings, a mid-stream cut, interleaved serials, the mux's file, and the
    two links of a chained file"""
    rng = np.random.default_rng(seed)
    pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
    gr = [int(g) for g in p.meta[:, 2]]
    rows = _files(p, seed)
    k = (len(pk) - 3) // 3
    rows.append(b"".join(ogg.write(pk[:3] + pk[3 + k:], [0, 0, 0] + gr[3 + k:], 5, rng, max_segs=17)))
    cases = dict(_damaged(p))
    rows.append(cases["foreign serial"])
    m = lib.ogg_mux([pk[3:]], [gr[3:]], headers=[pk[:3]], serials=[77])
    rows.append(m["pages"][0])
    chained = cases["chained"]
    links = lib.ogg_links([chained])["link_off"]
    rows += [chained[links[0]:links[1]], chained[links[1]:links[2]]]
    return rows


def _requests(files, length, bs, out_stride, rng, half):
    """seeded requests per row: starts at 0, at page granulepos +- blocksizes[1]/2, near and past the end"""
    hs = 1 if half else 0
    req = []
    for f, buf in enumerate(files):
        hd = orr.head(buf, bs, 1, half)
        n = int(length[f])
        starts = [0, n - 1, n, n + 5, max(n - out_stride // 2, 0)]
        gps = [g for g in ogg.demux(buf, 1 << 20)["packets"] if g[2] > 0]
        for g in gps[::max(len(gps) // 4, 1)]:
            t = (g[2] - hd["G0"]) >> hs
            starts += [max(t - (bs[1] // 2 >> hs), 0), t, t + (bs[1] // 2 >> hs)]
        starts += [int(x) for x in rng.integers(0, max(n, 1), 3)]
        for s in starts:
            req.append((max(s, 0), f, int(rng.choice([0, 1, int(rng.integers(1, out_stride + 1)), out_stride]))))
    return np.array(req, abi.PCM_RANGE_DTYPE)


def _equal_to_packet_table(ctx, files, what, half=False, out_stride=2500):
    res = lib.ogg_demux(files)
    assert (res["streams"]["status"] == 0).all(), what
    length = ctx.decode_streams_index(res["npkt"], res["info"], res["data"])["length"]
    req = _requests(files, length, ctx.bs, out_stride, np.random.default_rng(len(files)), half)
    for s16 in (False, True):
        want = ctx.decode_ranges(res["npkt"], res["info"], res["data"], req, out_stride, s16=s16)
        got = ctx.ogg_ranges(files, req, out_stride, PKT_CAP, s16=s16)
        assert np.array_equal(got["got"], want["got"]), "%s s16=%s: got %s, packet table %s" % (
            what, s16, got["got"], want["got"])
        bad = [i for i in range(len(req)) if got["pcm"][i].tobytes() != want["pcm"][i].tobytes()]
        assert not bad, "%s s16=%s: requests %s differ" % (what, s16, req[bad[:5]])
    return req


@pytest.mark.parametrize("ch,rate,q", CASES)
def test_equals_decode_ranges_on_demux_tables(cuda_ok, drivers, ch, rate, q):  # noqa: F811
    _need()
    p = _stock(ch, rate, q)
    files = _rows(p, seed=ch * 7 + rate)
    res = lib.ogg_demux(files[:1])
    ctx = _ctx(drivers, res["data"], res["streams"][0])
    _equal_to_packet_table(ctx, files, "stock %s" % ((ch, rate, q),))
    if ctx.bs[0] > 64:
        ctx.synthesis_halfrate(True, [lib.vorbis_window(ctx.bs[0] // 2), lib.vorbis_window(ctx.bs[1] // 2)])
        try:
            _equal_to_packet_table(ctx, files, "half rate %s" % ((ch, rate, q),), half=True)
        finally:
            ctx.synthesis_halfrate(False)


def _oracle_rows(ctx, files, req, out_stride, s16):
    """the rows oracle/ogg_ranges.py gives: its kept blocks decoded as one fresh stream each (no granulepos, so every
    block returns all it finishes) by vb200_decode_streams_packets, placed by their windows"""
    ch, bs = ctx.channels, ctx.bs
    plans = [orr.request(files[f], bs, 1, s, n) for s, f, n in req.tolist()]
    streams = [pl["kept"] for pl in plans if pl["kept"]]
    data, rows = bytearray(), []
    for kept in streams:
        r = []
        for j, b in enumerate(kept):
            r.append((len(data), -1, len(b["data"]), 0, j, 0))     # offset, granulepos, bytes, e_o_s, packetno
            data += b["data"]
        rows.append(r)
    mp = max([len(r) for r in rows] + [1])
    info = np.zeros((max(len(rows), 1), mp), abi.PACKET_INFO_DTYPE)
    npkt = np.zeros(max(len(rows), 1), np.int32)
    for s, r in enumerate(rows):
        npkt[s] = len(r)
        for j, x in enumerate(r):
            info[s, j] = x
    dec = ctx.decode_streams_packets(npkt, info, np.frombuffer(bytes(data) + b"\0", np.uint8),
                                     ctx.decode_streams_carry(len(npkt)), s16=s16) if rows else None
    out = np.zeros((len(req), out_stride, ch) if s16 else (len(req), ch, out_stride), np.int16 if s16 else np.float32)
    s = 0
    for i, pl in enumerate(plans):
        if not pl["kept"]:
            continue
        pcm, at = dec["pcm"][s], 0
        s += 1
        for j, b in enumerate(pl["kept"]):
            if j == 0:
                continue
            fin = bs[pl["kept"][j - 1]["W"]] // 4 + bs[b["W"]] // 4
            lo, hi = b["keep"]
            if hi > lo:
                if s16:
                    out[i, b["at"]:b["at"] + hi - lo] = pcm[at + lo:at + hi]
                else:
                    out[i, :, b["at"]:b["at"] + hi - lo] = pcm[:, at + lo:at + hi]
            at += fin
    return [pl["got"] for pl in plans], out


def test_damaged_files_equal_oracle(cuda_ok, drivers):  # noqa: F811
    _need()
    p = _stock(*CASES[0])
    rng = np.random.default_rng(41)
    pages = ogg.file_of(p, rng, serial=1000, max_segs=9)
    foreign = ogg.file_of(p, np.random.default_rng(4), serial=2000, max_segs=4)
    files = [_mutate(pages, foreign, rng)[0] for _ in range(24)]
    res = lib.ogg_demux([b"".join(pages)])
    ctx = _ctx(drivers, res["data"], res["streams"][0])
    out_stride = 1800
    n = int(p.meta[-1, 2])
    req = [(int(rng.integers(0, n + 2000)), f, int(rng.integers(0, out_stride + 1))) for f in range(len(files))
           for _ in range(4)]
    req = np.array(req, abi.PCM_RANGE_DTYPE)
    for s16 in (False, True):
        got = ctx.ogg_ranges(files, req, out_stride, PKT_CAP, s16=s16)
        want_got, want = _oracle_rows(ctx, files, req, out_stride, s16)
        assert list(got["got"]) == want_got
        for i in range(len(req)):
            assert got["pcm"][i].tobytes() == want[i].tobytes(), "request %d %s" % (i, req[i])


def test_small_pkt_cap(cuda_ok, drivers):  # noqa: F811
    _need()
    p = _stock(*CASES[0])
    files = _files(p, seed=3)[:1]
    res = lib.ogg_demux(files)
    ctx = _ctx(drivers, res["data"], res["streams"][0])
    n = int(p.meta[-1, 2])
    req = np.array([(n // 2, 0, 2000), (0, 0, 0)], abi.PCM_RANGE_DTYPE)
    big = ctx.ogg_ranges(files, req, 2000, PKT_CAP)
    small = ctx.ogg_ranges(files, req, 2000, 600)
    assert big["got"][0] == 2000 and small["got"][0] == EINVAL and small["got"][1] == 0
    assert not small["pcm"][0].any()


def test_dev_form_link_off_and_launches(cuda_ok, drivers):  # noqa: F811
    _need()
    import torch
    p = _stock(*CASES[0])
    chained = dict(_damaged(p))["chained"]
    links = lib.ogg_links([chained])["link_off"]
    rows = [chained[links[k]:links[k + 1]] for k in range(len(links) - 1)]
    res = lib.ogg_demux(rows[:1])
    ctx = _ctx(drivers, res["data"], res["streams"][0])
    dev = torch.device("cuda", 0)
    d_bytes = torch.from_numpy(np.frombuffer(chained, np.uint8).copy()).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(links, np.int64)).to(dev)
    out_stride = 1500
    rng = np.random.default_rng(5)
    n = int(p.meta[-1, 2])
    for nreq in (1, 600):
        req = np.array([(int(rng.integers(0, n)), k % 2, int(rng.integers(0, out_stride + 1))) for k in range(nreq)],
                       abi.PCM_RANGE_DTYPE)
        host = ctx.ogg_ranges(rows, req, out_stride, PKT_CAP)
        d_req = torch.from_numpy(req.view(np.uint8).copy()).to(dev)
        d_pcm = torch.full((nreq * ctx.channels * out_stride,), 7.0, dtype=torch.float32, device=dev)
        d_got = torch.zeros(nreq, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()

        l0 = ctx.launch_count()
        ctx.ogg_ranges_dev(len(links) - 1, d_bytes.data_ptr(), d_off.data_ptr(), nreq, d_req.data_ptr(), 0,
                           d_pcm.data_ptr(), out_stride, PKT_CAP, d_got.data_ptr())
        torch.cuda.synchronize()
        assert ctx.launch_count() - l0 == 3, "plan, entropy decode + DSP, synthesis"
        assert np.array_equal(d_got.cpu().numpy(), host["got"])
        assert d_pcm.cpu().numpy().tobytes() == host["pcm"].tobytes()
    L = lib.load()
    assert L.vb200_ogg_ranges_dev(ctx.h, 1, None, None, 1, None, 0, None, 10, 100, None, None) == EINVAL
    assert L.vb200_ogg_ranges_dev(ctx.h, 1, d_bytes.data_ptr(), d_off.data_ptr(), 1, d_req.data_ptr(), 0,
                                  d_pcm.data_ptr(), 10, -1, d_got.data_ptr(), None) == EINVAL
    assert L.vb200_ogg_ranges_dev(ctx.h, 1, None, None, 0, None, 0, None, 10, 100, None, None) == 0
