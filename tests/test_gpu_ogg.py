"""Ogg Vorbis files in on the device (vb200_ogg_demux[_dev]) against oracle/ogg.py and the stock decoder:
- stock-encoder streams of four setups (the last one 512/4096) and the tests/vorbis_gen.py INSIDE setups, written as Ogg
  files under three pagings: the packet tables, data and vb200_ogg_stream equal the oracle's byte for byte, the header
  and audio packets are the input's, granulepos sits on page-final packets;
- the demuxed tables go straight into vb200_decode_streams_packets and vb200_decode_ranges (float and int16) and give
  the stock pcmout loop's PCM bit for bit; half rate with vb200_vorbis_window(blocksize/2) against the stock half-rate
  decoder;
- damaged files (a CRC-flipped page, a removed page, garbage between pages, a truncated last page, interleaved pages of
  a foreign serial, a second chained link, a file with no Vorbis stream, max_packets too small) equal the oracle, and
  their PCM equals the stock decoder fed the oracle's packets;
- the four hand-worked files of tests/test_ogg_demux_oracle.py give their literal packet tables on the device;
- the _dev form equals the host form, and one call is one kernel launch at 1 and at 1000 files (counted with
  torch.profiler)."""
import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode
from oracle import decode_packets as dp
from oracle import decode_streams as ds
from oracle import ogg
from test_gpu_decode_streams import _check, drivers  # noqa: F401  (drivers: a fixture)
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
CASES = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2), (2, 44100, -0.1)]
PAGINGS = [dict(max_segs=255), dict(max_segs=4), dict(max_segs=255, headers_alone=False)]


def launched_kernels(call):
    """names of the kernels call() launches (it synchronises), from torch.profiler.  A profiler session can lose the
    record of the first kernel it sees, so a torch kernel (at::native, which the library never launches) runs first
    and is left out of the list.  The first session of a process (CUPTI starting up) can lose every record, so a
    session with only that torch kernel runs before the one that is read."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]):
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        call()
    return [e.name for e in prof.events() if e.device_type.name == "CUDA" and
            not e.name.startswith(("Memcpy", "Memset")) and "at::native" not in e.name]


def _need():
    if not (decode.available() and dp.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


_enc = {}


def _stock(ch, rate, q):
    if (ch, rate, q) not in _enc:
        _enc[(ch, rate, q)] = decode.encode(ch, rate, q, probe_signal(ch, rate, 0.7, seed=31))
    return _enc[(ch, rate, q)]


def _files(p, seed):
    rng = np.random.default_rng(seed)
    return [b"".join(ogg.file_of(p, rng, **kw)) for kw in PAGINGS]


def _equals_oracle(res, files, max_packets, what):
    """every file's vb200_ogg_stream, npkt, info rows and packet bytes against oracle.ogg.demux; the oracle results"""
    out = []
    for f, buf in enumerate(files):
        r = ogg.demux(buf, max_packets)
        st, base = res["streams"][f], int(res["file_off"][f])
        for k in ("status", "serial", "pages", "dropped", "holes", "foreign", "chained"):
            assert int(st[k]) == r[k], "%s file %d: %s %d, oracle %d" % (what, f, k, st[k], r[k])
        hdr = r["hdr"] + [(-1 - base, -1)] * (3 - len(r["hdr"]))
        assert [int(x) - base for x in st["hdr_offset"]] == [o for o, _ in hdr], "%s file %d: header offsets" % (what, f)
        assert [int(x) for x in st["hdr_bytes"]] == [n for _, n in hdr], "%s file %d: header sizes" % (what, f)
        n = int(res["npkt"][f])
        assert n == len(r["packets"]), "%s file %d: npkt" % (what, f)
        info = res["info"][f, :n]
        t = ogg.packet_table(r)
        assert (info["offset"] - base == t[:, 0]).all() and (info["bytes"] == t[:, 1]).all(), "%s file %d" % (what, f)
        assert (info["granulepos"] == t[:, 2]).all() and (info["e_o_s"] == t[:, 3]).all(), "%s file %d" % (what, f)
        assert (info["packetno"] == t[:, 4]).all() and not info["choice"].any(), "%s file %d" % (what, f)
        data = res["data"]
        for (o, m), want in zip(r["hdr"], r["hdr_data"]):
            assert data[base + o:base + o + m].tobytes() == want
        for row, want in zip(info, r["pkt_data"]):
            assert data[row["offset"]:row["offset"] + row["bytes"]].tobytes() == want, "%s file %d" % (what, f)
        out.append(r)
    return out


def _hdr_rows(st):
    return np.array([[st["hdr_offset"][k], st["hdr_bytes"][k], 0, 0, k] for k in range(3)], np.int64)


def _ctx(drivers, data, st):  # noqa: F811
    """the device context of the stream whose headers the demux found (the libvorbis-derived driver's)"""
    hdr = _hdr_rows(st)
    key = bytes(data[int(hdr[0, 0]):int(hdr[0, 0] + hdr[0, 1])]) + bytes(data[int(hdr[2, 0]):int(hdr[2, 0] + hdr[2, 1])])
    if key not in drivers:
        drivers[key] = dp.Driver(decode.Packets(data, np.concatenate([hdr, hdr[:1]])))
        assert drivers[key].on_device
    return drivers[key].ctx


def _audio_rows(info):
    return np.stack([info["offset"], info["bytes"], info["granulepos"], info["e_o_s"], info["packetno"]], 1)


def _decode_as_stock(ctx, res, files, ch, what, half=False):
    """decode_streams_packets and decode_ranges on the demux's own tables against ds.ref_decode of the same packets"""
    ns = len(files)
    data, npkt, info = res["data"], res["npkt"], res["info"]
    want = [ds.ref_decode(data, _hdr_rows(res["streams"][f]), _audio_rows(info[f, :npkt[f]]), ch, halfrate=half)
            for f in range(ns)]
    for s16 in (False, True):
        got = ctx.decode_streams_packets(npkt, info, data, ctx.decode_streams_carry(ns), s16=s16)
        _check(got, want, ch, s16, what)
    out_stride = 3000
    req = []
    for f in range(ns):
        n = want[f][0].shape[1]
        req += [(0, f, 1000), (max(n // 2 - 700, 0), f, out_stride), (max(n - 900, 0), f, 1200)]
    req = np.array(req, abi.PCM_RANGE_DTYPE)
    for s16 in (False, True):
        r = ctx.decode_ranges(npkt, info, data, req, out_stride, s16=s16)
        for i, (start, f, length) in enumerate(req.tolist()):
            whole = want[f][0]
            g = min(length, max(0, whole.shape[1] - start))
            assert r["got"][i] == g, "%s request %d" % (what, i)
            sl = whole[:, start:start + g]
            if s16:
                assert np.array_equal(r["pcm"][i][:g], ds.s16_of(sl)), "%s request %d: int16" % (what, i)
            else:
                assert np.array_equal(r["pcm"][i][:, :g].view(np.uint32), sl.view(np.uint32)), "%s request %d" % (what, i)


@pytest.mark.parametrize("ch,rate,q", CASES)
def test_stock_streams_from_files(cuda_ok, drivers, ch, rate, q):  # noqa: F811
    _need()
    p = _stock(ch, rate, q)
    files = _files(p, seed=ch * 7 + rate)
    res = lib.ogg_demux(files)
    orc = _equals_oracle(res, files, res["info"].shape[1], "stock %s" % ((ch, rate, q),))
    pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
    for f, r in enumerate(orc):
        assert r["status"] == 0 and r["hdr_data"] == pk[:3] and r["pkt_data"] == pk[3:], "file %d: packets" % f
        gp = res["info"][f, :res["npkt"][f]]["granulepos"]
        assert ((gp == -1) | (gp == p.meta[3:, 2])).all() and gp[-1] == p.meta[-1, 2]
    assert (res["info"][1, :res["npkt"][1]]["granulepos"] == -1).any(), "page-final granulepos only"
    ctx = _ctx(drivers, res["data"], res["streams"][0])
    _decode_as_stock(ctx, res, files, ch, "stock %s" % ((ch, rate, q),))
    if ctx.bs[0] > 64:
        ctx.synthesis_halfrate(True, [lib.vorbis_window(ctx.bs[0] // 2), lib.vorbis_window(ctx.bs[1] // 2)])
        try:
            _decode_as_stock(ctx, res, files, ch, "half rate", half=True)
        finally:
            ctx.synthesis_halfrate(False)


def test_generated_setups_from_files(cuda_ok, drivers):  # noqa: F811
    _need()
    import vorbis_gen as G
    from test_generated_setups_oracle import corpus
    for name in G.INSIDE:
        _, _, p = corpus(name)
        files = _files(p, seed=len(name))
        res = lib.ogg_demux(files)
        orc = _equals_oracle(res, files, res["info"].shape[1], name)
        pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
        for r in orc:
            assert r["status"] == 0 and r["hdr_data"] == pk[:3] and r["pkt_data"] == pk[3:], name
        ctx = _ctx(drivers, res["data"], res["streams"][0])
        _decode_as_stock(ctx, res, files, ctx.channels, name)


def _damaged(p):
    """a clean file (4 segments per page) and its damaged variants: [(what, bytes)]"""
    rng = np.random.default_rng(3)
    pages = ogg.file_of(p, rng, serial=1000, max_segs=4)
    k = len(pages) // 2
    flip = bytearray(pages[k])
    flip[40] ^= 0x10
    foreign = ogg.file_of(p, np.random.default_rng(4), serial=2000, max_segs=4)
    mixed = []
    for i, pg in enumerate(pages):
        mixed.append(pg)
        if i % 3 == 1 and i // 3 < len(foreign):
            mixed.append(foreign[i // 3])
    other = [ogg.page(2, 0, 9, 0, [30], b"\x01notvrb" + bytes(23)), ogg.page(4, 0, 9, 1, [10], bytes(10))]
    return [("clean", b"".join(pages)),
            ("crc flipped", b"".join(pages[:k] + [bytes(flip)] + pages[k + 1:])),
            ("page removed", b"".join(pages[:k] + pages[k + 1:])),
            ("garbage", b"".join(pages[:k] + [b"OOggS\x00garbage" + bytes(range(200))] + pages[k:])),
            ("truncated", b"".join(pages)[:-5]),
            ("foreign serial", b"".join(mixed)),
            ("chained", b"".join(pages + foreign)),
            ("no vorbis", b"".join(other)),
            ("headers only", b"".join(pages[:4]))]


def test_damaged_files(cuda_ok, drivers):  # noqa: F811
    _need()
    ch, rate, q = CASES[0]
    p = _stock(ch, rate, q)
    cases = _damaged(p)
    files = [b for _, b in cases]
    res = lib.ogg_demux(files)
    orc = _equals_oracle(res, files, res["info"].shape[1], "damaged")
    st = {w: (r["status"], r["dropped"], r["holes"], r["foreign"], r["chained"]) for (w, _), r in zip(cases, orc)}
    assert st["clean"] == (0, 0, 0, 0, 0)
    assert st["crc flipped"][1] >= 1 and st["crc flipped"][2] == 1
    assert st["page removed"][2] == 1 and st["garbage"][1] >= 2 and st["foreign serial"][3] > 0
    assert st["chained"][4] == 1 and st["no vorbis"][0] == ogg.ENOTVORBIS
    # max_packets too small
    small = lib.ogg_demux(files[:2], max_packets=20)
    _equals_oracle(small, files[:2], 20, "max_packets 20")
    assert (small["streams"]["status"] == ogg.EINVAL).all() and (small["npkt"] == 20).all()
    # the PCM of every file with a stream: the stock decoder fed the oracle's packets (the tables equal them)
    keep = [f for f, r in enumerate(orc) if r["status"] == 0 and r["packets"]]
    assert len(keep) >= 7
    sub = {"data": res["data"], "npkt": res["npkt"][keep], "info": res["info"][keep], "streams": res["streams"][keep]}
    ctx = _ctx(drivers, res["data"], res["streams"][0])
    _decode_as_stock(ctx, sub, [files[f] for f in keep], ch, "damaged")


def test_dev_form_and_launches(cuda_ok):
    _need()
    import torch
    p = _stock(*CASES[0])
    base = [b for _, b in _damaged(p)] + _files(p, seed=9)
    for nfiles in (1, 1000):
        files = [base[i % len(base)] for i in range(nfiles)]
        mp = 200
        host = lib.ogg_demux(files, max_packets=mp)
        dev = torch.device("cuda", 0)
        d_bytes = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
        d_off = torch.from_numpy(host["file_off"]).to(dev)
        d_info = torch.zeros((nfiles, mp * abi.PACKET_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        d_npkt = torch.zeros(nfiles, dtype=torch.int32, device=dev)
        d_data = torch.zeros_like(d_bytes)
        d_st = torch.zeros((nfiles, abi.OGG_STREAM_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()

        def call():
            lib.ogg_demux_dev(nfiles, d_bytes.data_ptr(), d_off.data_ptr(), mp, d_info.data_ptr(), d_npkt.data_ptr(),
                              d_data.data_ptr(), d_st.data_ptr())
            torch.cuda.synchronize()
        kernels = launched_kernels(call)
        assert kernels == ["k_ogg_demux"] or (len(kernels) == 1 and "k_ogg_demux" in kernels[0]), kernels
        npkt = d_npkt.cpu().numpy()
        assert (npkt == host["npkt"]).all()
        assert d_st.cpu().numpy().view(abi.OGG_STREAM_DTYPE).reshape(-1).tobytes() == host["streams"].tobytes()
        info = d_info.cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(nfiles, mp)
        data = d_data.cpu().numpy()
        for f in range(nfiles):
            assert info[f, :npkt[f]].tobytes() == host["info"][f, :npkt[f]].tobytes(), "file %d" % f
        assert np.array_equal(data, host["data"]), "data"           # both start from zeros
    L = lib.load()
    assert L.vb200_ogg_demux_dev(1, None, None, 1, None, None, None, None, None) == -131
    assert L.vb200_ogg_demux_dev(0, None, None, 1, None, None, None, None, None) == 0


def test_hand_worked_files(cuda_ok):
    """the device against packet tables worked out by hand, independently of oracle/ogg.py"""
    from test_ogg_demux_oracle import H, HAND, hand_rows
    names = sorted(HAND)
    files = [b"".join(HAND[n][0]) for n in names]
    res = lib.ogg_demux(files, max_packets=8)
    for f, name in enumerate(names):
        status, npages, holes = HAND[name][1]
        st, base = res["streams"][f], int(res["file_off"][f])
        assert (st["status"], st["pages"], st["holes"], st["dropped"], st["foreign"]) == (status, npages, holes, 0, 0)
        assert list(st["hdr_offset"] - base) == [0, 30, 40] and list(st["hdr_bytes"]) == [30, 10, 10], name
        for k in range(3):
            o = int(st["hdr_offset"][k])
            assert res["data"][o:o + 10 if k else o + 30].tobytes() == H[k], name
        info = res["info"][f, :res["npkt"][f]]
        got = np.stack([info["offset"] - base, info["bytes"], info["granulepos"], info["e_o_s"], info["packetno"]], 1)
        assert np.array_equal(got, hand_rows(name)), "%s: %s" % (name, got.tolist())
