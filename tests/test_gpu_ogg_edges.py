"""The Ogg demux on the device (vb200_ogg_demux[_dev]) at the page shapes stock files never make, under seeded random
damage, and through to the stock decoder's PCM:
- the writer's shapes of tests/test_ogg_demux_oracle.py in one call: all six pagings, 255-segment pages with a packet
  on four of them, and one segment per page; the tables equal the oracle's and give back the written packets;
- the page lengths and bit flips of tests/test_ogg_edges_oracle.py (the kernel's 32-lane CRC split with empty chunks,
  every residue mod 32, the 65 307-byte page), and its hand-worked stream rules (sequence wrap, 64-bit and negative
  granulepos, empty pages, EOS edges, other streams' and version-1 pages, a continued page after a hole, captures cut
  by the end of the file, 'O' runs across the 32-byte resync windows) give their literal tables on the device;
  files of 0, 1 and 26 bytes between them have no stream and nothing is written in their ranges;
- 2000 files made from the stock streams of four setups by 1-4 seeded mutations each (bit flips, byte inserts and
  deletes, dropped, duplicated and swapped pages, truncation, spliced pages of another serial, garbage with 'O' and
  "OggS"): every vb200_ogg_stream field, info row and packet equals the oracle's, with max_packets large and small;
  the files that keep a stream decode (vb200_decode_streams_packets and vb200_decode_ranges, float and int16) as the
  stock decoder fed the same packets;
- one CTA's four warps on a 20 MB file and three tiny ones (6 files); files at odd byte offsets after file_off[0] > 0,
  host and _dev forms; a _dev call with its files past 2^31 bytes of padding lands everything at the shifted
  offsets (skipped with less than 8 GB of free device memory)."""
import collections

import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode
from oracle import ogg
from test_gpu_decode_streams import _check, drivers  # noqa: F401  (drivers: a fixture)
from test_gpu_ogg import CASES, PAGINGS as STOCK_PAGINGS, _ctx, _decode_as_stock, _equals_oracle, _need
from test_ogg_demux_oracle import PAGINGS, H, _check_roundtrip, _packets
from test_ogg_edges_oracle import EDGE, NOT_VORBIS, SHORT, check_demux, crc_cases
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu
FIELDS = ("status", "serial", "pages", "dropped", "holes", "foreign", "chained")


def _as_oracle(res, f):
    """file f of a device result in oracle.ogg.demux's form (offsets from the file's first byte)"""
    st, base, data = res["streams"][f], int(res["file_off"][f]), res["data"]
    r = {k: int(st[k]) for k in FIELDS}
    r["hdr"] = [(int(o) - base, int(n)) for o, n in zip(st["hdr_offset"], st["hdr_bytes"]) if n >= 0]
    r["packets"] = [(int(i["offset"]) - base, int(i["bytes"]), int(i["granulepos"]), int(i["e_o_s"]),
                     int(i["packetno"])) for i in res["info"][f, :res["npkt"][f]]]
    r["hdr_data"] = [data[base + o:base + o + n].tobytes() for o, n in r["hdr"]]
    r["pkt_data"] = [data[base + o:base + o + n].tobytes() for o, n, _, _, _ in r["packets"]]
    return r


def _demux_at(buf, file_off, max_packets):
    """the host form on files bytes[file_off[f] .. file_off[f+1]) of buf, file_off[0] possibly > 0; lib.ogg_demux's
    result dict"""
    L = lib.load()
    buf = np.ascontiguousarray(np.frombuffer(bytes(buf), np.uint8))
    file_off = np.ascontiguousarray(file_off, np.int64)
    n = len(file_off) - 1
    info = np.zeros((n, max_packets), abi.PACKET_INFO_DTYPE)
    npkt = np.zeros(n, np.int32)
    data = np.zeros(len(buf), np.uint8)
    streams = np.zeros(n, abi.OGG_STREAM_DTYPE)
    rc = L.vb200_ogg_demux(n, buf.ctypes.data, file_off.ctypes.data, max_packets, info.ctypes.data, npkt.ctypes.data,
                           data.ctypes.data, streams.ctypes.data)
    assert rc == 0, L.vb200_last_error()
    return {"data": data, "file_off": file_off, "info": info, "npkt": npkt, "streams": streams}


# ---- 1. the writer's shapes ----------------------------------------------------------------------------------------
def _writer_files():
    """(packets, granules, pages) of every file tests/test_ogg_demux_oracle.py writes, and one of one-segment pages"""
    out = []
    for paging in range(len(PAGINGS)):
        rng = np.random.default_rng(100 + paging)
        pk = _packets(rng, 40)
        granules = [0, 0, 0] + [1000 + 7 * k for k in range(len(pk) - 3)]
        out.append((pk, granules, ogg.write(pk, granules, 0x1234 + paging, rng, **PAGINGS[paging])))
    rng = np.random.default_rng(7)
    pk = _packets(rng, 5)
    pk[4] = bytes(rng.integers(0, 256, 255 * 800, dtype=np.uint8))
    pk.append(bytes(255 * 3))
    granules = [0, 0, 0] + [1000 + k for k in range(len(pk) - 3)]
    out.append((pk, granules, ogg.write(pk, granules, 99, rng, min_segs=255, headers_alone=False)))
    rng = np.random.default_rng(8)
    pk = _packets(rng, 30)
    granules = [0, 0, 0] + [1000 + 7 * k for k in range(len(pk) - 3)]
    out.append((pk, granules, ogg.write(pk, granules, 5, rng, min_segs=1, max_segs=1, headers_alone=False)))
    return out


def test_writer_shapes(cuda_ok):
    written = _writer_files()
    assert max(p[26] for _, _, pages in written for p in pages) == 255
    assert all(p[26] == 1 for p in written[-1][2])
    files = [b"".join(pages) for _, _, pages in written]
    res = lib.ogg_demux(files, max_packets=100)
    _equals_oracle(res, files, 100, "writer")
    for f, (pk, granules, pages) in enumerate(written):
        _check_roundtrip(_as_oracle(res, f), pk, granules, pages)


# ---- 2. page lengths and bit flips for the CRC split ---------------------------------------------------------------
def test_crc_page_lengths(cuda_ok):
    cases = crc_cases()
    files = [c[0] for _, c in cases]
    res = lib.ogg_demux(files, max_packets=400)
    _equals_oracle(res, files, 400, "crc")
    for f, (name, (_, expect, rows, payloads)) in enumerate(cases):
        check_demux(_as_oracle(res, f), expect, rows, payloads, name)
    assert (res["streams"]["dropped"] == 0).sum() == sum(1 for n, _ in cases if "flipped" not in n)


# ---- 3. stream rules -----------------------------------------------------------------------------------------------
def test_stream_rules(cuda_ok):
    names = sorted(EDGE)
    files, what = [], []
    for k, name in enumerate(names):
        files.append(b"".join(EDGE[name][0]))
        what.append(name)
        files.append(SHORT[k % len(SHORT)])
        what.append(None)
    res = lib.ogg_demux(files, max_packets=16)
    _equals_oracle(res, files, 16, "rules")
    for f, name in enumerate(what):
        r = _as_oracle(res, f)
        if name is None:
            a, b = res["file_off"][f], res["file_off"][f + 1]
            assert tuple(r[k] for k in FIELDS if k != "serial") == NOT_VORBIS and r["serial"] == 0
            assert list(res["streams"][f]["hdr_offset"]) == [-1] * 3 and res["npkt"][f] == 0
            assert not res["data"][a:b].any(), "file %d of %d bytes: data written in its range" % (f, b - a)
        else:
            _, expect, rows, payloads = EDGE[name]
            check_demux(r, expect, rows, payloads, name)


# ---- 4. seeded random damage ---------------------------------------------------------------------------------------
SEED, PER_SETUP = 20261017, 500
PAGE_OPS = ("drop page", "duplicate page", "swap pages", "foreign page")
BYTE_OPS = ("bit flip", "insert byte", "delete byte", "truncate", "garbage")
_short = {}


def _short_stream(ch, rate, q):
    """the stock encoder's packets for 0.3-0.4 s of the probe signal"""
    if (ch, rate, q) not in _short:
        _short[(ch, rate, q)] = decode.encode(ch, rate, q, probe_signal(ch, rate, 0.3 if ch > 2 else 0.4, seed=41))
    return _short[(ch, rate, q)]


def _garbage(rng):
    g = bytearray(rng.integers(0, 256, int(rng.integers(1, 120)), dtype=np.uint8))
    for i in rng.integers(0, len(g), int(rng.integers(0, 6))):
        g[int(i)] = ord("O")
    i = int(rng.integers(0, len(g) + 1))
    g[i:i] = b"OggS" + bytes(rng.integers(0, 256, int(rng.integers(0, 30)), dtype=np.uint8))
    return bytes(g)


def _header_pages(pages):
    """how many pages the three header packets take"""
    ended = 0
    for k, p in enumerate(pages):
        ended += sum(v < 255 for v in p[27:27 + p[26]])
        if ended >= 3:
            return k + 1


def _mutate(pages, foreign, rng):
    """1-4 seeded mutations of a file given as its pages: (bytes, the mutations).  Three in four land after the
    header pages, so that most files keep a stream to decode."""
    ops = [str(o) for o in rng.choice(PAGE_OPS + BYTE_OPS, size=int(rng.integers(1, 5)))]
    nh = _header_pages(pages)
    lo = sum(len(p) for p in pages[:nh])
    pages = list(pages)
    for op in [o for o in ops if o in PAGE_OPS]:
        i = int(rng.integers(min(nh, len(pages) - 1) if rng.random() < 0.75 else 0, len(pages)))
        if op == "drop page" and len(pages) > 1:
            del pages[i]
        elif op == "duplicate page":
            pages.insert(i, pages[i])
        elif op == "swap pages" and i + 1 < len(pages):
            pages[i], pages[i + 1] = pages[i + 1], pages[i]
        elif op == "foreign page":
            pages.insert(i, foreign[int(rng.integers(0, len(foreign)))])
    b = bytearray(b"".join(pages))
    for op in [o for o in ops if o in BYTE_OPS]:
        i = int(rng.integers(min(lo, len(b) - 1) if rng.random() < 0.75 else 0, len(b)))
        if op == "bit flip":
            b[i] ^= 1 << int(rng.integers(0, 8))
        elif op == "insert byte":
            b.insert(i, int(rng.integers(0, 256)))
        elif op == "delete byte":
            del b[i]
        elif op == "truncate":
            del b[i:]
        else:
            b[i:i] = _garbage(rng)
    return bytes(b), ops


def _corpus():
    """[(setup index, file bytes)]: PER_SETUP damaged files per setup of CASES"""
    rng = np.random.default_rng(SEED)
    pagings = STOCK_PAGINGS + [dict(max_segs=17), dict(max_segs=1, headers_alone=False)]
    out = []
    for s, case in enumerate(CASES):
        p = _short_stream(*case)
        bases = [ogg.file_of(p, rng, **kw) for kw in pagings]
        foreign = ogg.file_of(p, rng, max_segs=8)
        for k in range(PER_SETUP):
            out.append((s, _mutate(bases[k % len(bases)], foreign, rng)[0]))
    return out


def test_random_damage(cuda_ok, drivers):  # noqa: F811
    _need()
    corpus = _corpus()
    files = [b for _, b in corpus]
    assert len(files) >= 2000
    mp = 400
    res = lib.ogg_demux(files, max_packets=mp)
    orc = _equals_oracle(res, files, mp, "random damage")
    hist = collections.Counter(r["status"] for r in orc)
    print("random damage: seed %d, %d files, %d bytes; status %s; dropped > 0: %d, holes > 0: %d, foreign > 0: %d, "
          "chained: %d" % (SEED, len(files), sum(map(len, files)), dict(sorted(hist.items())),
                           sum(r["dropped"] > 0 for r in orc), sum(r["holes"] > 0 for r in orc),
                           sum(r["foreign"] > 0 for r in orc), sum(r["chained"] for r in orc)))
    assert hist[ogg.EINVAL] == 0, "max_packets %d cut a file" % mp
    assert hist[0] >= 1000 and hist[ogg.EBADHEADER] >= 200 and hist[ogg.ENOTVORBIS] >= 100, hist
    assert sum(r["dropped"] > 0 for r in orc) >= 800 and sum(r["holes"] > 0 for r in orc) >= 500
    assert sum(r["foreign"] > 0 for r in orc) >= 200
    # max_packets small enough to cut most files
    small = lib.ogg_demux(files, max_packets=6)
    cut = _equals_oracle(small, files, 6, "random damage, max_packets 6")
    assert sum(r["status"] == ogg.EINVAL for r in cut) >= 600
    # the files that keep a stream, per setup: the stock decoder fed the same packets
    for s, (ch, rate, q) in enumerate(CASES):
        keep = [f for f, (cs, _) in enumerate(corpus) if cs == s and orc[f]["status"] == 0 and orc[f]["packets"]]
        assert len(keep) >= 200, (s, len(keep))
        keep = keep[:150]
        pk = _short_stream(ch, rate, q)
        want_hdr = [bytes(pk.buf[int(o):int(o + n)]) for o, n in pk.meta[:3, :2]]
        assert all(orc[f]["hdr_data"] == want_hdr for f in keep)
        sub = {"data": res["data"], "npkt": res["npkt"][keep], "info": res["info"][keep],
               "streams": res["streams"][keep]}
        ctx = _ctx(drivers, res["data"], res["streams"][keep[0]])
        _decode_as_stock(ctx, sub, [files[f] for f in keep], ch, "random damage %s" % ((ch, rate, q),))


# ---- 5. layout and scale -------------------------------------------------------------------------------------------
def test_unequal_files_in_one_cta(cuda_ok):
    rng = np.random.default_rng(12)
    sizes = rng.integers(1, 8000, 5200)
    blob = rng.integers(0, 256, int(sizes.sum()), dtype=np.uint8).tobytes()
    at = np.concatenate([[0], np.cumsum(sizes)])
    pk = H + [blob[at[k]:at[k + 1]] for k in range(len(sizes))]
    granules = [0, 0, 0] + [1000 + 64 * k for k in range(len(sizes))]
    pages = ogg.write(pk, granules, 31, rng, min_segs=255)
    big = b"".join(pages)
    assert len(big) > 20e6 and sum(p[26] == 255 for p in pages) > 250
    tiny = [b"".join(EDGE[n][0]) for n in sorted(EDGE)[:5]]
    files = [tiny[0], big] + tiny[1:]                 # CTA 0: tiny, 20 MB, tiny, tiny; CTA 1: two tiny
    res = lib.ogg_demux(files, max_packets=len(sizes) + 1)
    r = _as_oracle(res, 1)
    _check_roundtrip(r, pk, granules, pages)
    for f in (0, 2, 3, 4, 5):
        _, expect, rows, payloads = EDGE[sorted(EDGE)[f - (f > 1)]]
        check_demux(_as_oracle(res, f), expect, rows, payloads, "file %d" % f)


def _odd_layout():
    """EDGE files and two writer files at odd and even starts after 3 bytes that belong to no file"""
    files = [b"".join(EDGE[n][0]) for n in sorted(EDGE)] + [b"".join(w[2]) for w in _writer_files()[4:6]]
    files = [f + b"\x4f" * (k % 2) for k, f in enumerate(files)]   # an 'O' after every other file: odd lengths
    buf = b"OOO" + b"".join(files)
    file_off = 3 + np.concatenate([[0], np.cumsum([len(f) for f in files])])
    assert (file_off[:-1] % 2 == 1).sum() >= 4 and (file_off[:-1] % 2 == 0).sum() >= 4
    return files, buf, file_off


def test_odd_starts_host_and_dev(cuda_ok):
    import torch
    files, buf, file_off = _odd_layout()
    mp = 100
    host = _demux_at(buf, file_off, mp)
    _equals_oracle(host, files, mp, "odd starts")
    assert not host["data"][:3].any()
    n = len(files)
    dev = torch.device("cuda", 0)
    d_bytes = torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).to(dev)
    d_off = torch.from_numpy(file_off.astype(np.int64)).to(dev)
    d_info = torch.zeros((n, mp * abi.PACKET_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    d_npkt = torch.zeros(n, dtype=torch.int32, device=dev)
    d_data = torch.zeros_like(d_bytes)
    d_st = torch.zeros((n, abi.OGG_STREAM_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    lib.ogg_demux_dev(n, d_bytes.data_ptr(), d_off.data_ptr(), mp, d_info.data_ptr(), d_npkt.data_ptr(),
                      d_data.data_ptr(), d_st.data_ptr())
    torch.cuda.synchronize()
    npkt = d_npkt.cpu().numpy()
    assert (npkt == host["npkt"]).all()
    assert d_st.cpu().numpy().view(abi.OGG_STREAM_DTYPE).reshape(-1).tobytes() == host["streams"].tobytes()
    info = d_info.cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(n, mp)
    for f in range(n):
        assert info[f, :npkt[f]].tobytes() == host["info"][f, :npkt[f]].tobytes(), "file %d" % f
    assert np.array_equal(d_data.cpu().numpy(), host["data"])


def test_offsets_past_2_31(cuda_ok):
    """one _dev call whose files sit after 2^31 + 1 bytes of padding: every offset shifts by the padding, and the
    padding of data stays untouched"""
    import torch
    free = torch.cuda.mem_get_info()[0]
    if free < 8 << 30:
        pytest.skip("%.1f GB of device memory free, 8 GB needed" % (free / 2 ** 30))
    files, _, _ = _odd_layout()
    if decode.available():
        files.append(b"".join(ogg.file_of(_short_stream(*CASES[0]), np.random.default_rng(5))))
    mp = 200
    host = lib.ogg_demux(files, max_packets=mp)
    pad = (1 << 31) + 1
    total = int(host["file_off"][-1])
    n = len(files)
    dev = torch.device("cuda", 0)
    d_bytes = torch.full((pad + total,), ord("O"), dtype=torch.uint8, device=dev)
    d_bytes[pad:] = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
    d_data = torch.zeros(pad + total, dtype=torch.uint8, device=dev)
    d_off = torch.from_numpy(host["file_off"] + pad).to(dev)
    d_info = torch.zeros((n, mp * abi.PACKET_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    d_npkt = torch.zeros(n, dtype=torch.int32, device=dev)
    d_st = torch.zeros((n, abi.OGG_STREAM_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    try:
        lib.ogg_demux_dev(n, d_bytes.data_ptr(), d_off.data_ptr(), mp, d_info.data_ptr(), d_npkt.data_ptr(),
                          d_data.data_ptr(), d_st.data_ptr())
        torch.cuda.synchronize()
        assert not d_data[:pad].any().item(), "data written in the padding"
        assert np.array_equal(d_data[pad:].cpu().numpy(), host["data"])
        npkt = d_npkt.cpu().numpy()
        assert (npkt == host["npkt"]).all()
        st = d_st.cpu().numpy().view(abi.OGG_STREAM_DTYPE).reshape(-1)
        for k in FIELDS:
            assert (st[k] == host["streams"][k]).all(), k
        found = host["streams"]["hdr_bytes"] >= 0
        assert (st["hdr_bytes"] == host["streams"]["hdr_bytes"]).all()
        assert (st["hdr_offset"][found] == host["streams"]["hdr_offset"][found] + pad).all()
        assert (st["hdr_offset"][~found] == -1).all()
        info = d_info.cpu().numpy().view(abi.PACKET_INFO_DTYPE).reshape(n, mp)
        for f in range(n):
            got, want = info[f, :npkt[f]], host["info"][f, :npkt[f]]
            assert (got["offset"] == want["offset"] + pad).all() and (got["offset"] >= pad).all(), "file %d" % f
            for k in ("bytes", "granulepos", "e_o_s", "packetno", "choice"):
                assert (got[k] == want[k]).all(), "file %d: %s" % (f, k)
    finally:
        del d_bytes, d_data
        torch.cuda.empty_cache()
