"""Chained Ogg files on the device (vb200_ogg_links[_dev]) against oracle/ogg_links.py and the stock decoder:
- the hand-worked files of tests/test_ogg_links_oracle.py give their literal link_first / link_off;
- seeded chains of 1-12 links (stock setups and tests/vorbis_gen.py setups, per-link comment headers, some links
  multiplexed with a foreign stream's pages, some truncated, some with the serial of the link before) equal
  oracle.ogg_links.links, as built and again under the seeded random damage of tests/test_gpu_ogg_edges.py;
- links -> vb200_ogg_demux on link_off -> vb200_ogg_group -> vb200_vorbis_headers_parse -> vb200_decode_streams_packets
  and vb200_decode_ranges (float and int16): each link's PCM is the stock decoder's on that link's packets, and a
  chain of one setup is one group;
- where a file's first link ends with an EOS page, row 0 of the chained path is vb200_ogg_demux of the whole file in
  every field but `chained`;
- streams encoded on the device and muxed by one vb200_ogg_mux call, taken as files of consecutive streams, give back
  the mux's out_off;
- the _dev form equals the host form; link_cap = 0 sizes a call, too small a link_cap writes no link_off (the host form
  returns VB200_EINVAL); unequal files share one CTA; offsets past 2^31; one call is three kernel launches at 1 and at
  1000 files (counted with torch.profiler in a process of its own)."""
import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode
from oracle import ogg
from oracle import ogg_links
from test_gpu_ogg import _decode_as_stock, _need, launched_kernels
from test_gpu_ogg_edges import FIELDS, _demux_at, _header_pages, _mutate
from test_ogg_links_oracle import CASES, literal_table, table
from vorbis_b200 import lib

pytestmark = pytest.mark.gpu
EINVAL = -131
STOCK = [(2, 44100, 0.5), (1, 22050, 0.3)]
GEN = ["s64_64_mono", "s256_512_3ch"]


def _check_table(res, files, what):
    first, off = table(files)
    assert np.array_equal(res["link_first"], first), "%s: link_first %s" % (what, res["link_first"].tolist())
    assert np.array_equal(res["link_off"], off), "%s: link_off" % what


def test_hand_worked_files(cuda_ok):
    names = list(CASES)
    res = lib.ogg_links([CASES[n][0] for n in names])
    first, off = literal_table(names)
    assert np.array_equal(res["link_first"], first) and np.array_equal(res["link_off"], off)


# ---- seeded chains -------------------------------------------------------------------------------------------------
_src = {}


def _sources():
    """[(headers, audio packets, granules)]: the stock encoder's streams of STOCK and the generated setups of GEN"""
    if not _src:
        import vorbis_gen  # noqa: F401
        from test_generated_setups_oracle import corpus
        ps = [decode.encode(ch, rate, q, probe_signal(ch, rate, 0.4, seed=51)) for ch, rate, q in STOCK]
        ps += [corpus(name)[2] for name in GEN]
        for k, p in enumerate(ps):
            pk = [bytes(p.buf[int(o):int(o + n)]) for o, n in p.meta[:, :2]]
            _src[k] = (pk[:3], pk[3:], [int(g) for g in p.meta[3:, 2]])
    return [_src[k] for k in sorted(_src)]


def _comment(text):
    from test_gpu_ogg_headers import comment_packet
    return comment_packet([b"TITLE=" + text])


def _chain(rng, sources, nlinks, setups=None):
    """one chained file: (pages, link start offsets as built, the end).  Every link has its own comment header;
    about one in five is multiplexed with a foreign stream (its BOS page first, data pages after the headers), one in
    six loses its last audio pages (no EOS page), one in five takes the serial of the link before."""
    pages, starts, at, serial = [], [], 0, None
    for k in range(nlinks):
        s = int(setups[k % len(setups)]) if setups is not None else int(rng.integers(0, len(sources)))
        hdr, audio, gr = sources[s]
        n = int(rng.integers(1, len(audio) + 1))
        pk = [hdr[0], _comment(b"link %d of setup %d" % (k, s)), hdr[2]] + audio[:n]
        serial = serial if serial is not None and rng.random() < 0.2 else int(rng.integers(0, 1 << 32))
        lp = ogg.write(pk, [0, 0, 0] + gr[:n], serial, rng, max_segs=int(rng.choice([4, 17, 255])))
        nh = _header_pages(lp)
        if rng.random() < 1 / 6 and len(lp) > nh + 1:
            lp = lp[:int(rng.integers(nh + 1, len(lp)))]
        if rng.random() < 0.2:
            fs = serial ^ 0x5A5A
            lp = [ogg.page(2, 0, fs, 0, [30], b"\x80theora" + bytes(23))] + lp[:nh] + \
                 [ogg.page(0, 10 * j, fs, 1 + j, [9], bytes(9)) for j in range(2)] + lp[nh:]
        starts.append(at)
        pages += lp
        at += sum(len(p) for p in lp)
    return pages, starts, at


def _random_chains(seed, nfiles):
    rng = np.random.default_rng(seed)
    src = _sources()
    return [_chain(rng, src, int(rng.integers(1, 13))) for _ in range(nfiles)]


def test_random_chains(cuda_ok):
    _need()
    chains = _random_chains(20261018, 60)
    files = [b"".join(p) for p, _, _ in chains]
    for f, (_, starts, end) in enumerate(chains):
        assert ogg_links.links(files[f]) == starts + [end], "chain %d as built" % f
    res = lib.ogg_links(files)
    _check_table(res, files, "random chains")
    print("random chains: %d files, %d links, %d bytes" % (len(files), res["link_first"][-1], res["file_off"][-1]))
    # seeded damage, 1-4 mutations per file
    rng = np.random.default_rng(20261019)
    foreign = ogg.write([b"\x01vorbis" + bytes(23), b"x" * 40, b"y" * 70] + [b"z" * 90] * 6, [0] * 9, 77, rng,
                        max_segs=2)
    damaged = [_mutate(p, foreign, rng)[0] for p, _, _ in chains for _ in range(4)]
    dres = lib.ogg_links(damaged)
    _check_table(dres, damaged, "damaged chains")
    merged = sum(len(ogg_links.links(d)) != len(s) + 1 for d, (_, s, _) in zip(damaged, [c for c in chains for _ in range(4)]))
    print("damaged chains: %d files, %d links, %d with a link count other than as built" %
          (len(damaged), dres["link_first"][-1], merged))


# ---- end to end ----------------------------------------------------------------------------------------------------
def _chained_demux(files):
    """links, then the host demux on link_off: (links result, demux result)"""
    lk = lib.ogg_links(files)
    buf = b"".join(files)
    mp = max(1, len(buf) * 255 // 282 + 1) if len(buf) < 4000 else 2000
    return lk, _demux_at(buf, lk["link_off"], mp)


def test_end_to_end(cuda_ok):
    _need()
    rng = np.random.default_rng(77)
    src = _sources()
    mixed = _chain(rng, src, 7, setups=[0, 1, 2])
    single = _chain(rng, src, 5, setups=[0])
    files = [b"".join(mixed[0]), b"".join(single[0])]
    lk, res = _chained_demux(files)
    first = lk["link_first"]
    assert list(np.diff(first)) == [7, 5]
    st = res["streams"]
    assert (st["status"] == 0).all() and not st["chained"].any()
    g = lib.ogg_group(res)
    groups = g["groups"].tolist()
    assert len(groups) == 3
    for gi, (g0, nf, rep) in enumerate(groups):
        members = [int(x) for x in g["order"][g0:g0 + nf]]
        if rep == 0:                                      # setup 0: links of both files, the single chain whole
            assert set(range(int(first[1]), int(first[2]))) <= set(members)
        hb = [bytes(res["data"][int(st[rep]["hdr_offset"][k]):int(st[rep]["hdr_offset"][k] + st[rep]["hdr_bytes"][k])])
              for k in range(3)]
        h = lib.vorbis_headers(*hb)
        ctx = h.context()
        try:
            sub = {"data": res["data"], "npkt": g["npkt"][g0:g0 + nf], "info": g["info"][g0:g0 + nf],
                   "streams": st[members]}
            _decode_as_stock(ctx, sub, members, h.channels, "group %d" % gi)
        finally:
            ctx.close()
    # a file's PCM is its links' PCM in row order: the group keeps the single chain's rows in that order
    pos = {int(o): k for k, o in enumerate(g["order"])}
    rows = list(range(int(first[1]), int(first[2])))
    assert [pos[r] for r in rows] == list(range(pos[rows[0]], pos[rows[0]] + len(rows)))


def _ends_with_eos(link, serial):
    """the captured pages of the link alone reach its end, and the last is the EOS page of `serial`"""
    pg = ogg_links.pages_of(link)
    if not pg or pg[-1][1] != len(link):
        return False
    p = pg[-1][0]
    return bool(link[p + 5] & 4) and link[p + 4] == 0 and int.from_bytes(link[p + 14:p + 18], "little") == serial


def test_first_link_equals_whole_file_demux(cuda_ok):
    _need()
    chains = _random_chains(20261020, 40)
    rng = np.random.default_rng(5)
    files = [b"".join(p) for p, _, _ in chains]
    files += [_mutate(p, p[:1], rng)[0] for p, _, _ in chains]
    lk, res = _chained_demux(files)
    whole = _demux_at(b"".join(files), lk["file_off"], res["info"].shape[1])
    checked = 0
    for f, buf in enumerate(files):
        r0 = int(lk["link_first"][f])
        a, b = int(lk["link_off"][r0]), int(lk["link_off"][r0 + 1])
        st = res["streams"][r0]
        if st["status"] != 0 or not _ends_with_eos(buf[:b - a], int(st["serial"])):
            continue
        checked += 1
        w = whole["streams"][f]
        for k in FIELDS:
            if k != "chained":
                assert st[k] == w[k], "file %d: %s" % (f, k)
        assert list(st["hdr_offset"]) == list(w["hdr_offset"]) and list(st["hdr_bytes"]) == list(w["hdr_bytes"])
        n = int(res["npkt"][r0])
        assert n == whole["npkt"][f] and res["info"][r0, :n].tobytes() == whole["info"][f, :n].tobytes(), f
    assert checked >= 30, checked


# ---- the mux's files -----------------------------------------------------------------------------------------------
def test_device_encode_and_mux_round_trip(cuda_ok):
    from oracle import bitrate as B
    from test_gpu_encode_packets import _driver
    from test_gpu_stream_packets import _need_ref, _streams, _timelines
    _need_ref()
    ch, rate, q = 2, 44100, 0.5
    hdr = decode.encode(ch, rate, q, probe_signal(ch, rate, 0.2, seed=31))
    hdr = [bytes(hdr.buf[int(o):int(o + n)]) for o, n in hdr.meta[:3, :2]]
    d = _driver(ch, rate, q)
    try:
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p) for p in _streams(ch, rate, 0.5)] * 3
        tl, pcm_len, eof = _timelines(caps, ch)
        got = d.ctx.encode_streams_packets(tl, pcm_len, eof)
    finally:
        d.close()
    ns = len(caps)
    pk = [got["packets"][s] for s in range(ns)]
    info = [got["info"][s, :int(got["nblocks"][s])] for s in range(ns)]
    serials = [9 if s % 3 else 10 + s for s in range(ns)]                # neighbours that share a serial
    m = lib.ogg_mux(pk, [list(i["granulepos"]) for i in info], [list(i["e_o_s"].astype(bool)) for i in info],
                    headers=[hdr] * ns, serials=serials)
    out_off = m["out_off"]
    out = b"".join(m["pages"])
    cuts = [0, 1, 4, 5, 9, ns]                                           # files of 1, 3, 1, 4 and 3 streams
    files = [out[out_off[a]:out_off[b]] for a, b in zip(cuts, cuts[1:])]
    res = lib.ogg_links(files)
    assert np.array_equal(res["link_off"], out_off)
    assert list(res["link_first"]) == cuts


# ---- call form -----------------------------------------------------------------------------------------------------
def _dev_call(files, link_cap, pad=0, profiled=False):
    """vb200_ogg_links_dev on files after `pad` bytes of 'O': (link_first, link_off (filled with -7 first), kernels)"""
    import torch
    dev = torch.device("cuda", 0)
    buf = np.frombuffer(b"".join(files), np.uint8)
    off = pad + np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)
    d_bytes = torch.full((pad + buf.size + 1,), ord("O"), dtype=torch.uint8, device=dev)
    d_bytes[pad:pad + buf.size] = torch.from_numpy(buf.copy()).to(dev)
    d_off = torch.from_numpy(off).to(dev)
    d_first = torch.full((len(files) + 1,), -7, dtype=torch.int64, device=dev)
    d_links = torch.full((link_cap + 1,), -7, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()

    def call():
        lib.ogg_links_dev(len(files), d_bytes.data_ptr(), d_off.data_ptr(), d_first.data_ptr(), d_links.data_ptr(),
                          link_cap)
        torch.cuda.synchronize()
    kernels = None
    try:
        if profiled:
            kernels = launched_kernels(call)
        else:
            call()
        return d_first.cpu().numpy(), d_links.cpu().numpy(), kernels
    finally:
        del d_bytes
        torch.cuda.empty_cache()


def _mixed_files(n):
    base = [CASES[k][0] for k in CASES] + [b"".join(p) for p, _, _ in _random_chains(3, 6)]
    return [base[i % len(base)] for i in range(n)]


def test_dev_form_and_caps(cuda_ok):
    _need()
    for n in (1, 5, 1000):
        files = _mixed_files(n)
        host = lib.ogg_links(files)
        total = int(host["link_first"][-1])
        first, links, _ = _dev_call(files, total)
        assert np.array_equal(first, host["link_first"]) and np.array_equal(links, host["link_off"]), n
        # link_cap = 0 sizes the call; one short writes no link_off
        for cap in (0, total - 1):
            first, links, _ = _dev_call(files, cap)
            assert np.array_equal(first, host["link_first"]) and (links == -7).all(), (n, cap)
    files = _mixed_files(5)
    host = lib.ogg_links(files)
    total = int(host["link_first"][-1])
    L = lib.load()
    buf = np.frombuffer(b"".join(files), np.uint8)
    off = host["file_off"]
    first = np.zeros(6, np.int64)
    links = np.full(total + 1, -7, np.int64)
    assert L.vb200_ogg_links(5, buf.ctypes.data, off.ctypes.data, first.ctypes.data, links.ctypes.data, total - 1) \
        == EINVAL
    assert np.array_equal(first, host["link_first"]) and (links == -7).all()
    assert L.vb200_ogg_links(5, buf.ctypes.data, off.ctypes.data, first.ctypes.data, None, 0) == EINVAL
    assert L.vb200_ogg_links(5, buf.ctypes.data, off.ctypes.data, first.ctypes.data, links.ctypes.data, 1 << 40) == 0
    assert np.array_equal(links, host["link_off"])
    bad = off.copy()
    bad[2] = bad[3] + 1
    assert L.vb200_ogg_links(5, buf.ctypes.data, bad.ctypes.data, first.ctypes.data, links.ctypes.data, total) == EINVAL
    assert L.vb200_ogg_links_dev(1, None, None, None, None, 0, None) == EINVAL
    assert L.vb200_ogg_links(0, None, off.ctypes.data, first.ctypes.data, links.ctypes.data, 1) == 0
    assert first[0] == 0 and links[0] == 0
    r = lib.ogg_links([])
    assert list(r["link_first"]) == [0] and list(r["link_off"]) == [0]


def test_unequal_files_in_one_cta(cuda_ok):
    _need()
    rng = np.random.default_rng(12)
    src = _sources()
    big = b""
    while len(big) < 20e6:
        pages, _, _ = _chain(rng, src, 12)
        big += b"".join(pages)
    files = [CASES["empty"][0], big, CASES["same serial"][0], CASES["multiplexed"][0], CASES["single link"][0],
             CASES["truncated link"][0]]                   # CTA 0: tiny, 20 MB, tiny, tiny; CTA 1: two tiny
    _check_table(lib.ogg_links(files), files, "unequal files")


def test_offsets_past_2_31(cuda_ok):
    _need()
    import torch
    if torch.cuda.mem_get_info()[0] < 6 << 30:
        pytest.skip("6 GB of free device memory needed")
    files = _mixed_files(12)
    host = lib.ogg_links(files)
    pad = (1 << 31) + 1
    first, links, _ = _dev_call(files, int(host["link_first"][-1]), pad=pad)
    assert np.array_equal(first, host["link_first"]) and np.array_equal(links, host["link_off"] + pad)


def test_launches(cuda_ok):
    """three kernels (count, offsets, write) at 1 and at 1000 files, counted with torch.profiler in a process of its
    own (a profiler session of another test in the same process can lose the kernel records of a later one)"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_ogg_links as T; "
            "files = [T.CASES[k][0] for k in T.CASES] * 100; "
            "print(json.dumps([T._dev_call(files[:n], 10000, profiled=True)[2] for n in (1, 1000)]))" % (here, os.path.dirname(here)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=here)
    assert r.returncode == 0, r.stderr[-3000:]
    for kernels in json.loads(r.stdout.strip().splitlines()[-1]):
        assert len(kernels) == 3 and "k_ogg_links_count" in kernels[0] and "k_ds_scan" in kernels[1] and \
            "k_ogg_links_write" in kernels[2], kernels
