"""Ogg pages in plain Python: the demux rules of vb200_ogg_demux (include/vorbis_b200.h) restated one page at a time,
and a seeded page writer (RFC 3533) that makes the files the tests feed it.

demux() follows libogg's ogg_sync_pageseek (capture, CRC, resync at the next 'O'), ogg_stream_pagein and
ogg_stream_packetout (lacing, sequence holes, continued pages, granulepos on the last packet that ends on a page,
e_o_s) and vorbisfile's choice of the first Vorbis BOS page's serial, as the header states them.  It has not been run
against libogg itself.  Test infrastructure: nothing in the product imports it."""
import struct

import numpy as np

ENOTVORBIS, EBADHEADER, EINVAL = -132, -133, -131


def _crc_table():
    t = []
    for i in range(256):
        r = i << 24
        for _ in range(8):
            r = ((r << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if r & 0x80000000 else (r << 1) & 0xFFFFFFFF
        t.append(r)
    return t


CRC_TABLE = _crc_table()


def crc32(page):
    """the Ogg page CRC: polynomial 0x04c11db7, not reflected, initial 0, no final xor"""
    c, t = 0, CRC_TABLE
    for b in page:
        c = ((c << 8) & 0xFFFFFFFF) ^ t[(c >> 24) ^ b]
    return c


def page(flags, granulepos, serial, seq, lacing, body, version=0):
    """one page with its CRC"""
    head = b"OggS" + struct.pack("<BBqIIIB", version, flags, granulepos, serial, seq, 0, len(lacing)) + bytes(lacing)
    raw = bytearray(head + bytes(body))
    raw[22:26] = struct.pack("<I", crc32(raw))
    return bytes(raw)


def write(packets, granules, serial, rng, max_segs=255, min_segs=1, headers_alone=True, seq0=0):
    """packets (bytes; the three headers first) -> list of pages.  Packet 0 alone on the BOS page when headers_alone
    (and packets 1, 2 then end their own run of pages, as libvorbis' encoder flushes them); otherwise, and for the audio
    packets, each page takes a seeded number of segments in [min_segs, max_segs], so packets span pages and pages may end
    none.  granulepos of a page: that of the last packet ending on it, -1 where none ends.  BOS on the first page, EOS
    on the last."""
    segs = []                                   # (packet index, lacing value, the packet ends here)
    for i, p in enumerate(packets):
        n = len(p)
        lac = [255] * (n // 255) + [n % 255]
        segs += [(i, v, k == len(lac) - 1) for k, v in enumerate(lac)]
    blob = b"".join(packets)
    pages, at, pos, seq, cont = [], 0, 0, seq0, False
    while at < len(segs):
        if headers_alone and segs[at][0] < 3:
            # up to the end of the current header packet (at most 255 segments per page)
            end = at
            while end < len(segs) and end - at < 255 and segs[end][0] == segs[at][0]:
                end += 1
        else:
            end = min(len(segs), at + int(rng.integers(min_segs, max_segs + 1)))
        chunk = segs[at:end]
        nbytes = sum(v for _, v, _ in chunk)
        ends = [i for i, _, e in chunk if e]
        gp = int(granules[ends[-1]]) if ends else -1
        flags = (1 if cont else 0) | (2 if at == 0 else 0) | (4 if end == len(segs) else 0)
        pages.append(page(flags, gp, serial, seq, [v for _, v, _ in chunk], blob[pos:pos + nbytes]))
        cont = not chunk[-1][2]
        pos += nbytes
        seq += 1
        at = end
    return pages


def demux(buf, max_packets):
    """one Ogg file (bytes) -> dict: status, serial, pages, dropped, holes, foreign, chained, hdr [(offset, bytes)]
    (offsets counted from the file's first byte, as vb200_ogg_demux places them in data), packets [(offset, bytes,
    granulepos, e_o_s, packetno)] and the packet bytes of every entry ("hdr_data", "pkt_data")"""
    buf = bytes(buf)
    end = len(buf)
    r = dict(status=0, serial=0, pages=0, dropped=0, holes=0, foreign=0, chained=0)
    hdr, pkts = [], []
    out = bytearray(end)
    have_serial = done = have_seq = pending = stop = False
    next_seq = 0
    w = pstart = 0
    packetno = 0
    p = 0
    while not stop:
        if end - p < 27:
            break
        ok = buf[p:p + 4] == b"OggS"
        if ok:
            nseg = buf[p + 26]
            if end - p < 27 + nseg:
                break
            lace = list(buf[p + 27:p + 27 + nseg])
            body = sum(lace)
            if end - p < 27 + nseg + body:
                break
            raw = bytearray(buf[p:p + 27 + nseg + body])
            want = struct.unpack("<I", bytes(raw[22:26]))[0]
            raw[22:26] = b"\0\0\0\0"
            ok = crc32(raw) == want
        if not ok:
            r["dropped"] += 1
            q = buf.find(b"O", p + 1)
            p = end if q < 0 else q
            continue
        body0 = p + 27 + nseg
        ver, flags, granule, ser, seq = struct.unpack("<BBqII", buf[p + 4:p + 22])
        p = body0 + body
        if done:
            r["chained"] = 1 if flags & 2 else 0
            break
        if not have_serial:
            vorbis = False
            if flags & 2 and ver == 0:
                first = 0
                for v in lace:
                    first += v
                    if v < 255:
                        break
                vorbis = first >= 7 and buf[body0:body0 + 7] == b"\x01vorbis"
            if not vorbis:
                r["foreign"] += 1
                continue
            have_serial, r["serial"] = True, ser
        elif ser != r["serial"] or ver != 0:
            r["foreign"] += 1
            continue
        r["pages"] += 1
        if have_seq and seq != next_seq:
            if pending:
                w, pending = pstart, False
            r["holes"] += 1
            packetno += 1
            if len(hdr) < 3:
                break
        have_seq, next_seq = True, (seq + 1) & 0xFFFFFFFF
        seg, src = 0, body0
        if flags & 1 and not pending:
            while seg < nseg:
                v = lace[seg]
                seg += 1
                src += v
                if v < 255:
                    break
        ncopy = body0 + body - src
        out[w:w + ncopy] = buf[src:src + ncopy]
        lastc = max([i for i in range(seg, nseg) if lace[i] < 255], default=-1)
        if not pending:
            pstart = w
        q = w
        for i in range(seg, nseg):
            q += lace[i]
            if lace[i] == 255:
                continue
            n = q - pstart
            if len(hdr) < 3:
                hdr.append((pstart, n))
            elif len(pkts) == max_packets:
                r["status"], stop = EINVAL, True
                break
            else:
                pkts.append((pstart, n, granule if i == lastc else -1, 1 if flags & 4 and i == nseg - 1 else 0,
                             packetno))
            packetno += 1
            pstart = q
        w = q
        if nseg > seg:
            pending = lace[nseg - 1] == 255
        if flags & 4:
            done = True
    if not have_serial:
        r["status"] = ENOTVORBIS
    elif len(hdr) < 3:
        r["status"] = EBADHEADER
        pkts = []
    r["hdr"], r["packets"] = hdr, pkts
    r["hdr_data"] = [bytes(out[o:o + n]) for o, n in hdr]
    r["pkt_data"] = [bytes(out[o:o + n]) for o, n, _, _, _ in pkts]
    return r


def file_of(enc, rng, serial=None, **kw):
    """the pages of an Ogg file of one stream (oracle.decode.Packets: three headers, then audio); the packets' own
    granulepos go on the pages"""
    meta = enc.meta
    packets = [bytes(enc.buf[int(o):int(o + n)]) for o, n in meta[:, :2]]
    granules = [int(g) for g in meta[:, 2]]
    serial = int(rng.integers(0, 1 << 32)) if serial is None else serial
    return write(packets, granules, serial, rng, **kw)


def packet_table(r):
    """oracle demux result -> np.ndarray of (offset, bytes, granulepos, e_o_s, packetno) rows, int64"""
    return np.array([list(x) for x in r["packets"]], np.int64).reshape(-1, 5)
