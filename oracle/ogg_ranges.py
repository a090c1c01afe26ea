"""A plain restatement of vb200_ogg_ranges' plan (include/vorbis_b200.h), in Python: sample ranges of Ogg rows found
by a seek on page granulepos instead of a walk from the first packet.

  head(...)     the row's serial, its header packets and G0 from the first audio packet that carries a granulepos
  bisect(...)   the page P a request starts after: bisection over byte offsets, then a forward scan
  anchor(...)   block 1's granulepos and position, counted back from the next granulepos after P
  request(...)  one request: the mode (fresh, seek or empty), P, and decode_ranges.plan's (got, kept) form

The pages are captured with oracle.ogg_links.capture and walked with oracle.ogg.demux's pagein and packetout rules;
blockin's bookkeeping is that of oracle.decode_ranges.blocks.  The packet scratch is taken as large enough.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import struct

from oracle.decode_ranges import packet_header
from oracle.ogg_links import capture

ENOTVORBIS, EBADHEADER = -132, -133
SCAN = 8192                                          # the bisection's shortest window


def _page(buf, p):
    """(version, flags, granulepos, serial, sequence, lacing) of the captured page at p"""
    ver, flags, granule, ser, seq = struct.unpack("<BBqII", buf[p + 4:p + 22])
    nseg = buf[p + 26]
    return ver, flags, granule, ser, seq, list(buf[p + 27:p + 27 + nseg])


def walk(buf, p, serial=None, skip_page=-1, modebits=1):
    """the packets of one serial from byte p, as vb200_ogg_demux's walk takes them: yields ("hole", None) and
    ("packet", {W, data, granulepos, e_o_s, packetno, page}); the serial is fixed by the first Vorbis BOS page when
    None.  Packets that end on the page at skip_page are not yielded.  The walk ends past the serial's EOS page.
    The serial found is in walk.serial after the first yield (None when the row has none)."""
    end = len(buf)
    walk.serial = serial
    have_seq = pending = False
    next_seq = packetno = 0
    cur, W = bytearray(), -135
    while True:
        kind, at = capture(buf, p)
        if kind == "end":
            return
        if kind == "resync":
            p = at
            continue
        page = p
        ver, flags, granule, ser, seq, lace = _page(buf, p)
        nseg = len(lace)
        body0 = p + 27 + nseg
        p = at
        if walk.serial is None:
            vorbis = False
            if flags & 2 and ver == 0:
                first = 0
                for v in lace:
                    first += v
                    if v < 255:
                        break
                vorbis = first >= 7 and buf[body0:body0 + 7] == b"\x01vorbis"
            if not vorbis:
                continue
            walk.serial = ser
        elif ser != walk.serial or ver != 0:
            continue
        if have_seq and seq != next_seq:
            if pending:
                cur, pending = bytearray(), False
            packetno += 1
            yield "hole", None
        have_seq, next_seq = True, (seq + 1) & 0xFFFFFFFF
        seg, src = 0, body0
        if flags & 1 and not pending:
            while seg < nseg:
                v = lace[seg]
                seg += 1
                src += v
                if v < 255:
                    break
        lastc = max([i for i in range(seg, nseg) if lace[i] < 255], default=-1)
        for i in range(seg, nseg):
            v = lace[i]
            if not pending:
                pending, cur = True, bytearray()
                W = packet_header(buf, src, v, modebits)
            cur += buf[src:src + v]
            src += v
            if v == 255:
                continue
            pending = False
            k = dict(W=W, data=bytes(cur), granulepos=granule if i == lastc else -1,
                     e_o_s=1 if flags & 4 and i == nseg - 1 else 0, packetno=packetno, page=page)
            packetno += 1
            if page != skip_page:
                yield "packet", k
        if flags & 4:
            return


def _blockin(h, W, pgp, eos, pno, bs, hs):
    """blockin's bookkeeping for one accepted packet (oracle.decode_ranges.blocks' step): h = [gp, count, seq, lastW]
    advances; returns the window (lo, hi) of the block's finished samples"""
    gp, count, seq, lastW = h
    fin = (bs[lastW] // 4 + bs[W] // 4) >> hs if lastW >= 0 else 0
    if seq == -1 or seq + 1 != pno:
        gp, count = -1, -1
    seq = pno
    lo, hi = 0, fin
    count = 0 if count == -1 else count + bs[lastW] // 4 + bs[W] // 4
    if gp == -1:
        if pgp != -1:
            gp = pgp
            if count > gp:
                extra = max(count - pgp, 0)
                if eos:
                    hi -= min(extra, (hi - lo) << hs) >> hs
                else:
                    lo = min(lo + (extra >> hs), hi)
    else:
        gp += bs[lastW] // 4 + bs[W] // 4
        if pgp != -1 and gp != pgp:
            if gp > pgp and eos:
                hi -= max(min(gp - pgp, (hi - lo) << hs), 0) >> hs
            gp = pgp
    h[:] = [gp, count, seq, W]
    return lo, hi


def head(buf, bs, modebits, halfrate=False):
    """-> dict(status, serial, g1, c1, G0, a1 (the page that ends g1's packet), a1_end); g1 None without one"""
    hs = 1 if halfrate else 0
    returned, h, c1 = 0, [-1, -1, -1, -1], 0
    r = dict(status=0, serial=None, g1=None, c1=None, G0=None, a1=None, a1_end=None)
    for kind, k in walk(buf, 0, modebits=modebits):
        if kind == "hole":
            if returned < 3:
                break
            continue
        returned += 1
        if returned <= 3 or k["W"] < 0:
            continue
        lo, hi = _blockin(h, k["W"], k["granulepos"], k["e_o_s"], k["packetno"], bs, hs)
        c1 += hi - lo
        if k["granulepos"] != -1:
            r.update(g1=k["granulepos"], c1=c1, G0=k["granulepos"] - (c1 << hs), a1=k["page"],
                     a1_end=capture(buf, k["page"])[1])
            break
    r["serial"] = walk.serial
    if walk.serial is None:
        r["status"] = ENOTVORBIS
    elif returned < 3:
        r["status"] = EBADHEADER
    return r


def _next_gpage(buf, x, hi, serial):
    """the first page of the serial with a granulepos captured from byte x on and starting before hi: (offset, end,
    granulepos, flags) or None"""
    while x < hi:
        kind, at = capture(buf, x)
        if kind == "end":
            return None
        if kind == "resync":
            x = at
            continue
        ver, flags, granule, ser, _, _ = _page(buf, x)
        if ser == serial and ver == 0 and granule != -1:
            return x, at, granule, flags
        x = at
    return None


def bisect(buf, hd, T):
    """P for target granulepos T (hd["g1"] <= T): (offset, granulepos, flags)"""
    serial, end = hd["serial"], len(buf)
    best = (hd["a1"], hd["g1"], buf[hd["a1"] + 5])
    lo, hi = hd["a1_end"], end
    while hi - lo > SCAN:
        mid = lo + (hi - lo) // 2
        f = _next_gpage(buf, mid, hi, serial)
        if f is not None and not f[3] & 2 and f[2] <= T:
            best, lo = (f[0], f[2], f[3]), f[1]
        else:
            hi = mid
    x = lo
    while True:
        f = _next_gpage(buf, x, end, serial)
        if f is None or f[3] & 2 or f[2] > T:
            break
        best = (f[0], f[2], f[3])
        if f[3] & 4:
            break
        x = f[1]
    return best


def anchor(buf, hd, P, bs, modebits, halfrate=False):
    """(block 1's granulepos, its position) from the walk after P, or None (no anchor, or the e_o_s packet)"""
    hs = 1 if halfrate else 0
    lW, rel = -1, 0
    for kind, k in walk(buf, P, hd["serial"], P, modebits):
        if kind == "hole" or k["W"] < 0:
            continue
        if lW >= 0:
            rel += bs[lW] // 4 + bs[k["W"]] // 4
        lW = k["W"]
        if k["granulepos"] != -1:
            if k["e_o_s"]:
                return None
            g = k["granulepos"]
            return g - rel, ((g - hd["G0"]) >> hs) - (rel >> hs)
    return None


def request(buf, bs, modebits, start, length, halfrate=False, hd=None):
    """one request on one row (bytes) -> dict(got, mode ("fresh", "seek", "empty" or None on a row error), P, T,
    kept): kept in oracle.decode_ranges.plan's form (the priming block first; every later block with "keep" = (lo, hi)
    of its finished samples and "at" = where they go), each with its packet bytes as "data" and "W"."""
    buf = bytes(buf)
    hs = 1 if halfrate else 0
    hd = head(buf, bs, modebits, halfrate) if hd is None else hd
    out = dict(got=0, mode=None, P=None, T=None, kept=[], head=hd)
    if hd["status"]:
        out["got"] = hd["status"]
        return out
    if length == 0:
        return out
    P, a = None, None
    if hd["g1"] is not None:
        T = hd["G0"] + (start << hs) - bs[1] // 2
        out["T"] = T
        if hd["g1"] <= T:
            P, gP, fP = bisect(buf, hd, T)
            if fP & 4:
                out.update(mode="empty", P=P)
                return out
            a = anchor(buf, hd, P, bs, modebits, halfrate)
            if a is None:
                P = None
                if hd["g1"] <= gP - 1:
                    P, gP, fP = bisect(buf, hd, gP - 1)
                    a = None if fP & 4 else anchor(buf, hd, P, bs, modebits, halfrate)
                    if a is None:
                        P = None
    seek = P is not None
    out.update(mode="seek" if seek else "fresh", P=P)
    t0, t1 = start, start + length
    h = [-1, -1, -1, -1]
    pos = a[1] if seek else 0
    hdr, first = (0 if seek else 3), True
    nb, keep, cand, kept = 0, 0, None, []
    for kind, k in walk(buf, P if seek else 0, hd["serial"] if seek else None, P if seek else -1, modebits):
        if kind == "hole":
            continue
        if hdr > 0:
            hdr -= 1
            continue
        if k["W"] < 0:
            continue
        pgp = a[0] if seek and first else k["granulepos"]
        first = False
        lo, hi = _blockin(h, k["W"], pgp, k["e_o_s"], k["packetno"], bs, hs)
        ns = hi - lo
        blk = dict(W=k["W"], data=k["data"], lo=lo, hi=hi, pos=pos)
        if nb == 0:
            if ns == 0 or pos + ns <= t0:
                cand = blk
                pos += ns
                continue
            kept.append(cand)
            nb = 1
        a0, b0 = max(pos, t0), min(pos + ns, t1)
        blk["keep"] = (lo + a0 - pos, lo + b0 - pos) if a0 < b0 else (0, 0)
        blk["at"] = a0 - t0 if a0 < b0 else 0
        kept.append(blk)
        nb += 1
        if a0 < b0:
            keep = nb
        pos += ns
        if pos >= t1:
            break
    out["got"] = max(0, min(pos, t1) - t0)
    out["kept"] = kept[:keep]
    return out
