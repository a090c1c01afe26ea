"""The link rule of vb200_ogg_links (include/vorbis_b200.h) in plain Python, one captured page at a time.

capture() restates the page capture of oracle.ogg.demux (libogg's ogg_sync_pageseek: capture pattern, CRC, resync at
the next 'O', the end-of-file rules) as a step of its own, and links() walks the captured pages with the rule: a link
starts at the file's first byte and at every captured page with the BOS flag that follows a captured page without it.
Test infrastructure: nothing in the product imports it."""
import struct

from .ogg import crc32


def capture(buf, p):
    """ogg_sync_pageseek at byte p of one file (bytes): ("page", the page's end) for a captured page; ("resync", the
    next 'O' after p or the end of the file) for a failed capture; ("end", None) when fewer than 27 bytes are left or
    the page is cut short by the end of the file"""
    end = len(buf)
    if end - p < 27:
        return "end", None
    if buf[p:p + 4] == b"OggS":
        nseg = buf[p + 26]
        if end - p < 27 + nseg:
            return "end", None
        n = 27 + nseg + sum(buf[p + 27:p + 27 + nseg])
        if end - p < n:
            return "end", None
        raw = bytearray(buf[p:p + n])
        want = struct.unpack("<I", bytes(raw[22:26]))[0]
        raw[22:26] = b"\0\0\0\0"
        if crc32(raw) == want:
            return "page", p + n
    q = buf.find(b"O", p + 1)
    return "resync", end if q < 0 else q


def pages_of(buf):
    """the captured pages of one file (bytes), in order: [(offset, end)]"""
    buf = bytes(buf)
    out, p = [], 0
    while True:
        kind, at = capture(buf, p)
        if kind == "end":
            return out
        if kind == "page":
            out.append((p, at))
        p = at


def links(buf):
    """the links of one file (bytes), as vb200_ogg_links finds them: the byte offsets of its links' starts, from the
    file's first byte, then the end of the file"""
    buf = bytes(buf)
    out, after_data = [0], False
    for p, _ in pages_of(buf):
        bos = bool(buf[p + 5] & 2)
        if bos and after_data:
            out.append(p)
        after_data = not bos
    return out + [len(buf)]
