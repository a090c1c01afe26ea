"""Ogg pages out in plain Python: the page mux of vb200_ogg_mux (include/vorbis_b200.h) restated as libogg 1.3.x's
framing.c behaves, one packet at a time, the way examples/encoder_example.c drives it: ogg_stream_packetin of the three
header packets and ogg_stream_flush until it returns 0, then for every audio packet ogg_stream_packetin and
ogg_stream_pageout until it returns 0.

Stream is a literal restatement of the stream state (a FIFO of lacing values, each marked as the first of its packet
and carrying a granule, b_o_s, e_o_s, pageno) and of ogg_stream_flush_i, not a closed form, so that the device's
closed-form walk is checked against a step-by-step model.  It has not been run against libogg itself (libogg is not
part of this project); where it differs from libogg, libogg is right.  The page bytes come from oracle.ogg.page, the CRC
the demux checks.  Test infrastructure: nothing in the product imports it."""
from . import ogg

EINVAL = ogg.EINVAL
FRESH, WRITING, DONE = 0, 1, 2


class Stream:
    """ogg_stream_state, with the packet index of every lacing value kept so that a call can say which packets are
    not yet wholly on pages"""

    def __init__(self, serial, pageno=0, b_o_s=False):
        self.serial, self.pageno, self.b_o_s, self.e_o_s = serial, pageno, b_o_s, False
        self.lacing = []            # [value, first segment of its packet, granule, packet index, segment index]
        self.body = bytearray()

    def packetin(self, data, granule, eos, index=0, skip=0):
        """ogg_stream_packetin; skip > 0 leaves out the packet's first `skip` lacing values and their bytes (they are
        already on pages: the kept packet of a carry)"""
        n = len(data)
        vals = [255] * (n // 255) + [n % 255]
        for i, v in enumerate(vals):
            if i >= skip:
                self.lacing.append([v, i == 0, -1, index, i])
        self.lacing[-1][2] = granule
        self.body += bytes(data)[skip * 255:]
        if eos:
            self.e_o_s = True

    def flush_i(self, force, nfill=4096):
        """ogg_stream_flush_i: one page (bytes) or None"""
        fill = len(self.lacing)
        maxvals = min(fill, 255)
        if maxvals == 0:
            return None
        if not self.b_o_s:          # the initial header page: up to and including the first value below 255
            gp = 0
            vals = 0
            while vals < maxvals:
                last = self.lacing[vals][0] < 255
                vals += 1
                if last:
                    break
        else:
            acc = done = just = 0
            gp = -1
            vals = 0
            while vals < maxvals:
                if acc > nfill and just >= 4:
                    force = True
                    break
                v = self.lacing[vals]
                acc += v[0]
                if v[0] < 255:
                    gp = v[2]
                    done += 1
                    just = done
                else:
                    just = 0
                vals += 1
            if vals == 255:
                force = True
        if not force:
            return None
        flags = (0 if self.lacing[0][1] else 1) | (0 if self.b_o_s else 2) | (4 if self.e_o_s and fill == vals else 0)
        lac = [v[0] for v in self.lacing[:vals]]
        nb = sum(lac)
        pg = ogg.page(flags, gp, self.serial, self.pageno, lac, self.body[:nb])
        self.pageno = (self.pageno + 1) & 0xFFFFFFFF
        self.b_o_s = True
        del self.lacing[:vals]
        del self.body[:nb]
        return pg

    def pageout(self):
        return self.flush_i(bool(self.lacing) and (self.e_o_s or not self.b_o_s))

    def flush(self):
        return self.flush_i(True)


def _drain(step):
    out = []
    while True:
        pg = step()
        if pg is None:
            return out
        out.append(pg)


def mux(headers, packets, granules, eos, serial, hdr_granules=(0, 0, 0)):
    """three header packets and the audio packets (bytes; granules and eos per audio packet) -> list of pages, as
    encoder_example.c writes them"""
    os_ = Stream(serial)
    pages = []
    for h, g in zip(headers, hdr_granules):
        os_.packetin(h, g, False)
    pages += _drain(os_.flush)
    for p, g, e in zip(packets, granules, eos):
        os_.packetin(p, g, e)
        pages += _drain(os_.pageout)
    return pages


def fresh_carry(serial):
    return dict(serial=serial, pageno=0, state=FRESH, kept=0, kept_segs=0)


def mux_call(carry, headers, packets, granules, eos, hdr_granules=(0, 0, 0)):
    """one call of vb200_ogg_mux for one stream: the carry (a dict of vb200_ogg_mux_carry's fields), the header
    packets (read only for a fresh carry) and this call's audio packets, the carry's kept ones first.  Returns (status,
    pages, new carry); on EINVAL no pages and the carry as it was."""
    n = len(packets)
    bad = (not 0 <= carry["state"] <= DONE or n < carry["kept"] or carry["kept"] < 0 or carry["kept_segs"] < 0 or
           (carry["state"] == DONE and n) or (carry["state"] == FRESH and (headers is None or carry["kept"])) or
           any(eos[:-1]) or
           (carry["kept_segs"] and (not carry["kept"] or carry["kept_segs"] > len(packets[0]) // 255)))
    if bad:
        return EINVAL, [], dict(carry)
    os_ = Stream(carry["serial"], carry["pageno"], b_o_s=carry["state"] != FRESH)
    pages = []
    if carry["state"] == FRESH:
        for h, g in zip(headers, hdr_granules):
            os_.packetin(h, g, False, index=-1)
        pages += _drain(os_.flush)
    for k, (p, g, e) in enumerate(zip(packets, granules, eos)):
        os_.packetin(p, g, e, index=k, skip=carry["kept_segs"] if k == 0 else 0)
        pages += _drain(os_.pageout)
    new = dict(carry, pageno=os_.pageno)
    if carry["state"] == DONE or (n and eos[-1]):
        new.update(state=DONE, kept=0, kept_segs=0)
    else:
        new["state"] = WRITING
        new["kept"] = n - os_.lacing[0][3] if os_.lacing else 0
        new["kept_segs"] = os_.lacing[0][4] if os_.lacing else 0
    return 0, pages, new


def mux_pieces(headers, packets, granules, eos, serial, cuts, hdr_granules=(0, 0, 0)):
    """the same stream through calls with carries: call i passes the kept packets of the call before, then the new
    packets up to cuts[i] (non-decreasing; the last call ends at the last packet).  Returns (pages, carries after each
    call)"""
    carry, pages, carries, at = fresh_carry(serial), [], [], 0
    for end in list(cuts) + [len(packets)]:
        lo = at - carry["kept"]
        st, pg, carry = mux_call(carry, headers, packets[lo:end], granules[lo:end], eos[lo:end], hdr_granules)
        assert st == 0
        pages += pg
        carries.append(dict(carry))
        at = end
    return pages, carries
