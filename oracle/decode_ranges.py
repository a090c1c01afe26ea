"""A plain restatement of vb200_decode_ranges' plan, in Python: which blocks a range of a stream's output needs and
which of their finished samples it keeps.

  blocks(...)   the header of every packet and blockin's bookkeeping from a fresh state (lib/synthesis.c:41-71,
                lib/block.c:741-751, 835-941, >> hs at half rate): per packet its status, samples, granulepos and
                pcm_offset, the stream's length, and per decoded block its packet, window [lo, hi) and position
  plan(...)     for samples [start, start + length): the priming block (the decoded block before the first that
                meets the range), the blocks up to the last that meets it, and per block after the first the part of
                its finished samples the range keeps

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product.
"""
import numpy as np

from oracle.decode import META                      # audio rows: offset, bytes, granulepos, e_o_s, packetno

ENOTAUDIO, EBADPACKET = -135, -136


def packet_header(buf, off, nbytes, modebits):
    """vorbis_synthesis' header read: the block flag, or ENOTAUDIO / EBADPACKET (modes 0 and 1 have flags 0, 1)"""
    nbits, pos = 8 * max(int(nbytes), 0), 0

    def read(k):
        nonlocal pos
        if pos + k > nbits:
            pos = nbits + 1
            return -1
        v = 0
        for i in range(k):
            b = pos + i
            v |= ((int(buf[off + b // 8]) >> (b % 8)) & 1) << i
        pos += k
        return v

    if read(1) != 0:
        return ENOTAUDIO
    mode = read(modebits)
    if mode < 0 or mode > 1:
        return EBADPACKET
    if mode == 1:
        read(1)
        return EBADPACKET if read(1) == -1 else 1
    return 0


def blocks(buf, audio, bs, modebits, halfrate=False):
    """a stream's packets (audio rows into buf) decoded from a fresh state -> (length, packets, blocks) with
    packets int64 [npkt][4] = (pcm_offset, granulepos, samples, status) and blocks a list of dicts
    {k: packet index, W, offset, bytes, fin: the samples it finishes, lo, hi, pos: the stream's output before it}"""
    audio = np.asarray(audio, np.int64).reshape(-1, META)
    hs = 1 if halfrate else 0
    gp, count, seq, lastW = -1, -1, -1, -1
    pos = 0
    packets = np.zeros((len(audio), 4), np.int64)
    out = []
    for k, (off, nbytes, pgp, eos, pno) in enumerate(audio.tolist()):
        W = packet_header(buf, off, nbytes, modebits)
        if W < 0:
            packets[k] = (pos, gp, 0, W)
            continue
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
        lastW = W
        packets[k] = (pos, gp, hi - lo, 0)
        out.append(dict(k=k, W=W, offset=off, bytes=nbytes, fin=fin, lo=lo, hi=hi, pos=pos))
        pos += hi - lo
    return pos, packets, out


def plan(blks, start, length):
    """samples [start, start + length) of the stream whose blocks are blks -> (got, kept) where kept is the list of
    blocks to decode in order, the first of which primes, each after the first with "keep" = (lo, hi) of its
    finished samples and "at" = where they go in the range; kept is empty when nothing of the range exists"""
    t0, t1 = start, start + length
    meet = [j for j, b in enumerate(blks)
            if b["hi"] > b["lo"] and b["pos"] < t1 and b["pos"] + b["hi"] - b["lo"] > t0]
    if length == 0 or not meet:
        return 0, []
    j0, j1 = meet[0], meet[-1]
    assert j0 >= 1                                   # the first decoded block returns nothing
    kept = [dict(blks[j0 - 1])]
    for b in blks[j0:j1 + 1]:
        b = dict(b)
        a, e = max(b["pos"], t0), min(b["pos"] + b["hi"] - b["lo"], t1)
        b["keep"] = (b["lo"] + a - b["pos"], b["lo"] + e - b["pos"]) if a < e else (0, 0)
        b["at"] = a - t0
        kept.append(b)
    end = blks[-1]["pos"] + blks[-1]["hi"] - blks[-1]["lo"]
    return min(t1, end) - t0, kept


def capacity(out_stride, bs, channels, halfrate=False):
    """a request's block slots and residue floats in vb200_decode_ranges (rounded up to 64 floats)"""
    hs = 1 if halfrate else 0
    res = channels * (2 * (out_stride << hs) + 3 * (bs[1] // 2))
    return (out_stride << hs) // (bs[0] // 2) + 3, (res + 63) // 64 * 64
