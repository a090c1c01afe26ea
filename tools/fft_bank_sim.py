#!/usr/bin/env python
"""Shared-memory bank model of the real-FFT passes of k_phaseA_transform (dev_fft_pass4 / dev_fft_pass2 in
vorbis_b200/csrc/vb200_kernels.cuh), to choose a padding of the ping-pong buffers before spending GPU time.

Counts wavefronts per (block,channel) row the way the hardware serves a warp request: 32 banks x 4 B; a 32-bit
request costs max over banks of the number of distinct words; a 64-bit request is served per half-warp, a
128-bit one per quarter-warp.  Lanes of a warp that take different branches issue separate instructions.
Compare with the shared-memory bank conflicts by source line of a profile of k_phaseA_transform.

usage: tools/fft_bank_sim.py [N] [threads]
"""
import sys
from collections import defaultdict

N = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
NT = int(sys.argv[2]) if len(sys.argv) > 2 else 256


def wavefronts(addrs, width):
    """addrs: list of (lane, float_index) for the active lanes of ONE warp instruction; width in floats"""
    group = {1: 32, 2: 16, 4: 8}[width]
    total = 0
    for g0 in range(0, 32, group):
        words = defaultdict(set)
        for lane, a in addrs:
            if g0 <= lane < g0 + group:
                for w in range(width):
                    words[(a + w) % 32].add(a + w)
        if words:
            total += max(len(v) for v in words.values())
    return total


def passes(n):
    log2n = n.bit_length() - 1
    nf = (log2n + 1) >> 1
    l2 = n
    out = []
    for k1 in range(nf):
        ip = 2 if (k1 == nf - 1 and (log2n & 1)) else 4
        l1, ido = l2 // ip, n // l2
        out.append((ip, l1, ido, k1 == 0))
        l2 = l1
    return out


def sim(pad):
    """returns {pass: (load_wavefronts, store_wavefronts)} for one row"""
    res = {}
    for ip, l1, ido, first in passes(N):
        t0 = l1 * ido
        rd = (lambda e: pad(e)) if first else (lambda e: pad(e + 1))       # first pass reads the unshifted input
        wr = lambda e: pad(e + 1)
        loads = stores = 0
        if ido == 1:
            items = l1
        else:
            half = ido >> 1
            items = l1 * half + l1
        for w0 in range(0, items, 32):                                     # warps (NT only changes the order)
            ins_l, ins_s = defaultdict(list), defaultdict(list)            # (branch, slot, width) -> [(lane, addr)]
            for lane in range(32):
                v = w0 + lane
                if v >= items:
                    continue
                if ido == 1:
                    k = v
                    for s in range(ip):
                        ins_l[("a", s, 1)].append((lane, rd(k + s * t0)))
                    o = ip * k
                    if ip == 4:
                        ins_s[("a", 0, 1)].append((lane, wr(o)))
                        ins_s[("a", 1, 2)].append((lane, wr(o + 1)))
                        ins_s[("a", 2, 1)].append((lane, wr(o + 3)))
                    else:
                        ins_s[("a", 0, 1)].append((lane, wr(o)))
                        ins_s[("a", 1, 1)].append((lane, wr(o + 1)))
                    continue
                half = ido >> 1
                if v < l1 * half:
                    k, ii = v // half, v % half
                    c = [k * ido + s * t0 for s in range(ip)]
                    o = ip * k * ido
                    if ii == 0:
                        for s in range(ip):
                            ins_l[("b", s, 1)].append((lane, rd(c[s])))
                        tgt = [o, o + 4 * ido - 1, o + 2 * ido - 1, o + 2 * ido] if ip == 4 else [o, o + 2 * ido - 1]
                        for s, a in enumerate(tgt):
                            ins_s[("b", s, 1)].append((lane, wr(a)))
                    else:
                        i = 2 * ii
                        for s in range(ip):
                            ins_l[("c", s, 2)].append((lane, rd(c[s] + i - 1)))
                        ic = 2 * ido - i
                        tgt = ([o + i - 1, o + ic - 1, o + 2 * ido + i - 1, o + 2 * ido + ic - 1] if ip == 4
                               else [o + i - 1, o + ic - 1])
                        for s, a in enumerate(tgt):
                            ins_s[("c", s, 2)].append((lane, wr(a)))
                else:
                    k = v - l1 * half
                    c = [k * ido + s * t0 for s in range(ip)]
                    o = ip * k * ido
                    for s in range(ip):
                        ins_l[("d", s, 1)].append((lane, rd(c[s] + ido - 1)))
                    tgt = [o + ido - 1, o + 3 * ido - 1, o + ido, o + 3 * ido] if ip == 4 else [o + ido, o + ido - 1]
                    for s, a in enumerate(tgt):
                        ins_s[("d", s, 1)].append((lane, wr(a)))
            loads += sum(wavefronts(a, key[2]) for key, a in ins_l.items())
            stores += sum(wavefronts(a, key[2]) for key, a in ins_s.items())
        res[(ip, l1, ido)] = (loads, stores)
    return res


PADS = {
    "none": lambda a: a,
    "2 per 32": lambda a: a + 2 * (a >> 5),
    "2 per 32 + 2 per 512": lambda a: a + 2 * (a >> 5) + 2 * (a >> 9),
    "2 per 16": lambda a: a + 2 * (a >> 4),
    "4 per 64": lambda a: a + 4 * (a >> 6),
    "2 per 32 + 4 per 256": lambda a: a + 2 * (a >> 5) + 4 * (a >> 8),
}

if __name__ == "__main__":
    print("real FFT of N=%d, wavefronts per row (loads + stores); the ideal is one per 32 lanes x 4 B" % N)
    for name, pad in PADS.items():
        r = sim(pad)
        tot_l = sum(v[0] for v in r.values())
        tot_s = sum(v[1] for v in r.values())
        extra = max(pad(N + 1) - (N + 1), 0)
        print("%-22s loads %5d stores %5d total %5d  (+%d floats per buffer)" % (name, tot_l, tot_s, tot_l + tot_s, extra))
        if name in ("none", "2 per 32"):
            for (ip, l1, ido), (l, s) in r.items():
                print("      radix %d  l1=%4d ido=%4d   loads %5d stores %5d" % (ip, l1, ido, l, s))
