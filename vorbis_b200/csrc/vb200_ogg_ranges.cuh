// vb200_ogg_ranges.cuh — sample ranges straight from Ogg files (vb200_ogg_ranges[_dev], rules in
// include/vorbis_b200.h): what vb200_decode_ranges returns on the vb200_ogg_demux tables of the same rows, without
// demuxing the rows whole.
//
//   k_or_plan   one converged warp per request.  It walks the row's first pages (ogg_capture, the demux's pagein and
//               packetout rules) to the serial, the header packets and the first audio packet that carries a
//               granulepos, which fixes G0; bisects over byte offsets to the page P the request starts after; walks
//               from P to the next granulepos (the anchor) to fix the positions; then walks from P again, running
//               ds_blockin over the packets as k_dr_plan does, gathering the bytes of the packets it keeps into the
//               request's packet scratch and writing k_dr_plan's compacted block tables.
// then k_decode_packets<true> with requests as its streams and k_synthesis<*, *, SYN_RANGE> (vb200.cu), unchanged.
//
// Only the header bits of a packet decide its block flag, and they lie in its first lacing segment: a segment of
// 255 bytes holds them, a shorter one ends the packet.  So every walk reads the flag from the page the packet
// begins on, and only the final walk copies packet bytes.  While the range is not met the scratch holds the priming
// candidate at offset 0 and the packet being read after it; a candidate is moved to offset 0 when it completes.
#pragma once
#include <climits>
#include "vb200_decode_ranges.cuh"
#include "vb200_ogg.cuh"

constexpr int OR_WARPS = 4;
constexpr int64_t OR_SCAN = 8192;        // the bisection stops at a window this short; a forward scan finishes it

struct OrPlanArgs {
  int nrows, nreq, ch, hs, modebits;
  int bs[2];
  int out_stride;
  int nblk;                  // block slots per request (dr_blocks)
  long long res_cap;         // residue floats per request (dr_residue)
  long long pkt_cap;         // packet bytes per request
  const uint8_t *bytes;
  const int64_t *row_off;
  const vb200_pcm_range *req;
  uint8_t *pkt;              // [nreq][pkt_cap] the gathered packets: the data k_decode_packets<true> reads
  // outputs, as k_dr_plan writes them
  int *Wseq, *pkt_bytes, *count;
  long long *pkt_off, *coef_off, *pcm_off;
  int2 *win;
  long long *base;
  int *got;
};

// a packet the walk completed
struct OrPkt {
  int W;                     // ds_packet_header of its first segment
  int bytes;
  bool lost;                 // its bytes did not fit the scratch (gathering walks only)
  long long granulepos;      // the page's granulepos on the last packet that ends on it, else -1
  int e_o_s;
  long long packetno;        // counted from the walk's start, a hole counting one
  int64_t page;              // offset of the page it ends on
};

// the state of one walk over the pages of one serial: libogg's ogg_stream_pagein / ogg_stream_packetout as
// k_ogg_demux runs them, from byte p on
struct OrWalk {
  int64_t p, end;
  uint32_t serial, next_seq;
  bool have_serial, have_seq, pending, lost;
  long long packetno;
  int64_t skip_page;         // packets that end on the page at this offset are not visited
  uint8_t *dst;              // gathering: the scratch (nullptr: the walk copies nothing)
  long long cap, w, pstart;  // scratch bytes; next free byte; the current packet's first byte
  int W;                     // the current packet's block flag
};

__device__ __forceinline__ OrWalk or_walk_at(int64_t p, int64_t end, bool have_serial, uint32_t serial,
                                             int64_t skip_page, uint8_t *dst, long long cap) {
  OrWalk s;
  s.p = p; s.end = end; s.serial = serial; s.next_seq = 0;
  s.have_serial = have_serial; s.have_seq = false; s.pending = false; s.lost = false;
  s.packetno = 0; s.skip_page = skip_page; s.dst = dst; s.cap = cap; s.w = 0; s.pstart = 0; s.W = -135;
  return s;
}

// bytes [a, e) of the file belong to the current packet
__device__ __forceinline__ void or_piece(OrWalk &s, const uint8_t *bytes, int64_t a, int64_t e, int lane) {
  const long long n = e - a;
  if (s.w + n > s.cap) s.lost = true;
  else if (s.dst && !s.lost)
    for (long long i = lane; i < n; i += 32) s.dst[s.w + i] = bytes[a + i];
  s.w += n;
}

// the granulepos of a captured page
__device__ __forceinline__ int64_t or_granule(const uint8_t *pg) {
  return (int64_t)((uint64_t)ogg_le32(pg + 6) | ((uint64_t)ogg_le32(pg + 10) << 32));
}

// Walk pages from s.p to the end of the row or past the serial's EOS page.  Before the serial is known, the first
// captured Vorbis BOS page fixes it (k_ogg_demux's rule).  visit.packet(OrPkt) for every completed packet and
// visit.hole() at every sequence gap; either returns true to stop the walk.
template <class V>
__device__ __forceinline__ void or_walk(OrWalk &s, const uint8_t *bytes, int lane, const uint32_t *crc_tab,
                                        const uint32_t *xpw, int modebits, V &visit) {
  for (;;) {
    const int len = ogg_capture(bytes, s.p, s.end, lane, crc_tab, xpw);
    if (len < 0) return;
    if (len == 0) continue;
    const uint8_t *pg = bytes + s.p;
    const int64_t page = s.p, body0 = s.p + 27 + pg[26];
    const int nseg = pg[26], ver = pg[4], flags = pg[5];
    const uint32_t ser = ogg_le32(pg + 14), seq = ogg_le32(pg + 18);
    const int64_t granule = or_granule(pg);
    s.p += len;
    if (!s.have_serial) {
      bool vorbis = false;
      if ((flags & 2) && ver == 0) {
        int first = 0;
        for (int i = 0; i < nseg; i++) { first += pg[27 + i]; if (pg[27 + i] < 255) break; }
        const uint8_t *b = bytes + body0;
        vorbis = first >= 7 && b[0] == 1 && b[1] == 'v' && b[2] == 'o' && b[3] == 'r' && b[4] == 'b' && b[5] == 'i' &&
                 b[6] == 's';
      }
      if (!vorbis) continue;
      s.have_serial = true;
      s.serial = ser;
    } else if (ser != s.serial || ver != 0) {
      continue;
    }
    if (s.have_seq && seq != s.next_seq) {
      if (s.pending) { s.w = s.pstart; s.pending = false; }   // the partial packet is dropped
      s.packetno++;
      if (visit.hole()) return;
    }
    s.have_seq = true;
    s.next_seq = seq + 1;
    int seg = 0;
    int64_t src = body0;
    if ((flags & 1) && !s.pending)                       // continued page, nothing to continue: skip the fragment
      while (seg < nseg) {
        const int v = pg[27 + seg++];
        src += v;
        if (v < 255) break;
      }
    int lastc = -1;
    for (int i = seg; i < nseg; i++)
      if (pg[27 + i] < 255) lastc = i;
    int64_t a = src;                                     // the current packet's first byte on this page
    for (int i = seg; i < nseg; i++) {
      const int v = pg[27 + i];
      if (!s.pending) {
        s.pending = true; s.lost = false;
        s.pstart = s.w;
        s.W = ds_packet_header(EntReader{bytes + src, 8ll * v, 0}, modebits);
        a = src;
      }
      src += v;
      if (v == 255) continue;
      or_piece(s, bytes, a, src, lane);
      s.pending = false;
      OrPkt k;
      k.W = s.W; k.bytes = (int)(s.w - s.pstart); k.lost = s.lost;
      k.granulepos = i == lastc ? granule : -1;
      k.e_o_s = (flags & 4) && i == nseg - 1 ? 1 : 0;
      k.packetno = s.packetno++;
      k.page = page;
      if (page == s.skip_page) { s.w = s.pstart; continue; }
      if (visit.packet(k)) return;
    }
    if (s.pending) or_piece(s, bytes, a, src, lane);
    if (flags & 4) return;                               // the walk ends after the EOS page
  }
}

// A page of the serial with a granulepos at or after byte x and before hi: its offset (-1 when none), length,
// granulepos and flags
__device__ __forceinline__ int64_t or_next_gpage(const uint8_t *bytes, int64_t x, int64_t hi, int64_t end,
                                                 uint32_t serial, int lane, const uint32_t *crc_tab,
                                                 const uint32_t *xpw, int &len, int64_t &g, int &flags) {
  while (x < hi) {
    len = ogg_capture(bytes, x, end, lane, crc_tab, xpw);
    if (len < 0) break;
    if (len == 0) continue;
    const uint8_t *pg = bytes + x;
    if (ogg_le32(pg + 14) == serial && pg[4] == 0 && or_granule(pg) != -1) {
      g = or_granule(pg); flags = pg[5];
      return x;
    }
    x += len;
  }
  return -1;
}

// P: the last page of the serial from page A1 on (A1 qualifies) whose granulepos is at most T, by bisection over
// byte offsets while the window is longer than OR_SCAN, then a forward scan.  A page with the BOS flag ends the
// search (a later link); the scan stops after an EOS page.  Returns P's offset, its granulepos and flags.
__device__ __forceinline__ int64_t or_bisect(const uint8_t *bytes, int64_t a1, int64_t a1_end, int64_t g1,
                                             int a1_flags, int64_t end, uint32_t serial, long long T, int lane,
                                             const uint32_t *crc_tab, const uint32_t *xpw, int64_t &gP, int &fP) {
  int64_t best = a1, lo = a1_end, hi = end;
  gP = g1; fP = a1_flags;
  int len, flags;
  int64_t g;
  while (hi - lo > OR_SCAN) {
    const int64_t mid = lo + (hi - lo) / 2;
    const int64_t x = or_next_gpage(bytes, mid, hi, end, serial, lane, crc_tab, xpw, len, g, flags);
    if (x >= 0 && !(flags & 2) && g <= T) {
      best = x; gP = g; fP = flags;
      lo = x + len;
    } else {
      hi = mid;
    }
  }
  for (int64_t x = lo;;) {
    x = or_next_gpage(bytes, x, end, end, serial, lane, crc_tab, xpw, len, g, flags);
    if (x < 0 || (flags & 2) || g > T) break;
    best = x; gP = g; fP = flags;
    if (flags & 4) break;
    x += len;
  }
  return best;
}

__global__ void __launch_bounds__(32 * OR_WARPS)
k_or_plan(OrPlanArgs A) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t xpw[OGG_XPOW];
  ogg_crc_setup(crc_tab, xpw);
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * OR_WARPS + (threadIdx.x >> 5);
  if (r >= A.nreq) return;                                 // warp-uniform
  const vb200_pcm_range q = A.req[r];
  if (lane == 0) {
    A.base[r] = (long long)r * A.out_stride;
    if (r == A.nreq - 1) A.base[r + 1] = (long long)A.nreq * A.out_stride;
  }
  const int hs = A.hs;
  long long got = 0;
  int keep = 0;
  if (q.stream < 0 || q.stream >= A.nrows || q.start < 0 || q.length < 0 || q.length > A.out_stride) {
    got = VB200_EINVAL;
  } else {
    const int64_t beg = A.row_off[q.stream], end = A.row_off[q.stream + 1];
    // 1. the serial, the header packets and G0 from the first audio packet that carries a granulepos
    OrWalk s = or_walk_at(beg, end, false, 0, -1, nullptr, LLONG_MAX);
    int returned = 0;
    DsHead h;
    h.granulepos = -1; h.sample_count = -1; h.sequence = -1; h.W = -1; h.rate = 0;
    long long c1 = 0, g1 = -1;
    int64_t a1 = -1;
    int a1_flags = 0;
    struct {
      int &returned; DsHead &h; long long &c1, &g1; int64_t &a1; const OrPlanArgs &A;
      __device__ bool hole() { return returned < 3; }
      __device__ bool packet(const OrPkt &k) {
        if (returned++ < 3 || k.W < 0) return false;
        vb200_packet_info pi;
        pi.granulepos = k.granulepos; pi.e_o_s = k.e_o_s; pi.packetno = (int32_t)k.packetno;
        long long lo, hi;
        ds_blockin(h, k.W, pi, A.bs, A.hs, lo, hi);
        c1 += hi - lo;
        if (k.granulepos == -1) return false;
        g1 = k.granulepos; a1 = k.page;
        return true;
      }
    } head{returned, h, c1, g1, a1, A};
    or_walk(s, A.bytes, lane, crc_tab, xpw, A.modebits, head);
    const uint32_t serial = s.serial;
    const int64_t a1_end = s.p;
    if (a1 >= 0) a1_flags = A.bytes[a1 + 5];
    if (!s.have_serial) got = VB200_ENOTVORBIS;
    else if (returned < 3) got = VB200_EBADHEADER;
    else if (q.length > 0) {
      const long long G0 = g1 - (c1 << hs);
      const long long t0 = q.start, t1 = q.start > LLONG_MAX - q.length ? LLONG_MAX : q.start + q.length;
      // 2. P, and 3. the anchor: the first accepted packet after P with a granulepos, unless it ends the stream
      int64_t P = -1;
      long long gb1 = 0, pos1 = 0;                         // block 1's granulepos and output position
      bool empty = false;                                  // P is the EOS page: nothing follows it
      auto anchor = [&](int64_t from) -> bool {
        OrWalk w = or_walk_at(from, end, true, serial, from, nullptr, LLONG_MAX);
        struct {
          const int *bs; int lW; long long rel, g; int eos; bool found;
          __device__ bool hole() { return false; }
          __device__ bool packet(const OrPkt &k) {
            if (k.W < 0) return false;
            if (lW >= 0) rel += bs[lW] / 4 + bs[k.W] / 4;
            lW = k.W;
            if (k.granulepos == -1) return false;
            g = k.granulepos; eos = k.e_o_s; found = true;
            return true;
          }
        } v{A.bs, -1, 0, 0, 0, false};
        or_walk(w, A.bytes, lane, crc_tab, xpw, A.modebits, v);
        if (!v.found || v.eos) return false;
        gb1 = v.g - v.rel;
        pos1 = ((v.g - G0) >> hs) - (v.rel >> hs);
        return true;
      };
      if (a1 >= 0) {
        long long T;
        const long long x = (t0 << hs) - A.bs[1] / 2;
        if (t0 > (LLONG_MAX >> 2) || (G0 > 0 && x > LLONG_MAX - G0)) T = LLONG_MAX;
        else if (G0 < 0 && x < LLONG_MIN - G0) T = LLONG_MIN;
        else T = G0 + x;
        if (g1 <= T) {
          int64_t gP;
          int fP;
          P = or_bisect(A.bytes, a1, a1_end, g1, a1_flags, end, serial, T, lane, crc_tab, xpw, gP, fP);
          if (fP & 4) empty = true;
          else if (!anchor(P)) {                           // no anchor, or the e_o_s packet: one page further back
            P = -1;
            if (g1 <= gP - 1) {
              P = or_bisect(A.bytes, a1, a1_end, g1, a1_flags, end, serial, gP - 1, lane, crc_tab, xpw, gP, fP);
              if ((fP & 4) || !anchor(P)) P = -1;
            }
          }
        }
      }
      // 4. the plan: from P with block 1's granulepos fixed by the anchor, else from the row's first audio packet
      if (!empty) {
        const size_t row = (size_t)r * A.nblk;
        const long long res0 = (long long)r * A.res_cap, pk0 = (long long)r * A.pkt_cap;
        uint8_t *dst = A.pkt + pk0;
        const bool seek = P >= 0;
        OrWalk w = seek ? or_walk_at(P, end, true, serial, P, dst, A.pkt_cap)
                        : or_walk_at(beg, end, false, 0, -1, dst, A.pkt_cap);
        h.granulepos = -1; h.sample_count = -1; h.sequence = -1; h.W = -1; h.rate = 0;
        long long pos = seek ? pos1 : 0;
        long long coef = 0;
        int nb = 0, lost_at = INT_MAX, hdr = seek ? 0 : 3;
        int pW = 0, pbytes = 0;
        bool plost = false, first = true, over = false;
        auto put = [&](int k, int W, long long off, int bytes, long long lo, long long hi, long long o) {
          const long long need = (long long)A.ch * (A.bs[W] / 2);
          if (lane == 0 && k < A.nblk && coef + need <= A.res_cap) {
            A.Wseq[row + k] = W;
            A.pkt_off[row + k] = pk0 + off;
            A.pkt_bytes[row + k] = bytes;
            A.coef_off[row + k] = res0 + coef;
            A.pcm_off[row + k] = o;
            A.win[row + k] = make_int2((int)lo, (int)hi);
          }
          coef += need;
        };
        struct {
          OrWalk &w; decltype(put) &put; const OrPlanArgs &A; DsHead &h; int lane;
          long long &pos, &coef, t0, t1, gb1; int &nb, &keep, &lost_at, &hdr, &pW, &pbytes; bool &plost, &first, &over;
          __device__ bool hole() { return false; }
          __device__ bool packet(const OrPkt &k) {
            if (hdr > 0 || k.W < 0) {                      // a header packet, or dropped: nothing changes
              if (hdr > 0) hdr--;
              w.w = w.pstart;
              return false;
            }
            vb200_packet_info pi;
            pi.granulepos = first && gb1 != LLONG_MIN ? gb1 : k.granulepos;
            pi.e_o_s = k.e_o_s; pi.packetno = (int32_t)k.packetno;
            first = false;
            long long lo, hi;
            ds_blockin(h, k.W, pi, A.bs, A.hs, lo, hi);
            const long long ns = hi - lo;
            if (nb == 0) {
              if (ns == 0 || pos + ns <= t0) {             // before the range: the priming candidate, moved to 0
                if (!k.lost && w.pstart > 0)
                  for (long long i0 = 0; i0 < k.bytes; i0 += 32) {
                    __syncwarp();
                    const uint8_t b = i0 + lane < k.bytes ? w.dst[w.pstart + i0 + lane] : 0;
                    __syncwarp();
                    if (i0 + lane < k.bytes) w.dst[i0 + lane] = b;
                  }
                __syncwarp();
                pW = k.W; pbytes = k.bytes; plost = k.lost;
                w.w = k.lost ? 0 : k.bytes;
                pos += ns;
                return false;
              }
              put(0, pW, 0, pbytes, 0, 0, 0);
              if (plost) lost_at = 0;
              nb = 1;
            }
            const long long a = max(pos, t0), b = min(pos + ns, t1);
            if (a < b) put(nb, k.W, w.pstart, k.bytes, lo + (a - pos), lo + (b - pos), a - t0);
            else put(nb, k.W, w.pstart, k.bytes, 0, 0, 0);
            if (k.lost && lost_at == INT_MAX) lost_at = nb;
            nb++;
            if (a < b) {
              keep = nb;
              if (keep > A.nblk || coef > A.res_cap) { over = true; return true; }
            }
            pos += ns;
            return pos >= t1;
          }
        } plan{w, put, A, h, lane, pos, coef, t0, t1, seek ? gb1 : LLONG_MIN, nb, keep, lost_at, hdr, pW, pbytes,
               plost, first, over};
        or_walk(w, A.bytes, lane, crc_tab, xpw, A.modebits, plan);
        if (lost_at < keep) over = true;
        got = over ? VB200_EINVAL : max(0ll, min(pos, t1) - t0);
        if (over) keep = 0;
      }
    }
  }
  if (lane == 0) {
    A.count[r] = keep;
    A.got[r] = (int)got;
  }
}
