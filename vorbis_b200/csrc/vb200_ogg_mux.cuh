// vb200_ogg_mux.cuh — the Ogg page mux of vb200_ogg_mux[_dev] (rules in include/vorbis_b200.h).
//
// The pages are those libogg 1.3.x makes (framing.c: ogg_stream_packetin, ogg_stream_flush_i, ogg_stream_pageout,
// ogg_stream_flush) when driven as examples/encoder_example.c drives it; the rules are restated, not run against
// libogg, and where they differ from libogg, libogg is right.  A page's extent is a pure function of the packets from
// its first segment on: it ends at the first packet boundary where more than 4096 body bytes hold at least four
// packet ends (the boundary needs a packet after it), at 255 lacing values, or at the end of an e_o_s packet.  So a
// walk over the packets in order decides every page once, and whatever it leaves open at the end of a call is the
// caller's kept tail, passed again in the next call.
//
//   ogg_mux_walk     that walk, one warp per stream, every lane alike: the lanes load the next 32 packet rows at
//                    once and take them by shuffle; a packet of s segments costs O(1 + s/255).  Each decided page
//                    goes to a sink.
//   k_ogg_mux_count  validates the stream's rows and carry (status) and walks with a sink that sums the page bytes
//                    into out_off[s + 1]; k_ds_scan turns those into offsets.
//   k_ogg_mux_write  walks again with a sink that writes each page: the lanes write the header and the lacing table,
//                    gather the body from the packets' byte ranges, then take the CRC by the demux's chunk-and-shift
//                    method (ogg_page_crc) over the page just written, and lane 0 stores it.  Then the new carry.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"
#include "vb200_ogg.cuh"

constexpr int OGG_MUX_WARPS = 4;
constexpr int OGG_MUX_FRESH = 0, OGG_MUX_WRITING = 1, OGG_MUX_DONE = 2;   // vb200_ogg_mux_carry.state

struct OggMuxArgs {
  int nstreams;
  const uint8_t *data;
  long long data_bytes;
  const vb200_packet_info *hdr;     // [nstreams][3] or null
  int max_packets;
  const int32_t *npkt;              // [nstreams]
  const vb200_packet_info *info;    // [nstreams][max_packets]
  vb200_ogg_mux_carry *carry;       // [nstreams]
  uint8_t *out;
  long long out_cap;
  long long *out_off;               // [nstreams + 1]
  int32_t *status;                  // [nstreams]
};

// one decided page: its first segment is segment s0 of packet u0 (0..2 the header packets of a fresh carry, u >= 3
// audio row u - 3 of this call)
struct OggMuxPage {
  int u0, s0, vals, body, flags;
  long long granule;
};

__device__ __forceinline__ const vb200_packet_info *ogg_mux_row(const OggMuxArgs &A, int s, int u) {
  return u < 3 ? A.hdr + (size_t)s * 3 + u : A.info + (size_t)s * A.max_packets + (u - 3);
}

// The walk of one valid stream from its carry over this call's packets; sink.page(page, sequence number) for each
// page decided, in order.  Writes the carry the call leaves to *next.
template <class Sink>
__device__ void ogg_mux_walk(const OggMuxArgs &A, int s, const vb200_ogg_mux_carry &c, int lane, Sink &sink,
                             vb200_ogg_mux_carry *next) {
  const int n = A.npkt[s];
  const bool fresh = c.state == OGG_MUX_FRESH;
  const int u_end = 3 + n;
  const bool eos = n > 0 && A.info[(size_t)s * A.max_packets + n - 1].e_o_s != 0;
  uint32_t seq = c.pageno;
  int vals = 0, acc = 0, done = 0, u0 = 0, s0 = 0;
  long long granule = -1;
  bool initial = fresh;                                   // !b_o_s: the next page is the BOS page
  auto emit = [&](bool last) {
    OggMuxPage p;
    p.u0 = u0; p.s0 = s0; p.vals = vals; p.body = acc;
    p.flags = (s0 > 0 ? 1 : 0) | (initial ? 2 : 0) | (last ? 4 : 0);
    p.granule = initial ? 0 : granule;
    sink.page(p, seq);
    seq++;
    vals = 0; acc = 0; done = 0; granule = -1; initial = false;
  };
  if (c.state != OGG_MUX_DONE) {
    for (int ub = fresh ? 0 : 3; ub < u_end; ub += 32) {
      int mb = 0;
      long long mg = 0;
      if (ub + lane < u_end) {
        const vb200_packet_info *r = ogg_mux_row(A, s, ub + lane);
        mb = r->bytes;
        mg = r->granulepos;
      }
      const int m = min(32, u_end - ub);
      for (int j = 0; j < m; j++) {
        const int u = ub + j;
        const int b = __shfl_sync(0xffffffffu, mb, j);
        const long long g = __shfl_sync(0xffffffffu, mg, j);
        const int L = b / 255 + 1;                        // lacing values: b/255 of 255, then b % 255
        int sg = (u == 3 && !fresh) ? c.kept_segs : 0;
        if (vals > 0 && acc > 4096 && done >= 4) emit(false);   // the boundary before this packet ends the page
        while (sg < L) {
          if (vals == 0) { u0 = u; s0 = sg; }
          const int k = min(L - sg, 255 - vals);
          acc += (int)(min((long long)(sg + k) * 255, (long long)b) - (long long)sg * 255);
          vals += k;
          sg += k;
          if (sg == L) { done++; granule = g; }
          if (vals == 255 || initial) emit(eos && u == u_end - 1 && sg == L);
        }
        if (u == 2 && vals) emit(false);                 // ogg_stream_flush after the headers
      }
    }
    if (eos && vals) emit(true);
  }
  vb200_ogg_mux_carry o = c;
  o.pageno = seq;
  if (c.state == OGG_MUX_DONE || eos) {
    o.state = OGG_MUX_DONE; o.kept = 0; o.kept_segs = 0;
  } else {
    o.state = OGG_MUX_WRITING;
    o.kept = vals ? u_end - u0 : 0;
    o.kept_segs = vals ? s0 : 0;
  }
  *next = o;
}

struct OggMuxCount {
  long long bytes = 0;
  __device__ void page(const OggMuxPage &p, uint32_t) { bytes += 27 + p.vals + p.body; }
};

__global__ void __launch_bounds__(32 * OGG_MUX_WARPS)
k_ogg_mux_count(OggMuxArgs A) {
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * OGG_MUX_WARPS + (threadIdx.x >> 5);
  if (s >= A.nstreams) return;
  const vb200_ogg_mux_carry c = A.carry[s];
  const int n = A.npkt[s];
  bool bad = c.state < OGG_MUX_FRESH || c.state > OGG_MUX_DONE || c.kept < 0 || c.kept_segs < 0 || n < c.kept ||
             n > A.max_packets || (c.state == OGG_MUX_DONE && n > 0) ||
             (c.state == OGG_MUX_FRESH && (!A.hdr || c.kept != 0)) || (c.kept_segs > 0 && c.kept == 0);
  if (!bad) {
    const vb200_packet_info *inf = A.info + (size_t)s * A.max_packets;
    for (int k = lane; k < n; k += 32) {
      const vb200_packet_info r = inf[k];
      bad |= r.bytes < 0 || r.offset < 0 || r.offset > A.data_bytes - r.bytes || (r.e_o_s && k != n - 1);
      if (k == 0 && c.kept_segs > r.bytes / 255) bad = true;   // the kept packet has fewer segments than are paged
    }
    if (c.state == OGG_MUX_FRESH && lane < 3) {
      const vb200_packet_info r = A.hdr[(size_t)s * 3 + lane];
      bad |= r.bytes < 0 || r.offset < 0 || r.offset > A.data_bytes - r.bytes;
    }
  }
  bad = __any_sync(0xffffffffu, bad);
  OggMuxCount cnt;
  vb200_ogg_mux_carry next;
  if (!bad) ogg_mux_walk(A, s, c, lane, cnt, &next);
  if (lane == 0) {
    A.status[s] = bad ? VB200_EINVAL : 0;
    A.out_off[s + 1] = bad ? 0 : cnt.bytes;
  }
}

struct OggMuxWrite {
  const OggMuxArgs &A;
  int s, lane;
  uint32_t serial;
  long long pos;
  const uint32_t *crc_tab, *xpw;
  __device__ void page(const OggMuxPage &p, uint32_t seq) {
    uint8_t *pg = A.out + pos;
    if (lane < 27) {
      uint32_t v;
      if (lane < 4) v = lane == 0 ? 'O' : lane == 3 ? 'S' : 'g';
      else if (lane == 4) v = 0;                          // version
      else if (lane == 5) v = p.flags;
      else if (lane < 14) v = (uint32_t)((unsigned long long)p.granule >> (8 * (lane - 6)));
      else if (lane < 18) v = serial >> (8 * (lane - 14));
      else if (lane < 22) v = seq >> (8 * (lane - 18));
      else if (lane < 26) v = 0;                          // the CRC, stored below
      else v = p.vals;
      pg[lane] = (uint8_t)v;
    }
    uint8_t *lace = pg + 27, *body = pg + 27 + p.vals;
    int u = p.u0, sg = p.s0, left = p.vals, li = 0, bo = 0;
    while (left > 0) {                                    // the packets on the page, in order
      const vb200_packet_info *r = ogg_mux_row(A, s, u);
      const int b = r->bytes;
      const long long off = r->offset;
      const int L = b / 255 + 1, k = min(L - sg, left);
      for (int i = lane; i < k; i += 32) lace[li + i] = sg + i < L - 1 ? 255 : (uint8_t)(b % 255);
      const long long lo = (long long)sg * 255;
      const int nb = (int)(min((long long)(sg + k) * 255, (long long)b) - lo);
      const uint8_t *src = A.data + off + lo;
      for (int i = lane; i < nb; i += 32) body[bo + i] = src[i];
      li += k; bo += nb; left -= k; u++; sg = 0;
    }
    __syncwarp();                                         // the page is written: its CRC reads it back
    const uint32_t crc = ogg_page_crc(pg, 27 + p.vals + p.body, lane, crc_tab, xpw);
    if (lane < 4) pg[22 + lane] = (uint8_t)(crc >> (8 * lane));
    pos += 27 + p.vals + p.body;
  }
};

__global__ void __launch_bounds__(32 * OGG_MUX_WARPS)
k_ogg_mux_write(OggMuxArgs A) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t xpw[OGG_XPOW];
  if (A.out_off[A.nstreams] > A.out_cap) return;          // the sizing call (or too small a buffer): nothing written
  ogg_crc_setup(crc_tab, xpw);
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * OGG_MUX_WARPS + (threadIdx.x >> 5);
  if (s >= A.nstreams || A.status[s]) return;
  const vb200_ogg_mux_carry c = A.carry[s];
  OggMuxWrite w{A, s, lane, c.serial, A.out_off[s], crc_tab, xpw};
  vb200_ogg_mux_carry next;
  ogg_mux_walk(A, s, c, lane, w, &next);
  __syncwarp();
  if (lane == 0) A.carry[s] = next;
}
