// vb200_ogg.cuh — the Ogg page demux of vb200_ogg_demux[_dev] (rules in include/vorbis_b200.h).
//
//   k_ogg_demux   one warp per file walks its pages in file order; every branch depends on values all lanes hold, so
//                 the warp stays converged.  Per candidate page the lanes split the lacing sum (the table is staged in
//                 shared memory for the packet walk) and the CRC: lane i takes a contiguous chunk of the page, runs the
//                 table CRC over it from 0, and multiplies the result by x^(8 * bytes after the chunk) mod P.  The CRC
//                 has initial value 0 and no final xor, so it is linear and the xor of those products is the CRC of
//                 the page.  The per-lane loads are not coalesced, but every lane's first miss goes out at once and
//                 the rest of its chunk hits L1.  Staging the page in 1 KB shared-memory tiles (coalesced loads,
//                 slicing-by-4 tables, one fold per tile) measured slower on an H100 (500 files of the
//                 tools/ogg_demux_bench.py workload: 4.11 ms against 2.28 ms per call), because its tiles wait on
//                 their loads one after another.  A failed capture looks for the next 'O' 32 bytes at a time with a ballot.  An accepted
//                 page of the stream has its kept body copied by all lanes; the packet walk over the lacing values is
//                 done by every lane alike and lane 0 writes the records.
// and the link table of vb200_ogg_links[_dev]: three launches whatever nfiles is, one warp per file in the walks.
//   k_ogg_links_count  walks the file's captured pages as k_ogg_demux does (ogg_capture: capture pattern, the lanes'
//                      lacing sum and CRC split, the ballot resync) and counts the link starts into link_first[f + 1];
//                      k_ds_scan (vb200_decode_streams.cuh) turns the counts into offsets.
//   k_ogg_links_write  once the total fits link_cap, walks again and writes the file's link offsets from
//                      link_first[f] on.  Neither copies a page body.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

constexpr int OGG_WARPS = 4;
constexpr uint32_t OGG_POLY = 0x04c11db7u;
constexpr int OGG_XPOW = 17;            // x^(8 * 2^k) mod P for k < 17 covers every page length (< 65536 bytes)

// a(x) * b(x) mod P(x) over GF(2)
__device__ __forceinline__ uint32_t ogg_mulmod(uint32_t a, uint32_t b) {
  uint32_t r = 0;
  for (int i = 31; i >= 0; i--) {
    r = (r << 1) ^ ((r & 0x80000000u) ? OGG_POLY : 0u);
    if ((b >> i) & 1u) r ^= a;
  }
  return r;
}

__device__ __forceinline__ uint32_t ogg_le32(const uint8_t *p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// the byte table of the CRC and xpw[k] = x^(8 * 2^k) mod P in shared memory, built by the whole block
__device__ __forceinline__ void ogg_crc_setup(uint32_t *crc_tab, uint32_t *xpw) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t r = (uint32_t)i << 24;
    for (int k = 0; k < 8; k++) r = (r << 1) ^ ((r & 0x80000000u) ? OGG_POLY : 0u);
    crc_tab[i] = r;
  }
  if (threadIdx.x == 0) {
    xpw[0] = 0x100u;                                      // x^8
    for (int k = 1; k < OGG_XPOW; k++) xpw[k] = ogg_mulmod(xpw[k - 1], xpw[k - 1]);
  }
  __syncthreads();
}

// the CRC of pg[0 .. len) with bytes 22..25 taken as zero, by one converged warp: lane i runs the table over its
// chunk from 0 and shifts the result by x^(8 * bytes after the chunk); every lane returns the xor of the chunks
__device__ __forceinline__ uint32_t ogg_page_crc(const uint8_t *pg, int len, int lane, const uint32_t *crc_tab,
                                                 const uint32_t *xpw) {
  const int chunk = (len + 31) / 32;
  const int a = min(lane * chunk, len), e = min(a + chunk, len);
  uint32_t c = 0;
  for (int i = a; i < e; i++) {
    const uint32_t v = (i >= 22 && i < 26) ? 0u : pg[i];
    c = (c << 8) ^ crc_tab[(c >> 24) ^ v];
  }
  if (c) {
    uint32_t m = 1u;
    for (int k = 0, n = len - e; n; k++, n >>= 1)
      if (n & 1) m = ogg_mulmod(m, xpw[k]);
    c = ogg_mulmod(c, m);
  }
  for (int o = 16; o; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
  return c;
}

// ogg_sync_pageseek at byte p of a file that ends at `end`, by one converged warp, as k_ogg_demux captures.  Returns
// the captured page's length, 0 when the capture failed (p then moved to the next 'O' after it, or to end), or -1 when
// fewer than 27 bytes are left or the page is cut short by the end of the file.  k_ogg_demux keeps this step and its
// packet walk written out in its loop, with one copy of each page body: the demux on this function and k_or_plan's
// walk (or_walk, which copies packet by packet so that its visitors can move and drop packets) measured slower on an
// H100 once many files share the GPU (INTEGRATION §2g).  The tests hold this step to oracle/ogg_links.py and the
// demux's copy to oracle/ogg.py, which capture pages alike.
__device__ __forceinline__ int ogg_capture(const uint8_t *bytes, int64_t &p, int64_t end, int lane,
                                           const uint32_t *crc_tab, const uint32_t *xpw) {
  if (end - p < 27) return -1;
  const uint8_t *pg = bytes + p;
  bool ok = pg[0] == 'O' && pg[1] == 'g' && pg[2] == 'g' && pg[3] == 'S';
  int len = 0;
  if (ok) {
    const int nseg = pg[26];
    if (end - p < 27 + nseg) return -1;
    int body = 0;
    for (int i = lane; i < nseg; i += 32) body += pg[27 + i];
    for (int o = 16; o; o >>= 1) body += __shfl_xor_sync(0xffffffffu, body, o);
    len = 27 + nseg + body;
    if (end - p < len) return -1;
    ok = ogg_page_crc(pg, len, lane, crc_tab, xpw) == ogg_le32(pg + 22);
  }
  if (ok) return len;
  int64_t q = end;                                        // lose sync: resume at the next 'O'
  for (int64_t b = p + 1; b < end; b += 32) {
    const int64_t i = b + lane;
    const unsigned m = __ballot_sync(0xffffffffu, i < end && bytes[i] == 'O');
    if (m) { q = b + __ffs(m) - 1; break; }
  }
  p = q;
  return 0;
}

__global__ void __launch_bounds__(32 * OGG_WARPS)
k_ogg_demux(int nfiles, const uint8_t *__restrict__ bytes, const int64_t *__restrict__ file_off, int max_packets,
            vb200_packet_info *__restrict__ info, int32_t *__restrict__ npkt_out, uint8_t *__restrict__ data,
            vb200_ogg_stream *__restrict__ streams) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t xpw[OGG_XPOW];
  __shared__ uint8_t lace_all[OGG_WARPS][256];
  ogg_crc_setup(crc_tab, xpw);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int f = blockIdx.x * OGG_WARPS + wib;
  if (f >= nfiles) return;
  uint8_t *lace = lace_all[wib];
  const int64_t beg = file_off[f], end = file_off[f + 1];
  vb200_packet_info *inf = info + (size_t)f * max_packets;

  int status = 0, pages = 0, dropped = 0, holes = 0, foreign = 0, chained = 0;
  bool have_serial = false, done = false, have_seq = false, pending = false, stop = false;
  uint32_t serial = 0, next_seq = 0;
  int64_t hoff[3] = {-1, -1, -1};
  int32_t hbytes[3] = {-1, -1, -1};
  int64_t w = beg, pstart = beg;     // next free byte of data; first byte of the packet being assembled
  int64_t packetno = 0;
  int returned = 0, np = 0;          // packets returned (headers included); audio packets in the table
  int64_t p = beg;
  while (!stop) {
    __syncwarp();                                         // the previous page's walk is done with `lace`
    if (end - p < 27) break;
    const uint8_t *pg = bytes + p;
    bool ok = pg[0] == 'O' && pg[1] == 'g' && pg[2] == 'g' && pg[3] == 'S';
    int nseg = 0, body = 0;
    if (ok) {
      nseg = pg[26];
      if (end - p < 27 + nseg) break;
      for (int i = lane; i < nseg; i += 32) {
        const uint8_t v = pg[27 + i];
        lace[i] = v;
        body += v;
      }
      for (int o = 16; o; o >>= 1) body += __shfl_xor_sync(0xffffffffu, body, o);
      if (end - p < 27 + nseg + body) break;
      ok = ogg_page_crc(pg, 27 + nseg + body, lane, crc_tab, xpw) == ogg_le32(pg + 22);
    }
    if (!ok) {                                            // lose sync: resume at the next 'O'
      dropped++;
      int64_t q = end;
      for (int64_t b = p + 1; b < end; b += 32) {
        const int64_t i = b + lane;
        const unsigned m = __ballot_sync(0xffffffffu, i < end && bytes[i] == 'O');
        if (m) { q = b + __ffs(m) - 1; break; }
      }
      p = q;
      continue;
    }
    __syncwarp();                                         // `lace` is complete
    const int64_t body0 = p + 27 + nseg;
    const int ver = pg[4], flags = pg[5];
    const uint32_t ser = ogg_le32(pg + 14), seq = ogg_le32(pg + 18);
    const int64_t granule = (int64_t)((uint64_t)ogg_le32(pg + 6) | ((uint64_t)ogg_le32(pg + 10) << 32));
    p = body0 + body;
    if (done) { chained = (flags & 2) ? 1 : 0; break; }
    if (!have_serial) {
      bool vorbis = false;
      if ((flags & 2) && ver == 0) {
        int first = 0;
        for (int i = 0; i < nseg; i++) { first += lace[i]; if (lace[i] < 255) break; }
        const uint8_t *b = bytes + body0;
        vorbis = first >= 7 && b[0] == 1 && b[1] == 'v' && b[2] == 'o' && b[3] == 'r' && b[4] == 'b' && b[5] == 'i' &&
                 b[6] == 's';
      }
      if (!vorbis) { foreign++; continue; }
      have_serial = true;
      serial = ser;
    } else if (ser != serial || ver != 0) {
      foreign++;
      continue;
    }
    // ogg_stream_pagein
    pages++;
    if (have_seq && seq != next_seq) {
      if (pending) { w = pstart; pending = false; }       // the partial packet is dropped
      holes++;
      packetno++;                                         // the hole: packetout returns no packet for it
      if (returned < 3) break;
    }
    have_seq = true;
    next_seq = seq + 1;
    int seg = 0;
    int64_t src = body0;
    if ((flags & 1) && !pending)                          // continued page, nothing to continue: skip the fragment
      while (seg < nseg) {
        const int v = lace[seg++];
        src += v;
        if (v < 255) break;
      }
    const int64_t ncopy = body0 + body - src;
    for (int64_t i = lane; i < ncopy; i += 32) data[w + i] = bytes[src + i];
    int lastc = -1;                                       // the last segment that ends a packet on this page
    for (int i = seg; i < nseg; i++)
      if (lace[i] < 255) lastc = i;
    if (!pending) pstart = w;
    int64_t q = w;
    for (int i = seg; i < nseg && !stop; i++) {
      q += lace[i];
      if (lace[i] == 255) continue;
      // ogg_stream_packetout: packet [pstart, q)
      const int32_t n = (int32_t)(q - pstart);
      if (returned < 3) {
        hoff[returned] = pstart;
        hbytes[returned] = n;
      } else if (np == max_packets) {
        status = VB200_EINVAL;
        stop = true;
        break;
      } else {
        if (lane == 0) {
          vb200_packet_info r;
          r.offset = pstart;
          r.granulepos = i == lastc ? granule : -1;
          r.bytes = n;
          r.e_o_s = (flags & 4) && i == nseg - 1 ? 1 : 0;
          r.packetno = (int32_t)packetno;
          r.choice = 0;
          inf[np] = r;
        }
        np++;
      }
      returned++;
      packetno++;
      pstart = q;
    }
    w = q;
    if (nseg > seg) pending = lace[nseg - 1] == 255;
    if (flags & 4) done = true;                           // the EOS page: look at the next page for a chain
  }
  if (!have_serial) status = VB200_ENOTVORBIS;
  else if (returned < 3) status = VB200_EBADHEADER;
  if (lane == 0) {
    vb200_ogg_stream o;
    o.status = status; o.serial = serial; o.pages = pages; o.dropped = dropped; o.holes = holes; o.foreign = foreign;
    o.chained = chained; o.pad = 0; o.pad2 = 0;
    for (int k = 0; k < 3; k++) { o.hdr_offset[k] = hoff[k]; o.hdr_bytes[k] = hbytes[k]; }
    streams[f] = o;
    npkt_out[f] = status == VB200_EBADHEADER ? 0 : np;
  }
}

// The link starts of one file after its first byte, by one converged warp: at(offset) for every captured page with
// the BOS flag that follows a captured page without it (rule in include/vorbis_b200.h, vb200_ogg_links).
template <class At>
__device__ __forceinline__ void ogg_links_walk(const uint8_t *bytes, int64_t beg, int64_t end, int lane,
                                               const uint32_t *crc_tab, const uint32_t *xpw, At &at) {
  bool after_data = false;                                // the last captured page has no BOS flag
  int64_t p = beg;
  for (;;) {
    const int len = ogg_capture(bytes, p, end, lane, crc_tab, xpw);
    if (len < 0) break;
    if (len == 0) continue;
    const bool bos = (bytes[p + 5] & 2) != 0;
    if (bos && after_data) at(p);
    after_data = !bos;
    p += len;
  }
}

// link_first[f + 1] = file f's link count; k_ds_scan then turns the counts into offsets
__global__ void __launch_bounds__(32 * OGG_WARPS)
k_ogg_links_count(int nfiles, const uint8_t *__restrict__ bytes, const int64_t *__restrict__ file_off,
                  long long *__restrict__ link_first) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t xpw[OGG_XPOW];
  ogg_crc_setup(crc_tab, xpw);
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * OGG_WARPS + (threadIdx.x >> 5);
  if (f >= nfiles) return;
  long long n = 1;
  auto at = [&](int64_t) { n++; };
  ogg_links_walk(bytes, file_off[f], file_off[f + 1], lane, crc_tab, xpw, at);
  if (lane == 0) link_first[f + 1] = n;
}

// link_off[link_first[f] ..] = file_off[f], then the offsets of the file's later links' first pages; the last file's
// warp also writes link_off[total] = file_off[nfiles].  Nothing is written when total > link_cap.
__global__ void __launch_bounds__(32 * OGG_WARPS)
k_ogg_links_write(int nfiles, const uint8_t *__restrict__ bytes, const int64_t *__restrict__ file_off,
                  const long long *__restrict__ link_first, int64_t *__restrict__ link_off, long long link_cap) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t xpw[OGG_XPOW];
  if (link_first[nfiles] > link_cap) return;              // the sizing call (or too small a table): nothing written
  ogg_crc_setup(crc_tab, xpw);
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * OGG_WARPS + (threadIdx.x >> 5);
  if (f >= nfiles) return;
  long long row = link_first[f];
  if (lane == 0) {
    link_off[row] = file_off[f];
    if (f == nfiles - 1) link_off[link_first[nfiles]] = file_off[nfiles];
  }
  auto at = [&](int64_t p) {
    row++;
    if (lane == 0) link_off[row] = p;
  };
  ogg_links_walk(bytes, file_off[f], file_off[f + 1], lane, crc_tab, xpw, at);
}
