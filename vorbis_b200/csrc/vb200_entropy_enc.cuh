// vb200_entropy_enc.cuh — the entropy coding of mapping0_forward (lib/mapping0.c:596-687) on the device, un-managed:
// the packet header, floor1_encode's bits (lib/floor1.c:786-921) and the residue forward of types 1 and 2
// (lib/res0.c:534-648, 725-809), byte-identical to the reference.
//
// One CTA codes one packet in two passes over the same work items.  Pass 1 computes the length in bits of every
// piece of the packet; a block-wide exclusive scan in the reference's stream order turns the lengths into bit
// offsets; pass 2 recomputes every piece and ORs its bits in at its offset with 32-bit atomics (a <= 32-bit
// codeword touches at most two words; bit k of the packet is bit k%8 of byte k/8, oggpack's order).
//   pieces:  [header] [floor of channel 0 .. ch-1] [residue slots of submap 0] [submap 1] ...
//   residue slots of a submap, stage-major: at stage 0 the phrase words of every coded vector come before each
//   group of partitions_per_word partitions; within a group partition-major, then vector.  Later stages have no
//   phrase words.
// A floor is a serial chain of at most 31 partitions, so one thread codes one channel's floor.  A residue item is
// one (partition, coded vector); its residual only feeds the same item at the next stage, so one thread owns an
// item through all stages, working on a private copy of its samples (iwork itself is read-only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"
#include "vb200_floor1.cuh"
#include "vb200_entropy.cuh"

namespace vb200 {

struct EncBook {                       // vb200_enc_codebook; off indexes the flat length / codeword arrays
  int dim, entries, minval, delta, quantvals, off;
};

struct EncEntDev {
  const EncBook *books;
  const unsigned char *len;
  const uint32_t *cw;
  const EntFloor *floor[2];            // [VB200_MAX_SUBMAPS] per block size
  const EntRes *res[2];
  int submaps[2], slots[2];            // slots: pieces of one packet of that size (shared-memory ints)
  int bound[2];                        // vb200_encode_packet_bound
  int ch, modebits;
};

struct EncArgs {
  EncEntDev E;
  const Floor1Dev *f1;                 // [VB200_MAX_SUBMAPS] of this block size
  const unsigned char *chmux;
  const vb200_block_desc *desc;
  const int *posts, *nonzero, *iwork, *classes;
  long long curve_rows;                // rows (block x channel) from one curve to the next: blockIdx.y (curves: k)
  int *work;                           // [gridDim.y][gridDim.x][ch*n] private copies of the residue
  int W, nblocks, n, class_stride;
  long long pkt_stride;
  int *pkt_bits;
  unsigned char *data;
};

constexpr int ENC_THREADS = 128;

__device__ __forceinline__ void enc_put(uint32_t *out, int pos, uint32_t v, int len) {
  if (len <= 0) return;
  if (len < 32) v &= (1u << len) - 1u;
  const int w = pos >> 5, sh = pos & 31;
  atomicOr(out + w, v << sh);
  if (sh + len > 32) atomicOr(out + w + 1, v >> (32 - sh));
}

// vorbis_book_encode (lib/codebook.c:288-292) at pos, which it advances: nothing for an entry out of range
template <bool WR>
__device__ __forceinline__ void enc_word(const EncEntDev &E, int book, long long a, uint32_t *out, int &pos) {
  const EncBook &B = E.books[book];
  if (a < 0 || a >= B.entries) return;
  const int l = E.len[B.off + a];
  if (WR) enc_put(out, pos, E.cw[B.off + a], l);
  pos += l;
}

// local_book_besterror (lib/res0.c:322-384) on a[0..dim): the lattice entry, or where that entry is unused the
// closest used one by a serial walk of the value pattern of vq/; subtracts the chosen vector from a
__device__ int enc_besterror(const EncEntDev &E, const EncBook &B, int *a) {
  const int dim = B.dim, minval = B.minval, del = B.delta, qv = B.quantvals, ze = qv >> 1;
  int p[8], index = 0;
  for (int o = dim - 1; o >= 0; o--) {
    const int v = del != 1 ? (a[o] - minval + (del >> 1)) / del : a[o] - minval;
    const int m = v < ze ? ((ze - v) << 1) - 1 : ((v - ze) << 1);
    index = index * qv + (m < 0 ? 0 : (m >= qv ? qv - 1 : m));
    p[o] = v * del + minval;
  }
  const unsigned char *len = E.len + B.off;
  if (len[index] == 0) {
    int e[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    int best = -1;
    const int maxval = minval + del * (qv - 1);
    for (int i = 0; i < B.entries; i++) {
      if (len[i] > 0) {
        unsigned d = 0;                                 // int arithmetic of the reference, wrapping
        for (int j = 0; j < dim; j++) { const unsigned t = (unsigned)(e[j] - a[j]); d += t * t; }
        if (best == -1 || (int)d < best) {
          for (int j = 0; j < 8; j++) p[j] = e[j];
          best = (int)d;
          index = i;
        }
      }
      int j = 0;
      while (j < 8 && e[j] >= maxval) e[j++] = 0;
      if (e[j] >= 0) e[j] += del;
      e[j] = -e[j];
    }
  }
  for (int i = 0; i < dim; i++) a[i] -= p[i];
  return index;
}

// the wrapped deviation of post i from its prediction (lib/floor1.c:786-827), 0 where floor1_encode writes 0.
// Masked neighbour values never change after they are used, so this is a pure function of the posts the encode
// chain returns.
__device__ __forceinline__ int enc_floor_out(const Floor1Dev &L, const EntFloor &F, const int *p, int i) {
  const int ln = L.lo[i - 2], hn = L.hi[i - 2];
  const int predicted = f1_point(L.postlist[ln], L.postlist[hn], p[ln], p[hn], L.postlist[i], L.prcp[i - 2]);
  if ((p[i] & 0x8000) || (p[i] & 0x7fff) == predicted) return 0;
  const int headroom = F.quant_q - predicted < predicted ? F.quant_q - predicted : predicted;
  const int val = p[i] - predicted;
  if (val < 0) return val < -headroom ? headroom - val - 1 : -1 - (val * 2);
  return val >= headroom ? val + headroom : val << 1;
}

// floor1_encode's bits for one channel (lib/floor1.c:835-921 and :949): returns the length in bits
template <bool WR>
__device__ int enc_floor(const EncEntDev &E, const Floor1Dev &L, const EntFloor &F, const int *p, uint32_t *out,
                         int pos) {
  int any = 0;
  for (int i = 0; i < F.posts; i++) any |= p[i];
  const int start = pos;
  if (WR) enc_put(out, pos, any ? 1u : 0u, 1);
  pos++;
  if (!any) return 1;
  if (WR) { enc_put(out, pos, (uint32_t)p[0], F.qbits); enc_put(out, pos + F.qbits, (uint32_t)p[1], F.qbits); }
  pos += 2 * F.qbits;
  for (int i = 0, j = 2; i < F.partitions; i++) {
    const int cls = F.pclass[i], cdim = F.cdim[cls], csubs = F.csubs[cls], csub = 1 << csubs;
    int bookas[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (csubs) {
      int maxval[8];
      for (int k = 0; k < csub; k++) maxval[k] = F.subbook[cls][k] < 0 ? 1 : E.books[F.subbook[cls][k]].entries;
      int cval = 0, cshift = 0;
      for (int k = 0; k < cdim; k++) {
        const int v = enc_floor_out(L, F, p, j + k);
        for (int l = 0; l < csub; l++)
          if (v < maxval[l]) { bookas[k] = l; break; }
        cval |= bookas[k] << cshift;
        cshift += csubs;
      }
      enc_word<WR>(E, F.cbook[cls], cval, out, pos);
    }
    for (int k = 0; k < cdim; k++) {
      const int book = F.subbook[cls][bookas[k]];
      if (book >= 0) enc_word<WR>(E, book, enc_floor_out(L, F, p, j + k), out, pos);   // none past entries (:901)
    }
    j += cdim;
  }
  return pos - start;
}

// what one submap of one block codes: the bundle's channels and the vectors the residue forward sees
struct EncSub {
  int cib, nvec, items, groups, slot0, nslots;
  unsigned char chan[VB200_MAX_CHANNELS + 1];         // the bundle's channels in order
  unsigned char vec[VB200_MAX_CHANNELS + 1];          // type 1: the used channels (res1_forward's compaction)
};

// One residue item (t = partition * nvec + vector) through all stages: pass 1 stores every stage's length, pass 2
// writes at the scanned offsets.  Slot of the item at stage 0: after the phrase words of its own and all earlier
// partition groups; at stage s > 0: after stage 0 and s-1 full stages.
template <bool WR>
__device__ void enc_res_item(const EncArgs &A, const EntRes &R, const EncSub &S, int blk, int t, int *slot,
                             uint32_t *out, int *work) {
  const EncEntDev &E = A.E;
  const int i = t / S.nvec, j = t - i * S.nvec;
  const int first = (R.type == 2 ? S.chan[0] : S.vec[j]);
  const int cls = A.classes[((size_t)blk * E.ch + first) * A.class_stride + i];
  const int off = R.begin + i * R.grouping;
  const size_t row0 = (size_t)blk * E.ch;
  int *w = work + (R.type == 2 ? 0 : (size_t)j * A.n) + off;
  for (int k = 0; k < R.grouping; k++) {
    const int x = off + k;
    w[k] = R.type == 2 ? A.iwork[(row0 + S.chan[x % S.cib]) * A.n + x / S.cib] : A.iwork[(row0 + S.vec[j]) * A.n + x];
  }
  for (int s = 0; s < R.stages; s++) {
    const int idx = s == 0 ? S.slot0 + (i / R.ppw + 1) * S.nvec + t : S.slot0 + S.groups * S.nvec + s * S.items + t;
    const int book = R.stagebook[cls][s];
    if (book < 0) { if (!WR) slot[idx] = 0; continue; }
    const EncBook &B = E.books[book];
    int pos = WR ? slot[idx] : 0;
    for (int q = 0; q + B.dim <= R.grouping; q += B.dim)    // _encodepart (lib/res0.c:390-410)
      enc_word<WR>(E, book, enc_besterror(E, B, w + q), out, pos);
    if (!WR) slot[idx] = pos;
  }
}

// stage 0 phrase word of vector j before partition group g (lib/res0.c:587-605)
template <bool WR>
__device__ void enc_res_phrase(const EncArgs &A, const EntRes &R, const EncSub &S, int blk, int g, int j, int *slot,
                               uint32_t *out) {
  const int i = g * R.ppw;
  const int first = (R.type == 2 ? S.chan[0] : S.vec[j]);
  const int *pw = A.classes + ((size_t)blk * A.E.ch + first) * A.class_stride;
  long long val = pw[i];
  for (int k = 1; k < R.ppw; k++) {
    val *= R.partitions;
    if (i + k < R.partvals) val += pw[i + k];
  }
  const int idx = S.slot0 + g * S.nvec * (R.ppw + 1) + j;
  int pos = WR ? slot[idx] : 0;
  enc_word<WR>(A.E, R.groupbook, val, out, pos);        // nothing when val >= entries (:597)
  if (!WR) slot[idx] = pos;
}

__device__ void enc_scan(int *v, int count, int *s_warp, int *total) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int per = (count + ENC_THREADS - 1) / ENC_THREADS, a = tid * per, b = min(count, a + per);
  int sum = 0;
  for (int k = a; k < b; k++) sum += v[k];
  int inc = sum;
  for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += y; }
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  int base = 0;
  for (int k = 0; k < wid; k++) base += s_warp[k];
  if (tid == ENC_THREADS - 1) *total = base + inc;
  int run = base + inc - sum;
  for (int k = a; k < b; k++) { const int x = v[k]; v[k] = run; run += x; }
  __syncthreads();
}

template <bool WR>
__device__ void enc_pass(const EncArgs &A, const EncSub *subs, int blk, const int *posts, int *slot, uint32_t *out,
                         int *work) {
  const EncEntDev &E = A.E;
  const int tid = threadIdx.x;
  if (tid == 0) {                                       // packet type, mode, window flags (lib/mapping0.c:603-610)
    const int hb = 1 + E.modebits + (A.W ? 2 : 0);
    if (WR) {
      const int pos = slot[0];
      enc_put(out, pos, 0u, 1);
      enc_put(out, pos + 1, (uint32_t)A.W, E.modebits);
      if (A.W) { enc_put(out, pos + 1 + E.modebits, (uint32_t)A.desc[blk].lW, 1); enc_put(out, pos + 2 + E.modebits, (uint32_t)A.desc[blk].nW, 1); }
    } else slot[0] = hb;
  }
  for (int c = tid; c < E.ch; c += ENC_THREADS) {
    const int sm = A.chmux[c];
    const int l = enc_floor<WR>(E, A.f1[sm], E.floor[A.W][sm], posts + (size_t)c * VB200_FLOOR1_STRIDE, out,
                                WR ? slot[1 + c] : 0);
    if (!WR) slot[1 + c] = l;
  }
  for (int sm = 0; sm < E.submaps[A.W]; sm++) {       // the submaps share the CTA's work copy: one at a time
    const EncSub &S = subs[sm];
    const EntRes &R = E.res[A.W][sm];
    if (S.nvec == 0) continue;
    __syncthreads();
    for (int x = tid; x < S.groups * S.nvec; x += ENC_THREADS)
      enc_res_phrase<WR>(A, R, S, blk, x / S.nvec, x % S.nvec, slot, out);
    for (int t = tid; t < S.items; t += ENC_THREADS) enc_res_item<WR>(A, R, S, blk, t, slot, out, work);
  }
}

// CURVES = false: one packet per block of curve blockIdx.y (posts and nonzero rows blockIdx.y * curve_rows on;
// classes and iwork of curve 0).  CURVES = true (bitrate-managed): the VB200_PACKETBLOBS packets of every block, the
// (curve, block) pairs folded into the CTA's grid-stride loop so that work stays [gridDim.x][ch*n]; curve k of block
// b reads posts / nonzero / iwork row k*curve_rows + b*ch and classes row (k*nblocks + b)*ch, and writes packet
// k*nblocks + b (gridDim.y must be 1).
template <bool CURVES>
__device__ __forceinline__ void encode_packets_body(const EncArgs &A) {
  extern __shared__ int s_slot[];
  __shared__ EncSub s_sub[VB200_MAX_SUBMAPS];
  __shared__ int s_warp[ENC_THREADS / 32], s_total;
  const EncEntDev &E = A.E;
  const int tid = threadIdx.x, ch = E.ch;
  const long long row_y = (long long)blockIdx.y * A.curve_rows;
  int *work = A.work + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * ch * A.n;
  EncArgs C;                                            // CURVES: A with iwork and classes moved to the curve
  if constexpr (CURVES) C = A;
  for (int it = blockIdx.x; it < (CURVES ? VB200_PACKETBLOBS : 1) * A.nblocks; it += gridDim.x) {
    const int curve = CURVES ? it / A.nblocks : 0, blk = it - curve * A.nblocks;
    if constexpr (CURVES) {
      C.iwork = A.iwork + (size_t)curve * A.curve_rows * A.n;
      C.classes = A.classes + (size_t)curve * A.nblocks * ch * A.class_stride;
    }
    const EncArgs &P = CURVES ? C : A;
    const size_t row0 = (size_t)(CURVES ? curve * A.curve_rows : row_y) + (size_t)blk * ch;
    const int *posts = A.posts + row0 * VB200_FLOOR1_STRIDE, *nz = A.nonzero + row0;
    const long long pk = CURVES ? it : (long long)blockIdx.y * A.nblocks + blk;
    uint32_t *out = (uint32_t *)(A.data + pk * A.pkt_stride);
    if (tid < E.submaps[A.W]) {                         // the bundles (lib/mapping0.c:660-683, lib/res0.c:725-809)
      EncSub &S = s_sub[tid];
      const EntRes &R = E.res[A.W][tid];
      int cib = 0, used = 0;
      for (int c = 0; c < ch; c++)
        if (A.chmux[c] == tid) {
          S.chan[cib++] = (unsigned char)c;
          if (nz[c]) S.vec[used++] = (unsigned char)c;
        }
      S.cib = cib;
      S.nvec = R.type < 0 || used == 0 ? 0 : (R.type == 2 ? 1 : used);
      const int pv = R.type < 0 ? 0 : (R.end - R.begin) / R.grouping;
      S.items = pv * S.nvec;
      S.groups = R.type < 0 ? 0 : (pv + R.ppw - 1) / R.ppw;
      S.nslots = S.nvec ? S.groups * S.nvec + R.stages * S.items : 0;
    }
    __syncthreads();
    if (tid == 0) {
      int at = 1 + ch;
      for (int sm = 0; sm < E.submaps[A.W]; sm++) { s_sub[sm].slot0 = at; at += s_sub[sm].nslots; }
      s_total = at;
    }
    __syncthreads();
    const int nslots = s_total;
    enc_pass<false>(P, s_sub, blk, posts, s_slot, out, work);
    __syncthreads();
    enc_scan(s_slot, nslots, s_warp, &s_total);
    const int bits = s_total;
    for (int k = tid; k < (bits + 31) >> 5; k += ENC_THREADS) out[k] = 0u;
    __syncthreads();
    enc_pass<true>(P, s_sub, blk, posts, s_slot, out, work);
    if (tid == 0) A.pkt_bits[pk] = bits;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(ENC_THREADS)
k_encode_packets(EncArgs A) {
  encode_packets_body<false>(A);
}

__global__ void __launch_bounds__(ENC_THREADS)
k_encode_packets_curves(EncArgs A) {
  encode_packets_body<true>(A);
}

// host forms: byte offsets of the packed packets (one CTA, an exclusive scan of (bits + 7) / 8) ...
__global__ void __launch_bounds__(1024)
k_packet_offsets(const int *__restrict__ bits, int n, long long *__restrict__ off) {
  __shared__ long long s_warp[32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int per = (n + 1023) / 1024, a = tid * per, b = min(n, a + per);
  long long sum = 0;
  for (int k = a; k < b; k++) sum += (bits[k] + 7) >> 3;
  long long inc = sum;
  for (int d = 1; d < 32; d <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += y; }
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  long long run = inc - sum;
  for (int k = 0; k < wid; k++) run += s_warp[k];
  for (int k = a; k < b; k++) { off[k] = run; run += (bits[k] + 7) >> 3; }
  if (tid == 1023) off[n] = run;
}

// ... and the byte gather of every packet from its strided slot, where it fits below cap
__global__ void __launch_bounds__(256)
k_packet_gather(const unsigned char *__restrict__ src, long long stride, const int *__restrict__ bits,
                const long long *__restrict__ off, int n, long long cap, unsigned char *__restrict__ dst) {
  if (off[n] > cap) return;
  for (int b = blockIdx.x; b < n; b += gridDim.x) {
    const int nb = (bits[b] + 7) >> 3;
    for (int k = threadIdx.x; k < nb; k += blockDim.x) dst[off[b] + k] = src[(long long)b * stride + k];
  }
}

}  // namespace vb200
