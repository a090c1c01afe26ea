// vb200_streams.cuh — whole streams: from envelope marks to the per-size block batches (SURVEY §8 a12, a15).
//
//  k_env_marks     lib/envelope.c:254-264   mark[] of a stream from the per-step trigger bits
//  k_plan_blocks   lib/block.c:534-689      what vorbis_analysis_blockout decides per block, with the cursor /
//                                           curmark walk of _ve_envelope_search (lib/envelope.c:269-327) and
//                                           _ve_envelope_mark (:329-356); one thread per stream (a few integer
//                                           operations per 64-sample step; the streams are the parallelism)
//  k_plan_offsets / k_plan_fill              give every block its slot in the batch of its size, in (stream, k)
//                                           order, and build that batch's gather table and descriptors
//  k_ampmax_plan   lib/block.c:626-628, lib/psy.c:837-848   the decay chain along a stream ACROSS block sizes
//  k_env_marks_carry / k_plan_blocks_carry / k_ampmax_plan_carry   the same bodies (CARRY = true) starting from and
//                  returning to a stream's PlanCarry: vb200_encode_streams_packets[_managed]_resume
//
// The planner works in the reference's own relative coordinates: after every block everything is re-based by
// movementW (lib/block.c:654-686, lib/envelope.c:358-379); `shift` is the sum of those moves, so relative
// sample r is timeline sample r + shift.  movementW is a multiple of the 64-sample search step as long as
// blocksizes[0]/4 is (checked on the host).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

namespace vb200 {

constexpr int PLAN_STEP = 64;   // envelope_lookup.searchstep
constexpr int PLAN_VE_WIN = 4;  // VE_WIN, lib/envelope.h:24

// What a stream carries from one call to the next (vb200_encode_streams_packets[_managed]_resume): the public head
// (vb200_encode_carry), then the planner's state in the coordinates of the next call's buffer, whose sample 0 is
// timeline sample `base` (the reference's v->pcm[][0] after the last vorbis_analysis_blockout).
struct PlanCarry {
  long long base, granulepos;        // vb200_encode_carry
  int packetno, done;
  long long kept;                    // v->pcm_current: samples the next buffer starts with again
  long long centerW, cursor, curmark, current;   // v->centerW, ve->cursor, ve->curmark, ve->current
  long long base_in;                 // this call's base and packetno, for the gather
  int packetno_in, W, lW;
  float gmax, prev;                  // g->ampmax and the previous block's vbi->ampmax (lib/block.c:626-628)
  int ch, bs0, bs1, mark_cap;        // the setup the carry belongs to
  int br_ready;                      // the bitrate state was initialised from a managed vb200_bitrate_setup
};

// The device copy of the carries of one call, structure of arrays: marks [n][cap] is the window of ve->mark that
// _ve_envelope_shift keeps (current/64 + VE_POST entries); first / count the envelope steps analysed this call.
struct CarryDev {
  PlanCarry *pc;
  uint8_t *marks;
  int cap;
  int32_t *env;                      // [n][VB200_VE_STATE_WORDS(ch)]
  vb200_bitrate_state *br;           // [n]
  const int32_t *first, *count;
  int32_t *overflow;                 // set when a stream's window does not fit cap
};

// mark[i] = 1 iff step i triggered (pre or post echo), or step i-1 saw a pre-echo, or step i+1 a post-echo:
// the closed form of the replay at lib/envelope.c:254-264 (a step only ever clears a mark two ahead of
// itself, before anything could have set it).  Steps at or past the stream's own `last` were never analysed.
// CARRY: steps [first, first + count) were analysed this call (ret relative to first); the carried window holds
// the marks of the steps before, and step first - 1 set the last ones it could.
template <bool CARRY>
__device__ __forceinline__ void env_marks_body(int nstreams, int nsteps_max, const uint8_t *__restrict__ ret,
                                               const int64_t *__restrict__ pcm_len, int32_t *__restrict__ mark,
                                               long long mark_stride, const CarryDev &K) {
  const long long total = (long long)nstreams * mark_stride;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int st = (int)(t / mark_stride), i = (int)(t - (long long)st * mark_stride);
    int m = 0;
    if (CARRY) {
      const int f = K.first[st], last = f + K.count[st];
      const uint8_t *r = ret + (size_t)st * nsteps_max - f;
      if (i >= f && i < last && (r[i] & 3)) m = 1;
      if (i - 1 >= f && i - 1 < last && (r[i - 1] & 1)) m = 1;
      if (i + 1 >= f && i + 1 < last && (r[i + 1] & 2)) m = 1;
      if (i < f + 2 && i < K.cap && !K.pc[st].done && K.marks[(size_t)st * K.cap + i]) m = 1;
    } else {
      long long last = pcm_len[st] / PLAN_STEP - PLAN_VE_WIN;
      if (last > nsteps_max) last = nsteps_max;
      const uint8_t *r = ret + (size_t)st * nsteps_max;
      if (i < last && (r[i] & 3)) m = 1;
      if (i >= 1 && i - 1 < last && (r[i - 1] & 1)) m = 1;
      if (i + 1 < last && (r[i + 1] & 2)) m = 1;
    }
    mark[t] = m;
  }
}

__global__ void __launch_bounds__(256)
k_env_marks(int nstreams, int nsteps_max, const uint8_t *__restrict__ ret, const int64_t *__restrict__ pcm_len,
            int32_t *__restrict__ mark, long long mark_stride) {
  env_marks_body<false>(nstreams, nsteps_max, ret, pcm_len, mark, mark_stride, CarryDev{});
}

__global__ void __launch_bounds__(256)
k_env_marks_carry(int nstreams, int nsteps_max, const uint8_t *__restrict__ ret, int32_t *__restrict__ mark,
                  long long mark_stride, CarryDev K) {
  env_marks_body<true>(nstreams, nsteps_max, ret, nullptr, mark, mark_stride, K);
}

// CARRY: the stream starts from its carried state (nothing for a done stream) instead of a fresh one, eof is in
// timeline samples, and the state where planning stopped goes back to the carry with the mark window it needs.
template <bool CARRY>
__device__ __forceinline__ void plan_blocks_body(int nstreams, int bs0, int bs1, const int32_t *__restrict__ mark,
                                                 long long mark_stride, int nsteps_max,
                                                 const int64_t *__restrict__ pcm_len, const int64_t *__restrict__ eof,
                                                 int max_blocks, vb200_stream_block *__restrict__ plan,
                                                 int32_t *__restrict__ nblocks, int32_t *__restrict__ counts,
                                                 const CarryDev &K) {
  const int st = blockIdx.x * blockDim.x + threadIdx.x;
  if (st >= nstreams) return;
  const int32_t *mk = mark + (size_t)st * mark_stride;
  vb200_stream_block *out = plan + (size_t)st * max_blocks;
  const long long bs[2] = {bs0, bs1};
  const long long step = PLAN_STEP;
  int lW = 0, W = 0, nW = 0;
  long long centerW = bs1 / 2, cursor = bs1 / 2, curmark = 0, shift = 0;     // _vds_shared_init; _ve_envelope_init (calloc)
  long long pcm_current = pcm_len[st];
  long long eofflag = eof ? eof[st] : 0;
  long long last = pcm_current / step - PLAN_VE_WIN;
  if (last > nsteps_max) last = nsteps_max;
  if (last < 0) last = 0;
  long long current = last * step;                                           // ve->current
  if (CARRY) {
    const PlanCarry &p = K.pc[st];
    if (p.done) { nblocks[st] = 0; counts[2 * st] = counts[2 * st + 1] = 0; return; }
    W = p.W; lW = p.lW; centerW = p.centerW; cursor = p.cursor; curmark = p.curmark;
    if (current < p.current) current = p.current;
    if (eofflag) eofflag -= p.base;                                          // > 0: checked on the host
  }
  int nb = 0, cnt[2] = {0, 0};
  while (nb < max_blocks) {
    if (eofflag == -1) break;                                                // lib/block.c:547
    long long bp = -1;
    {                                                                        // lib/envelope.c:269-327
      const long long testW = centerW + bs[W] / 4 + bs1 / 2 + bs0 / 4;
      long long j = cursor;
      while (j < current - step) {
        if (j >= testW) { bp = 1; break; }
        cursor = j;
        if (mk[(j + shift) / step]) {
          if (j > centerW) {
            curmark = j;
            bp = j >= testW ? 1 : 0;
            break;
          }
        }
        j += step;
      }
    }
    if (bp == -1) {
      if (eofflag == 0) break;                                               // not enough data to decide yet
      nW = 0;
    } else {
      nW = bs0 == bs1 ? 0 : (int)bp;
    }
    const long long centerNext = centerW + bs[W] / 4 + bs[nW] / 4;
    if (pcm_current < centerNext + bs[nW] / 2) break;                        // lib/block.c:581-590
    int blocktype;
    if (W) {
      blocktype = (!lW || !nW) ? 0 : 1;                                      // BLOCKTYPE_TRANSITION : BLOCKTYPE_LONG
    } else {                                                                 // _ve_envelope_mark
      const long long beginW = centerW - bs0 / 4 - bs0 / 4, endW = centerW + bs0 / 4 + bs0 / 4;
      bool hit = curmark >= beginW && curmark < endW;
      for (long long i = beginW / step; !hit && i < endW / step; i++) hit = mk[i + shift / step] != 0;
      blocktype = hit ? 0 : 1;                                               // BLOCKTYPE_IMPULSE : BLOCKTYPE_PADDING
    }
    vb200_stream_block b;
    b.pos = (int32_t)(shift + centerW - bs[W] / 2);
    b.slot = cnt[W]++;                                                       // within the stream for now
    b.W = W; b.lW = lW; b.nW = nW; b.blocktype = blocktype;
    out[nb++] = b;
    if (eofflag && centerW >= eofflag) {                                     // the last block, lib/block.c:645-651
      if (CARRY) eofflag = -1;
      break;
    }
    const long long movementW = centerNext - bs1 / 2;
    if (movementW > 0) {                                                     // lib/block.c:654-686
      current -= movementW;
      if (curmark >= 0) curmark -= movementW;
      cursor -= movementW;
      pcm_current -= movementW;
      shift += movementW;
      lW = W; W = nW; centerW = bs1 / 2;
      if (eofflag) {
        eofflag -= movementW;
        if (eofflag <= 0) eofflag = -1;
      }
    }
  }
  nblocks[st] = nb;
  counts[2 * st] = cnt[0];
  counts[2 * st + 1] = cnt[1];
  if (CARRY) {
    PlanCarry &p = K.pc[st];
    p.base_in = p.base; p.packetno_in = p.packetno;
    p.base += shift; p.packetno += nb; p.done = eofflag == -1;
    p.kept = pcm_current; p.centerW = centerW; p.cursor = cursor; p.curmark = curmark; p.current = current;
    p.W = W; p.lW = lW;
    if (!p.done) {                                                           // _ve_envelope_shift (lib/envelope.c:358-372)
      const long long need = current / step + 2;
      if (need > K.cap) {
        atomicOr(K.overflow, 1);
      } else {
        uint8_t *cm = K.marks + (size_t)st * K.cap;
        for (long long i = 0; i < K.cap; i++) cm[i] = i < need && mk[i + shift / step] ? 1 : 0;
      }
    }
  }
}

__global__ void __launch_bounds__(128)
k_plan_blocks(int nstreams, int bs0, int bs1, const int32_t *__restrict__ mark, long long mark_stride,
              int nsteps_max, const int64_t *__restrict__ pcm_len, const int64_t *__restrict__ eof, int max_blocks,
              vb200_stream_block *__restrict__ plan, int32_t *__restrict__ nblocks, int32_t *__restrict__ counts) {
  plan_blocks_body<false>(nstreams, bs0, bs1, mark, mark_stride, nsteps_max, pcm_len, eof, max_blocks, plan, nblocks,
                          counts, CarryDev{});
}

__global__ void __launch_bounds__(128)
k_plan_blocks_carry(int nstreams, int bs0, int bs1, const int32_t *__restrict__ mark, long long mark_stride,
                    int nsteps_max, const int64_t *__restrict__ pcm_len, const int64_t *__restrict__ eof, int max_blocks,
                    vb200_stream_block *__restrict__ plan, int32_t *__restrict__ nblocks, int32_t *__restrict__ counts,
                    CarryDev K) {
  plan_blocks_body<true>(nstreams, bs0, bs1, mark, mark_stride, nsteps_max, pcm_len, eof, max_blocks, plan, nblocks,
                         counts, K);
}

// exclusive prefix sums of the per-stream block counts, one thread per block size (a few thousand adds);
// offs[2*st + W]; totals[W] at the end
__global__ void k_plan_offsets(int nstreams, const int32_t *__restrict__ counts, int32_t *__restrict__ offs,
                               int32_t *__restrict__ totals) {
  const int W = threadIdx.x;
  if (W > 1) return;
  int acc = 0;
  for (int st = 0; st < nstreams; st++) { offs[2 * st + W] = acc; acc += counts[2 * st + W]; }
  totals[W] = acc;
}

// slots + the gather table and descriptors of the two batches (entries past cap[W] are dropped; the host
// checks the totals)
__global__ void __launch_bounds__(128)
k_plan_fill(int nstreams, int max_blocks, vb200_stream_block *__restrict__ plan, const int32_t *__restrict__ nblocks,
            const int32_t *__restrict__ offs, int cap0, int cap1,
            int2 *__restrict__ src0, int2 *__restrict__ src1,
            vb200_block_desc *__restrict__ desc0, vb200_block_desc *__restrict__ desc1) {
  const int st = blockIdx.x * blockDim.x + threadIdx.x;
  if (st >= nstreams) return;
  vb200_stream_block *p = plan + (size_t)st * max_blocks;
  const int nb = nblocks[st];
  for (int k = 0; k < nb; k++) {
    const int W = p[k].W;
    const int slot = p[k].slot + offs[2 * st + W];
    p[k].slot = slot;
    if (slot < (W ? cap1 : cap0)) {
      vb200_block_desc d;
      d.lW = p[k].lW; d.nW = p[k].nW; d.blocktype = p[k].blocktype; d.ampmax = 0.f;
      (W ? src1 : src0)[slot] = make_int2(st, p[k].pos);
      (W ? desc1 : desc0)[slot] = d;
    }
  }
}

// every block's global_ampmax: the decay chain of vorbis_analysis_blockout along the stream
// (lib/block.c:626-628: g = max(g, previous block's ampmax on exit); g = _vp_ampmax_decay(g) with the CURRENT
// block's size, lib/psy.c:837-848), then the block's own local maxima (lib/mapping0.c:244,346)
template <bool CARRY>
__device__ __forceinline__ void ampmax_plan_body(int nstreams, int max_blocks, int ch,
                                                 const vb200_stream_block *__restrict__ plan,
                                                 const int32_t *__restrict__ nblocks, const float *__restrict__ lmax0,
                                                 const float *__restrict__ lmax1, float secs_att0, float secs_att1,
                                                 float *__restrict__ gmax0, float *__restrict__ gmax1, PlanCarry *pc) {
  const int st = blockIdx.x * blockDim.x + threadIdx.x;
  if (st >= nstreams) return;
  const vb200_stream_block *p = plan + (size_t)st * max_blocks;
  const int nb = nblocks[st];
  float g = -9999.f, prev = -9999.f;
  if (CARRY) { g = pc[st].gmax; prev = pc[st].prev; }
  for (int k = 0; k < nb; k++) {
    const int W = p[k].W, slot = p[k].slot;
    if (prev > g) g = prev;
    g = g + (W ? secs_att1 : secs_att0);
    if (g < -9999.f) g = -9999.f;
    float o = g;
    const float *lm = (W ? lmax1 : lmax0) + (size_t)slot * ch;
    for (int c = 0; c < ch; c++) o = fmaxf(o, lm[c]);
    (W ? gmax1 : gmax0)[slot] = o;
    prev = o;
  }
  if (CARRY) { pc[st].gmax = g; pc[st].prev = prev; }
}

__global__ void __launch_bounds__(128)
k_ampmax_plan(int nstreams, int max_blocks, int ch, const vb200_stream_block *__restrict__ plan,
              const int32_t *__restrict__ nblocks, const float *__restrict__ lmax0, const float *__restrict__ lmax1,
              float secs_att0, float secs_att1, float *__restrict__ gmax0, float *__restrict__ gmax1) {
  ampmax_plan_body<false>(nstreams, max_blocks, ch, plan, nblocks, lmax0, lmax1, secs_att0, secs_att1, gmax0, gmax1,
                          nullptr);
}

// g and prev start from the carry and go back to it
__global__ void __launch_bounds__(128)
k_ampmax_plan_carry(int nstreams, int max_blocks, int ch, const vb200_stream_block *__restrict__ plan,
                    const int32_t *__restrict__ nblocks, const float *__restrict__ lmax0, const float *__restrict__ lmax1,
                    float secs_att0, float secs_att1, float *__restrict__ gmax0, float *__restrict__ gmax1,
                    PlanCarry *__restrict__ pc) {
  ampmax_plan_body<true>(nstreams, max_blocks, ch, plan, nblocks, lmax0, lmax1, secs_att0, secs_att1, gmax0, gmax1, pc);
}

}  // namespace vb200
