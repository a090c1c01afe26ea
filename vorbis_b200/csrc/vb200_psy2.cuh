// vb200_psy2.cuh — k_phaseA_psy2: the fused noise/tone/mix kernel, occupancy-first layout.
//
// The psy stage is latency bound and its throughput scales with resident
// CTAs, so this version minimises shared memory per (block,channel) row:
//   * every per-bin value a thread needs twice (logmdct, first-pass noise) stays in
//     registers: thread t owns bins t, t+128, ... in every per-bin phase;
//   * the tone scratch (logfft copy, seeds, chase stacks, run records) is dead before the
//     noise prefix sums start, so it aliases the 5x(n+4) prefix-sum area;
//   * the tone curve is never materialised: bins read their group's minimum (grp_min).
// => 5(n+4)+ngrp+1 floats (22 KB at n=1024) instead of 54 KB: 8-9 CTAs/SM instead of 4.
// All phases use all 128 threads; seed_chase runs block-wide with the same exact
// segmentation as dev_tone_chase_gather (restart points = strict records).
#pragma once
#include "vb200_kernels.cuh"

namespace vb200 {

struct PhaseA2Args {
  const float *mdct_in;   // [rows][n] raw mdct
  const float *logfft;    // [rows][n]
  const float *lmax;      // [rows]
  const float *gmax;      // [blocks]
  const vb200_block_desc *desc;
  float *mdct_out;        // [rows][n] (may alias mdct_in)
  float *logmdct;         // [rows][n]
  float *logmask;         // [rows][n]
  float *ampmax_out;      // [blocks]
  float *tap_noise, *tap_tone;
  int dbg_skip;           // timing experiments only (VB200_DEBUG_SKIP); 0 in production
  unsigned long long *dbg_cycles;   // optional [16]: per-phase SM cycles summed over rows (thread 0 of each CTA)
};

constexpr int PSY2_THREADS = 128;
#ifndef PSY2_MINB
#define PSY2_MINB 8
#endif

__host__ __device__ inline size_t psy2_floats(int n, int total, int nruns, int ngrp) {
  const int tp = (total + 7) & ~7, rp = (nruns + 3) & ~3;
  size_t tone = (size_t)n + 2 * (size_t)tp + tp / 2 + 4 * (size_t)rp;       // fft, seed, astk, pstk, run records
  size_t recs = (size_t)((((total + 3) / 4 + 31) & ~31) * 4 + 1) / 2 + 8;   // 4 chunks of shorts
  if (recs < 4 * 224 / 2 + 8) recs = 4 * 224 / 2 + 8;
  if (4 * (size_t)rp < recs) tone += recs - 4 * (size_t)rp;
  const size_t scan = 5 * (size_t)(n + 4);
  return (scan > tone ? scan : tone) + (size_t)((ngrp + 1 + 3) & ~3) + 16;
}

// The per-bin regression and mix are called 8x (bins per thread) x 3 (windows); inlining them
// made the kernel ~93 KB of SASS and 11 % of the stall samples were instruction-cache misses.
// They are real functions here (scalars only in the signature, so nothing spills to local).
template <int NS>
__device__ __forceinline__ float dev_regress_bin(const int *__restrict__ bark, int bfe, int ffe, const float *S,
                                                 int i, float offset, int fixed) {
  Abd cur; cur.A = 0.f; cur.B = 0.f; cur.D = 1.f;
  if (bfe > 0) {
    const int wb = i < bfe ? i : bfe - 1;
    const int bk = __ldg(bark + wb);
    cur = dev_window_abd(bk >> 16, bk & 0xffff, S, NS);
  }
  const float x = (float)i;
  float R = (cur.A + x * cur.B) / cur.D;
  if (R < 0.f) R = 0.f;
  float v = R - offset;
  if (fixed > 0) {
    if (ffe > 0) {
      const int wb = i < ffe ? i : ffe - 1;
      const int hi = wb + fixed / 2, lo = hi - fixed;
      cur = dev_window_abd(lo, hi, S, NS);
    } else if (bfe > 0 && i < bfe) {
      const int bk = __ldg(bark + (bfe - 1));
      cur = dev_window_abd(bk >> 16, bk & 0xffff, S, NS);
    }
    const float R2 = (cur.A + x * cur.B) / cur.D;
    if (R2 - offset < v) v = R2 - offset;
  }
  return v;
}

template <int NS>
__device__ __noinline__ float regress_core(const int *__restrict__ bark, int bfe, int ffe, const float *S,
                                           int i, float offset, int fixed) {
  return dev_regress_bin<NS>(bark, bfe, ffe, S, i, offset, fixed);
}

// final step of _vp_noisemask for one bin + tone lookup + _vp_offset_and_mix(select 1);
// returns logmask, updates m (the mdct value), writes the optional taps
struct MixConst { float noisemaxsupp, toneatt, m_val, att; };
__device__ __noinline__ float final_mix_core(float p2, float L, float p1, float noff, float ath, float gmin,
                                             const float *__restrict__ compand, MixConst C, float &m,
                                             float &nz_out, float &tn_out) {
  const float work = L - p1;                       // lib/psy.c:717
  const float base = L - work;                     // lib/psy.c:722
  int dB = (int)((double)p2 + .5);
  if (dB >= VB200_COMPAND_LEVELS) dB = VB200_COMPAND_LEVELS - 1;
  if (dB < 0) dB = 0;
  const float nz = base + __ldg(compand + dB);
  float tn = ath + C.att;                          // lib/psy.c:771, then max_seeds' flr update
  if (tn < gmin) tn = gmin;
  nz_out = nz; tn_out = tn;
  float val = nz + noff;                           // lib/psy.c:789-791
  if (val > C.noisemaxsupp) val = C.noisemaxsupp;
  const float t = tn + C.toneatt;
  const float logmask = val < t ? t : val;
  const float coeffi = -17.2f;
  float de;
  val = val - L;
  if (val > coeffi) {
    de = (float)(1.0 - ((double)(val - coeffi) * 0.005 * (double)C.m_val));
    if (de < 0.f) de = 0.0001f;
  } else {
    de = (float)(1.0 - ((double)(val - coeffi) * 0.0003 * (double)C.m_val));
  }
  m *= de;
  return logmask;
}

// block-wide seed_chase (see dev_tone_chase_gather for the exactness argument)
__device__ __forceinline__ void dev_chase_block(const PsyDev &P, const ToneSmem &T, int *s_misc,
                                                int tid, unsigned long long *dbg = nullptr) {
  long long tc = dbg ? clock64() : 0;
#define CHASE_MARK(slot) do { if (dbg && tid == 0) { const long long tn_ = clock64(); atomicAdd(dbg + (slot), (unsigned long long)(tn_ - tc)); tc = tn_; } } while (0)
  const int total = P.total, linesper = P.linesper;
  const int lane = tid & 31, warp = tid >> 5;
  float *seed = T.seed; short *pstk = T.pstk; float *astk = T.astk; short *rec = T.rec;
  const unsigned full = 0xffffffffu;
  // 1. restart points.  Thread t owns positions [t*RB, t*RB+RB); with L = linesper <= RB+1 the
  // window maxima over the previous / next L-1 seeds come from the suffix maximum of the previous
  // block, the prefix/suffix maxima inside the own block and the prefix maximum of the next block.
  //   rule A: seeds[i] > max(seeds[i-L+1 .. i-1])   (strict; positions < 0 do not exist)
  //   rule C: seeds[i] > max(seeds[i+1 .. i+L-1])   (strict; positions >= total do not exist)
  constexpr int RB = 7;
  const int C = 32 * RB;                                    // positions per warp
  int m = 0;
  if (linesper - 1 <= RB && total <= PSY2_THREADS * RB) {
    const float NINF = -3.0e38f;                            // below every seed (>= -9999)
    float v[3 * RB];
    const int p0 = tid * RB - RB;
#pragma unroll
    for (int j = 0; j < 3 * RB; j++) { const int p = p0 + j; v[j] = (p >= 0 && p < total) ? seed[p] : NINF; }
    unsigned flags = 0;
#pragma unroll
    for (int j = 0; j < RB; j++) {
      const int i = tid * RB + j;
      float mb = NINF, mf = NINF;
#pragma unroll
      for (int d = 1; d <= RB; d++) {
        if (d < linesper) { mb = fmaxf(mb, v[RB + j - d]); mf = fmaxf(mf, v[RB + j + d]); }
      }
      const bool r = i < total && (v[RB + j] > mb || v[RB + j] > mf);
      flags |= (r ? 1u : 0u) << j;
    }
    // ordered compaction: records are numbered by position = by (thread, j)
    const int cnt = __popc(flags);
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(full, incl, o); if (lane >= o) incl += t; }
    int w = warp * C + incl - cnt;
#pragma unroll
    for (int j = 0; j < RB; j++) if (flags & (1u << j)) rec[w++] = (short)(tid * RB + j);
    m = __shfl_sync(full, incl, 31);
  } else {
    const int Cg = (((total + 3) >> 2) + 31) & ~31;
    for (int base = warp * Cg; base < (warp + 1) * Cg && base < total; base += 32) {
      const int i = base + lane;
      bool r = i < total;
      {
        const float vv = r ? seed[i] : 0.f;
        bool ra = r, rc = r;
        for (int d = 1; d < linesper; d++) {
          const int j = i - d, h = i + d;
          const float u = (r && j >= 0) ? seed[j] : 0.f;
          const float ww = (r && h < total) ? seed[h] : 0.f;
          ra = ra && (j < 0 || vv > u);
          rc = rc && (h >= total || vv > ww);
        }
        r = ra || rc;
      }
      const unsigned bb = __ballot_sync(full, r);
      if (r) rec[warp * Cg + m + __popc(bb & ((1u << lane) - 1u))] = (short)i;
      m += __popc(bb);
    }
  }
  const int Cw = (linesper - 1 <= RB && total <= PSY2_THREADS * RB) ? C : ((((total + 3) >> 2) + 31) & ~31);
  if (lane == 0) s_misc[warp] = m;
  __syncthreads();
  CHASE_MARK(11);   // records
  const int m0 = s_misc[0], m1 = s_misc[1], m2 = s_misc[2], m3 = s_misc[3];
  const int M = m0 + m1 + m2 + m3;
  auto REC = [&](int g) -> int {
    if (g < m0) return rec[g];
    g -= m0; if (g < m1) return rec[Cw + g];
    g -= m1; if (g < m2) return rec[2 * Cw + g];
    return rec[3 * Cw + g - m2];
  };
  // 2. this thread's segment [start, end]
  const int r0 = (tid * M) >> 7, r1 = ((tid + 1) * M) >> 7;
  int start = 0, end = 0, cnt = 0;
  if (r0 < r1) {
    start = REC(r0);
    end = r1 < M ? REC(r1) : total;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    int l0 = 0, l1 = 0, l2 = 0, c = 0, stack = 0;
    const unsigned as_ = smem_u32(seed), aa = smem_u32(astk) + 4u * start, ap = smem_u32(pstk) + 2u * start;
    const int last = end < total ? end : total - 1;
    float s = lds_f32(as_ + 4u * start);
    for (int i = start; i <= last; i++) {
      const float snext = lds_f32(as_ + 4u * (i + 1 < total ? i + 1 : i));
      if (stack >= 2 && !(s < a0)) {
        for (;;) {
          if (c < 2) { a1 = lds_f32(aa + 4u * (stack - 2)); l1 = lds_s16(ap + 2u * (stack - 2)) + linesper; c = 2; }
          if (!(i < l0 && a0 <= a1 && i < l1)) break;
          stack--;
          a0 = a1; l0 = l1; a1 = a2; l1 = l2; c--;
          if (stack < 2 || s < a0) break;
        }
      }
      if (i < end) {
        sts_f32(aa + 4u * stack, s); sts_s16(ap + 2u * stack, i);
        a2 = a1; l2 = l1; a1 = a0; l1 = l0; a0 = s; l0 = i + linesper;
        stack++;
        c = c < 3 ? c + 1 : 3;
      }
      s = snext;
    }
    cnt = stack;
  }
  __syncthreads();
  CHASE_MARK(12);   // simulate
  // 3. fill: exclusive prefix-max of every thread's furthest endpos = its starting cursor
  int Mx = 0;
  for (int j = 0; j < cnt; j++) {
    const float a = astk[start + j];
    int endpos;
    const int nx = j + 1 < cnt ? start + j + 1 : (end < total ? end : -1);
    if (nx >= 0 && astk[nx] > a) endpos = pstk[nx];
    else endpos = pstk[start + j] + linesper + 1;
    if (endpos > total) endpos = total;
    if (endpos > Mx) Mx = endpos;
  }
  int incl = Mx;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(full, incl, o);
    if (lane >= o && t > incl) incl = t;
  }
  if (lane == 31) s_misc[4 + warp] = incl;
  int cursor = __shfl_up_sync(full, incl, 1);
  if (lane == 0) cursor = 0;
  __syncthreads();
  for (int w = 0; w < warp; w++) { const int t = s_misc[4 + w]; if (t > cursor) cursor = t; }
  for (int j = 0; j < cnt; j++) {
    const float a = astk[start + j];
    int endpos;
    const int nx = j + 1 < cnt ? start + j + 1 : (end < total ? end : -1);
    if (nx >= 0 && astk[nx] > a) endpos = pstk[nx];
    else endpos = pstk[start + j] + linesper + 1;
    if (endpos > total) endpos = total;
    for (int p = cursor; p < endpos; p++) seed[p] = a;
    if (endpos > cursor) cursor = endpos;
  }
  __syncthreads();
  CHASE_MARK(13);   // fill
#undef CHASE_MARK
}

template <int K>   // K = n / 128 bins per thread
__global__ void __launch_bounds__(PSY2_THREADS, PSY2_MINB)
k_phaseA_psy2(PsyDev P0, PsyDev P1, int ch, int nrows, PhaseA2Args A) {
  extern __shared__ __align__(16) float sm[];
  constexpr int nt = PSY2_THREADS;
  const int n = K * nt, ns = n + 4, tid = threadIdx.x, lane = tid & 31;
  const int total = P0.total > P1.total ? P0.total : P1.total;
  const int nruns = P0.nruns > P1.nruns ? P0.nruns : P1.nruns;
  const int ngrp = P0.ngrp > P1.ngrp ? P0.ngrp : P1.ngrp;
  const int tp = (total + 7) & ~7, rp = (nruns + 3) & ~3;
  // carve: [ scan area | tone scratch (aliased) ] [ grp_min ] [ misc ]
  float *S = sm;
  float *s_fft = sm;
  ToneSmem T;
  T.seed = s_fft + n; T.astk = T.seed + tp; T.pstk = reinterpret_cast<short *>(T.astk + tp);
  T.run_rec = reinterpret_cast<int4 *>(T.astk + tp + tp / 2);
  T.rec = reinterpret_cast<short *>(T.run_rec);
  (void)rp;
  const size_t area = psy2_floats(n, total, nruns, ngrp) - (size_t)((ngrp + 1 + 3) & ~3) - 16;
  float *grp_min = sm + area;
  int *s_misc = reinterpret_cast<int *>(grp_min + ((ngrp + 1 + 3) & ~3));
  for (int row = blockIdx.x; row < nrows; row += gridDim.x) {
    const int blk = row / ch;
    const PsyDev &P = A.desc[blk].blocktype ? P1 : P0;
    const float *gm = A.mdct_in + (size_t)row * n;
    const float *lf = A.logfft + (size_t)row * n;
    const float g = A.gmax[blk], lmax = A.lmax[row];
    float L[K], M[K], p1[K];
    long long tmark = A.dbg_cycles ? clock64() : 0;
    int tph = 0;
#define PHASE_MARK()                                                              \
    do {                                                                          \
      if (A.dbg_cycles && tid == 0) {                                             \
        const long long tnow = clock64();                                         \
        atomicAdd(A.dbg_cycles + tph, (unsigned long long)(tnow - tmark));        \
        tmark = tnow;                                                             \
      }                                                                           \
      tph++;                                                                      \
    } while (0)
#pragma unroll
    for (int k = 0; k < K; k++) {
      const int i = tid + k * nt;
      M[k] = __ldcs(gm + i);                            // streaming: keep L1 for the lookup tables
      s_fft[i] = __ldcs(lf + i);
    }
#pragma unroll
    for (int k = 0; k < K; k++) {
      L[k] = add345(todB_dev(M[k]));                    // lib/mapping0.c:384-385
      __stcs(A.logmdct + (size_t)row * n + tid + k * nt, L[k]);
    }
    __syncthreads();
    PHASE_MARK();   // 0 load
    dev_tone_runs(P, s_fft, g, lmax, T, tid, nt);
    __syncthreads();
    PHASE_MARK();   // 1 runs
    dev_tone_slots(P, T, tid, nt);
    __syncthreads();
    PHASE_MARK();   // 2 scatter
    dev_chase_block(P, T, s_misc, tid, A.dbg_cycles);
    PHASE_MARK();   // 3 chase
    // max_seeds gather, first half: one minimum per static group (lib/psy.c:522-533)
    for (int q = tid; q <= P.ngrp; q += nt) {
      float minV;
      if (q < P.ngrp) {
        const int4 gg = __ldg(P.grps + q);
        if (gg.y - gg.x > 16) continue;                // long fold: done by a whole warp below
        int pos = gg.x;
        minV = T.seed[pos];
        if (minV > P.tone_abs_limit) minV = P.tone_abs_limit;
        while (pos < gg.y) {
          pos++;
          const float s = T.seed[pos];
          if ((s > VB_NEGINF && s < minV) || minV == VB_NEGINF) minV = s;
        }
      } else {
        minV = T.seed[P.total - 1];                    // tail bins (lib/psy.c:540-544)
      }
      grp_min[q] = minV;
    }
    // long groups (the first few bins span tens of seed slots): the fold equals the minimum over
    // the non-NEGINF seeds of the range, joined by tone_abs_limit iff the first seed is not
    // NEGINF, and NEGINF if there is none - associative, so a warp reduces it with shuffles
    for (int li = tid >> 5; li < P.nlong; li += nt >> 5) {
      const int q = __ldg(P.long_grp + li);
      const int4 gg = __ldg(P.grps + q);
      float mn = 3.0e38f;
      int any = 0;
      for (int pos = gg.x + lane; pos <= gg.y; pos += 32) {
        const float s = T.seed[pos];
        if (s > VB_NEGINF) {
          any = 1;
          if (s < mn) mn = s;
          if (pos == gg.x && P.tone_abs_limit < mn) mn = P.tone_abs_limit;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        any |= __shfl_xor_sync(0xffffffffu, any, o);
      }
      if (lane == 0) grp_min[q] = any ? mn : VB_NEGINF;
    }
    __syncthreads();                                   // tone scratch is dead from here on
    PHASE_MARK();   // 4 group minima
    // ---- noise mask, pass 1 (offset 140, bark windows)
#pragma unroll
    for (int k = 0; k < K; k++) dev_noise_term1(tid + k * nt, L[k], 140.f, S, ns);
    __syncthreads();
    PHASE_MARK();   // 5 terms 1
    if (tid < 32) dev_noise_scan(n, S, ns, lane);
    __syncthreads();
    PHASE_MARK();   // 6 scan 1
#pragma unroll
    for (int k = 0; k < K; k++)
      p1[k] = regress_core<K * PSY2_THREADS + 4>(P.bark, P.bark_first_extra, P.fixed_first_extra, S, tid + k * nt, 140.f, -1);
    __syncthreads();
    PHASE_MARK();   // 7 regress 1
    // ---- pass 2 on logmdct - p1 (offset 0, bark + fixed windows)
#pragma unroll
    for (int k = 0; k < K; k++) dev_noise_term1(tid + k * nt, L[k] - p1[k], 0.f, S, ns);
    __syncthreads();
    PHASE_MARK();   // 8 terms 2
    if (tid < 32) dev_noise_scan(n, S, ns, lane);
    __syncthreads();
    PHASE_MARK();   // 9 scan 2
    MixConst MC;
    MC.noisemaxsupp = P.noisemaxsupp; MC.toneatt = P.tone_masteratt[1]; MC.m_val = P.m_val;
    MC.att = tone_att(P, lmax);
    const float *noff = P.noiseoffset + n;             // offset_select 1
    const int *bark = P.bark; const float *athp = P.ath, *compand = P.noisecompand;
    const short *bin_grp = P.bin_grp;
    const int bfe = P.bark_first_extra, ffe = P.fixed_first_extra, fixedw = P.noisewindowfixed;
#pragma unroll
    for (int k = 0; k < K; k++) {
      const int i = tid + k * nt;
      const float p2 = regress_core<K * PSY2_THREADS + 4>(bark, bfe, ffe, S, i, 0.f, fixedw);
      float m = M[k], nz, tn;
      const float lm = final_mix_core(p2, L[k], p1[k], __ldg(noff + i), __ldg(athp + i),
                                      grp_min[__ldg(bin_grp + i)], compand, MC, m, nz, tn);
      __stcs(A.logmask + (size_t)row * n + i, lm);
      __stcs(A.mdct_out + (size_t)row * n + i, m);
      if (A.tap_noise) A.tap_noise[(size_t)row * n + i] = nz;
      if (A.tap_tone) A.tap_tone[(size_t)row * n + i] = tn;
    }
    if (tid == 0 && (row % ch) == 0) A.ampmax_out[blk] = g;   // lib/mapping0.c:576
    __syncthreads();
    PHASE_MARK();   // 10 regress 2 + final + mix
#undef PHASE_MARK
  }
}

}  // namespace vb200
