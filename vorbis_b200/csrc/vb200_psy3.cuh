// vb200_psy3.cuh — k_phaseA_psy3: the fused noise/tone/mix kernel, instruction-count-first layout.
//
// The kernel is issue bound, not DRAM bound.  Every 128 threads work on one (block,channel) row, with
// the per-bin values in registers and the tone scratch aliased with the prefix-sum area, and the
// phases are laid out so that few lanes sit idle:
//
//  * seed_curve scatter (lib/psy.c:390-415).  A run only has ~13 usable curve points (6..43 on
//    the bench signal), so walking one run with 16 lanes spent ~50 instructions per 26 useful
//    updates.  Here every warp owns a PRIVATE copy of the seed vector and walks a quarter of the
//    runs of all eight residue classes at once: 4 lanes per class, lane q owning the class slots
//    = q (mod 4), so that no two lanes ever touch the same slot (no __syncwarp, no atomics) and
//    the 32 lanes of a warp hit 32 different banks.  The four copies are max-merged afterwards;
//    max is order independent, so the result is bit-identical to the sequential scatter.
//  * seed_chase (lib/psy.c:454-508): restart points from van Herk prefix/suffix maxima (7-wide
//    windows = linesper-1), segments by position (no compaction), and ONE predicated loop whose
//    iteration is either a pop or a push, so that lanes that pop do not stall lanes that push.
//  * the two sequential prefix sums run without register copies (two alternating register sets).
//
// Requires linesper == 8 (always, lib/modes/psych_*.h eighth_octave_lines) and
// total_octave_lines <= 896; other setups use the generic k_phaseA_psy.  The exactness argument for
// the restart points is in vb200_kernels.cuh (dev_tone_chase_gather).
#pragma once
#include "vb200_kernels.cuh"

namespace vb200 {

constexpr int PSY3_THREADS = 128;
constexpr int PSY3_L = 8;            // eighth_octave_lines
constexpr int PSY3_RB = 7;           // chase positions per thread = linesper - 1
#ifndef PSY3_MINB
#define PSY3_MINB 8
#endif

__host__ __device__ inline bool psy3_supported(int n, int total, int linesper) {
  return linesper == PSY3_L && total <= PSY3_THREADS * PSY3_RB && total >= 2 * PSY3_L &&
         (n == 128 || n == 256 || n == 512 || n == 1024 || n == 2048);
}

// floats of dynamic shared memory: [ scan area | tone scratch (aliased) ] [ grp_min ] [ misc ]
__host__ __device__ inline size_t psy3_tone_floats(int n, int total, int nruns) {
  const int tp = (total + 7) & ~7, rp = (nruns + 3) & ~3;
  size_t a0 = 4 * (size_t)tp;                       // four private seed copies; the logfft copy aliases them
  if (a0 < (size_t)n) a0 = n;
  return a0 + 4 * (size_t)rp;                       // + run records (int4)
}
__host__ __device__ inline size_t psy3_floats(int n, int total, int nruns, int ngrp) {
  const size_t tone = psy3_tone_floats(n, total, nruns);
  const size_t scan = 5 * (size_t)(n + 4);
  return (scan > tone ? scan : tone) + (size_t)((ngrp + 1 + 3) & ~3) + 16;
}

// ---- seed_loop: one item per run -> 16-byte record (peak, first curve index, first slot, count)
__device__ __forceinline__ void dev_tone_runs3(const PsyDev &P, const float *logfft, float gmax, float att,
                                               int4 *run_rec, int tid) {
  const float dBoffset = P.max_curve_dB - gmax;
  const int total = P.total;
#pragma unroll 1
  for (int k = tid; k < P.nruns; k += PSY3_THREADS) {
    const int4 rr = __ldg(P.runrec + k);             // lo|hi<<16, oc - firstoc, band, bits(ath[hi])
    const int lo = rr.x & 0xffff, hi = rr.x >> 16;
    float mx = logfft[lo];
#pragma unroll 1
    for (int i = lo + 1; i <= hi; i++) { const float v = logfft[i]; if (v > mx) mx = v; }
    int4 rec = make_int4(__float_as_int(mx), 0, 0, 0);
    if (mx + 6.f > __int_as_float(rr.w) + att) {     // lib/psy.c:438
      int choice = (int)((((double)(mx + dBoffset)) - 30.) * (double).1f);   // P_LEVEL_0 is a double
      if (choice < 0) choice = 0;
      if (choice > VB200_P_LEVELS - 1) choice = VB200_P_LEVELS - 1;
      const int cbase = (rr.z * VB200_P_LEVELS + choice) * (VB200_EHMER_MAX + 2);
      int post0 = (int)__ldg(P.tonecurves + cbase), post1 = (int)__ldg(P.tonecurves + cbase + 1);
      // clip to slots 1..total-1:  sp(i) = oc + (i-16)*L - L/2   (lib/psy.c:403-413)
      const int sp_at0 = rr.y - 16 * PSY3_L - (PSY3_L >> 1);
      const int ilo = sp_at0 > 0 ? 0 : ((-sp_at0) >> 3) + 1;               // smallest i with sp(i) > 0
      const int ihi = total - sp_at0 <= 0 ? 0 : (total - sp_at0 + PSY3_L - 1) >> 3;   // smallest i with sp(i) >= total
      if (post0 < ilo) post0 = ilo;
      if (post1 > ihi) post1 = ihi;
      if (post0 < post1) {
        rec.y = cbase + 2 + post0;
        rec.z = sp_at0 + post0 * PSY3_L;
        rec.w = post1 - post0;
      }
    }
    run_rec[k] = rec;
  }
}

// ---- seed_curve for all runs: private copy per warp, 4 lanes per residue class
__device__ __forceinline__ void dev_tone_scatter3(const PsyDev &P, float *copies, int tp, const int4 *run_rec, int tid) {
  const int w = tid >> 5, lane = tid & 31, c = lane >> 2, q = lane & 3;
  float *my = copies + w * tp;
  {
    const float4 ninf = make_float4(VB_NEGINF, VB_NEGINF, VB_NEGINF, VB_NEGINF);
#pragma unroll 1
    for (int v = lane; v < (tp >> 2); v += 32) reinterpret_cast<float4 *>(my)[v] = ninf;
  }
  __syncwarp();
  const int k0 = __ldg(P.cls_off + c), k1 = __ldg(P.cls_off + c + 1);
  const int trips = (P.max_cls_len - w + 3) >> 2;    // warp-uniform
  const unsigned a_my = smem_u32(my), a_rec = smem_u32(run_rec);
  const float *__restrict__ curves = P.tonecurves;
#pragma unroll 1
  for (int it = 0; it < trips; it++) {
    const int k = k0 + w + 4 * it;                   // this warp's it-th run of class c
    if (k < k1) {
      const int4 r = lds_v4(a_rec + 16u * (unsigned)k);
      const float mx = __int_as_float(r.x);
      const int cnt = r.w;
      int j = (q - (r.z >> 3)) & 3;                  // first point that lands on a slot this lane owns
      const float *cp = curves + r.y + j;
      unsigned a = a_my + 4u * (unsigned)(r.z + PSY3_L * j);
#pragma unroll 1
      while (j < cnt) {
        const bool p1 = j + 4 < cnt, p2 = j + 8 < cnt, p3 = j + 12 < cnt;
        const float v0 = __ldg(cp);
        const float v1 = p1 ? __ldg(cp + 4) : 0.f;
        const float v2 = p2 ? __ldg(cp + 8) : 0.f;
        const float v3 = p3 ? __ldg(cp + 12) : 0.f;
        sts_f32(a, fmaxf(lds_f32(a), mx + v0));       // if(seed[seedptr]<lin)seed[seedptr]=lin
        if (p1) sts_f32(a + 128u, fmaxf(lds_f32(a + 128u), mx + v1));
        if (p2) sts_f32(a + 256u, fmaxf(lds_f32(a + 256u), mx + v2));
        if (p3) sts_f32(a + 384u, fmaxf(lds_f32(a + 384u), mx + v3));
        j += 16; cp += 16; a += 512u;
      }
    }
  }
}

// ---- merge of the four copies + seed_chase, block wide.  On return copies[0..total) holds the chased seeds.
template <bool DBG>
__device__ __forceinline__ void dev_chase3(const PsyDev &P, float *copies, int tp, int *s_misc, int tid,
                                           unsigned long long *dbg = nullptr) {
  constexpr int RB = PSY3_RB, L = PSY3_L;
  long long tc = (DBG && dbg) ? clock64() : 0;
#define CHASE_MARK(slot) do { if (DBG && dbg && tid == 0) { const long long tn_ = clock64(); atomicAdd(dbg + (slot), (unsigned long long)(tn_ - tc)); tc = tn_; } } while (0)
  const int total = P.total;
  const int lane = tid & 31, warp = tid >> 5;
  const unsigned full = 0xffffffffu;
  float *seed = copies, *astk = copies + tp;
  int *lstk = reinterpret_cast<int *>(copies + 2 * tp);      // position + L of every stack entry (what the pop test compares)
  const float NINF = -3.0e38f;                       // below every seed (>= -9999)
  const int p0 = tid * RB;
  // 0. merge: this thread's RB positions
  float own[RB];
#pragma unroll
  for (int j = 0; j < RB; j++) {
    const int p = p0 + j;
    float v = NINF;
    if (p < total) {
      v = fmaxf(fmaxf(copies[p], copies[tp + p]), fmaxf(copies[2 * tp + p], copies[3 * tp + p]));
      seed[p] = v;
    }
    own[j] = v;
  }
  __syncthreads();
  // 1. restart points:  rule A: seeds[i] > max(seeds[i-L+1 .. i-1]);  rule C: seeds[i] > max(seeds[i+1 .. i+L-1])
  // (positions outside [0,total) do not exist).  With RB = L-1 the two windows of position p0+j are
  // prev[j..] + own[..j-1] and own[j+1..] + next[..j]: suffix/prefix maxima (van Herk).
  unsigned flags = 0;
  {
    float prev[RB], next[RB], pre[RB], suf[RB];
#pragma unroll
    for (int j = 0; j < RB; j++) {
      const int pp = p0 - RB + j, pn = p0 + RB + j;
      prev[j] = (pp >= 0 && pp < total) ? seed[pp] : NINF;
      next[j] = pn < total ? seed[pn] : NINF;
    }
#pragma unroll
    for (int j = RB - 2; j >= 0; j--) prev[j] = fmaxf(prev[j], prev[j + 1]);
#pragma unroll
    for (int j = 1; j < RB; j++) next[j] = fmaxf(next[j], next[j - 1]);
    pre[0] = own[0]; suf[RB - 1] = own[RB - 1];
#pragma unroll
    for (int j = 1; j < RB; j++) pre[j] = fmaxf(pre[j - 1], own[j]);
#pragma unroll
    for (int j = RB - 2; j >= 0; j--) suf[j] = fmaxf(suf[j + 1], own[j]);
#pragma unroll
    for (int j = 0; j < RB; j++) {
      const float mb = j == 0 ? prev[0] : fmaxf(prev[j], pre[j - 1]);
      const float mf = j == RB - 1 ? next[RB - 1] : fmaxf(suf[j + 1], next[j]);
      const bool r = p0 + j < total && (own[j] > mb || own[j] > mf);
      flags |= (r ? 1u : 0u) << j;
    }
  }
  // 2. segments by position: a thread with a restart point in its block simulates from its first one up to
  // the first restart point of the next such thread (position 0 always is one, so the segments tile [0,total))
  const int BIG = 1 << 20;
  const int start = flags ? p0 + __ffs((int)flags) - 1 : BIG;
  int sfx = start;                                   // inclusive suffix minimum over the warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_down_sync(full, sfx, o);
    if (lane + o < 32 && t < sfx) sfx = t;
  }
  if (lane == 0) s_misc[warp] = sfx;
  int end = __shfl_down_sync(full, sfx, 1);          // exclusive
  if (lane == 31) end = BIG;
  __syncthreads();
  CHASE_MARK(11);   // merge + restart points
  for (int w2 = warp + 1; w2 < (PSY3_THREADS >> 5); w2++) { const int t = s_misc[w2]; if (t < end) end = t; }
  if (end > total) end = total;
  // 3. the stack algorithm on [start, end) plus the pop phase of `end`.  One loop, one action per iteration:
  // pop the top entry, or push seeds[i] and advance.  Top two entries in registers (l = pos + L).
  int cnt = 0;
  if (start < BIG) {
    const unsigned as_ = smem_u32(seed), aa = smem_u32(astk) + 4u * (unsigned)start, dl = smem_u32(lstk) - smem_u32(astk);
    const int last = end < total ? end : total - 1;
    float a0 = 0.f, a1 = 0.f;
    int l0 = 0, l1 = 0, depth = 0, i = start;
    float s = lds_f32(as_ + 4u * (unsigned)i);
    const unsigned tl = (unsigned)(total - 1);
    unsigned top = aa;                               // address of the first free stack slot (amplitudes; positions at + dl)
    while (i <= last) {
      // lib/psy.c:465-484: pop while !(seeds[i] < amp[top]) and the two top entries both reach past i and
      // amp[top] <= amp[top-1]; otherwise push.  Branch free: every lane does exactly one of the two per
      // iteration, the memory operations are predicated.
      const bool pop = depth >= 2 && !(s < a0) && i < l0 && a0 <= a1 && i < l1;
      const bool push = !pop && i < end;             // i == end: only the pops belong to this segment
      const bool rel = pop && depth >= 3;            // the new second entry comes back from shared memory
      const unsigned o = pop ? top - 12u : top;
      const float ra = lds_f32_if(o, a1, rel);
      const int rl = lds_s32_if(o + dl, l1, rel);
      sts_f32_if(o, s, push);
      sts_s32_if(o + dl, i + L, push);
      const float na0 = pop ? a1 : (push ? s : a0);
      const int nl0 = pop ? l1 : (push ? i + L : l0);
      a1 = pop ? ra : (push ? a0 : a1);
      l1 = pop ? rl : (push ? l0 : l1);
      a0 = na0; l0 = nl0;
      const int dd = pop ? -1 : (push ? 1 : 0);
      depth += dd; top += 4 * dd;
      i += pop ? 0 : 1;
      const unsigned in = (unsigned)i < tl ? (unsigned)i : tl;
      s = lds_f32_if(as_ + 4u * in, s, !pop);
    }
    cnt = depth;
  }
  __syncthreads();
  CHASE_MARK(12);   // simulate
  // 4. fill (lib/psy.c:489-503): entry k is written from the running cursor to endpos_k; the cursor is the
  // running maximum of the earlier endpos values = exclusive prefix maximum over the threads
  int Mx = 0;
#pragma unroll 1
  for (int d = 0; d < cnt; d++) {
    const float a = astk[start + d];
    float an; int pn;
    if (d + 1 < cnt) { an = astk[start + d + 1]; pn = lstk[start + d + 1] - L; }
    else if (end < total) { an = astk[end]; pn = end; }          // first entry of the next segment
    else { an = NINF; pn = 0; }
    int endpos = an > a ? pn : lstk[start + d] + 1;
    if (endpos > total) endpos = total;
    lstk[start + d] = endpos;
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
  for (int w2 = 0; w2 < warp; w2++) { const int t = s_misc[4 + w2]; if (t > cursor) cursor = t; }
#pragma unroll 1
  for (int d = 0; d < cnt; d++) {
    const float a = astk[start + d];
    const int endpos = lstk[start + d];
#pragma unroll 1
    for (int p = cursor; p < endpos; p++) seed[p] = a;
    if (endpos > cursor) cursor = endpos;
  }
  __syncthreads();
  CHASE_MARK(13);   // fill
#undef CHASE_MARK
}

// The running sums are strictly sequential fp32 (order matters, SURVEY fact 8): five lanes, one array each.
// Two register sets alternate so that the next 16 values are in flight while 16 are accumulated and
// nothing is copied between registers.
__device__ __forceinline__ void dev_noise_scan3(int n, float *arr) {
  // explicit shared-window addresses: with generic pointers the compiler re-derived the base (S2R + IMAD, a
  // ~25-cycle scoreboard wait) inside the loop, on the one warp everybody else is waiting for
  unsigned a = smem_u32(arr);
  const int q = n >> 2;                   // float4 count, a multiple of 8 (n is a multiple of 128)
  float t = 0.f;
  float4 v0 = lds_f4(a), v1 = lds_f4(a + 16), v2 = lds_f4(a + 32), v3 = lds_f4(a + 48);
  float4 w0, w1, w2, w3;
#define SCAN4(v) do { t += v.x; v.x = t; t += v.y; v.y = t; t += v.z; v.z = t; t += v.w; v.w = t; } while (0)
#pragma unroll 1                       // one warp runs this: unrolled, the loop was 6.5 KB of once-through code per scan
  for (int i = 8; i < q; i += 8, a += 128) {
    w0 = lds_f4(a + 64); w1 = lds_f4(a + 80); w2 = lds_f4(a + 96); w3 = lds_f4(a + 112);
    SCAN4(v0); SCAN4(v1); SCAN4(v2); SCAN4(v3);
    sts_f4(a, v0); sts_f4(a + 16, v1); sts_f4(a + 32, v2); sts_f4(a + 48, v3);
    v0 = lds_f4(a + 128); v1 = lds_f4(a + 144); v2 = lds_f4(a + 160); v3 = lds_f4(a + 176);
    SCAN4(w0); SCAN4(w1); SCAN4(w2); SCAN4(w3);
    sts_f4(a + 64, w0); sts_f4(a + 80, w1); sts_f4(a + 96, w2); sts_f4(a + 112, w3);
  }
  w0 = lds_f4(a + 64); w1 = lds_f4(a + 80); w2 = lds_f4(a + 96); w3 = lds_f4(a + 112);
  SCAN4(v0); SCAN4(v1); SCAN4(v2); SCAN4(v3);
  sts_f4(a, v0); sts_f4(a + 16, v1); sts_f4(a + 32, v2); sts_f4(a + 48, v3);
  SCAN4(w0); SCAN4(w1); SCAN4(w2); SCAN4(w3);
  sts_f4(a + 64, w0); sts_f4(a + 80, w1); sts_f4(a + 96, w2); sts_f4(a + 112, w3);
#undef SCAN4
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

// Two bins per call: halves the call overhead of the (deliberately not inlined, see above) per-bin
// regression and gives the scheduler two independent dependency chains.
template <int NS>
__device__ __noinline__ float2 regress_pair(const int *__restrict__ bark, int bfe, int ffe, const float *S,
                                            int i0, int i1, float offset, int fixed) {
  float2 r;
  r.x = dev_regress_bin<NS>(bark, bfe, ffe, S, i0, offset, fixed);
  r.y = dev_regress_bin<NS>(bark, bfe, ffe, S, i1, offset, fixed);
  return r;
}

// final step of _vp_noisemask + tone lookup + _vp_offset_and_mix(select 1) for one bin, everything by value
struct MixConst { float noisemaxsupp, toneatt, m_val, att; };
struct MixOut { float logmask, m, nz, tn; };
__device__ __noinline__ MixOut final_mix_val(float p2, float L, float p1, float noff, float ath, float gmin,
                                             const float *__restrict__ compand, MixConst C, float m) {
  MixOut o;
  const float work = L - p1;                       // lib/psy.c:717
  const float base = L - work;                     // lib/psy.c:722
  int dB = (int)((double)p2 + .5);
  if (dB >= VB200_COMPAND_LEVELS) dB = VB200_COMPAND_LEVELS - 1;
  if (dB < 0) dB = 0;
  const float nz = base + __ldg(compand + dB);
  float tn = ath + C.att;                          // lib/psy.c:771, then max_seeds' flr update
  if (tn < gmin) tn = gmin;
  o.nz = nz; o.tn = tn;
  float val = nz + noff;                           // lib/psy.c:789-791
  if (val > C.noisemaxsupp) val = C.noisemaxsupp;
  const float t = tn + C.toneatt;
  o.logmask = val < t ? t : val;
  const float coeffi = -17.2f;
  float de;
  val = val - L;
  if (val > coeffi) {
    de = (float)(1.0 - ((double)(val - coeffi) * 0.005 * (double)C.m_val));
    if (de < 0.f) de = 0.0001f;
  } else {
    de = (float)(1.0 - ((double)(val - coeffi) * 0.0003 * (double)C.m_val));
  }
  o.m = m * de;
  return o;
}

// K = n / 128 bins per thread; R = rows per CTA (128 threads each).  The R rows of a CTA run in lockstep and
// share ONE scan warp: its lanes 5r..5r+4 carry the five running sums of row r, so the 1024 dependent
// warp-level FADDs per scan are paid once per R rows.
// DBG = true: the instance with the per-phase clock marks (tools/phase_timing.py) and the noise / tone taps of the
// stage-level API; the production instance carries neither (code size: instruction fetch is a first-order cost here)
template <int K, int R, bool DBG>
__global__ void __launch_bounds__(PSY3_THREADS * R, PSY3_MINB / R)
k_phaseA_psy3(PsyDev P0, PsyDev P1, int ch, int nrows, PsyArgs A) {
  extern __shared__ __align__(16) float sm_cta[];
  constexpr int nt = PSY3_THREADS;
  const int n = K * nt, ns = n + 4, tid = threadIdx.x & (nt - 1), half = threadIdx.x >> 7, lane = tid & 31;
  const int total = P0.total > P1.total ? P0.total : P1.total;
  const int nruns = P0.nruns > P1.nruns ? P0.nruns : P1.nruns;
  const int ngrp = P0.ngrp > P1.ngrp ? P0.ngrp : P1.ngrp;
  const int tp = (total + 7) & ~7;
  const size_t row_floats = (psy3_floats(n, total, nruns, ngrp) + 3) & ~(size_t)3;
  float *sm = sm_cta + half * row_floats;
  // carve (per row): [ scan area | tone scratch (aliased) ] [ grp_min ] [ misc ]
  float *S = sm;
  float *s_fft = sm;                                 // dead once the run records exist
  float *copies = sm;                                // 4 x tp
  size_t a0 = 4 * (size_t)tp; if (a0 < (size_t)n) a0 = n;
  int4 *run_rec = reinterpret_cast<int4 *>(sm + a0);
  const size_t area = psy3_floats(n, total, nruns, ngrp) - (size_t)((ngrp + 1 + 3) & ~3) - 16;
  float *grp_min = sm + area;
  int *s_misc = reinterpret_cast<int *>(grp_min + ((ngrp + 1 + 3) & ~3));
  for (int row0 = blockIdx.x * R; row0 < nrows; row0 += gridDim.x * R) {
    // an odd tail: the spare half repeats the last row in lockstep but stores none of the mix (the mix re-reads the
    // raw MDCT, which the other half may already have overwritten: mdct_out may alias mdct_in)
    const bool spare = row0 + half >= nrows;
    const int row = spare ? nrows - 1 : row0 + half;
    const int blk = row / ch;
    const PsyDev &P = A.desc[blk].blocktype ? P1 : P0;
    const float *gm = A.mdct_in + (size_t)row * n;
    const float *lf = A.logfft + (size_t)row * n;
    const float g = A.gmax[blk], lmax = A.lmax[row];
    const float att = tone_att(P, lmax);
    float L[K], p1[K];                                // the raw MDCT is read again by the mix: holding it here spilled
    long long tmark = (DBG && A.dbg_cycles) ? clock64() : 0;
    int tph = 0;
#define PHASE_MARK()                                                              \
    do {                                                                          \
      if (DBG && A.dbg_cycles && threadIdx.x == 0) {                                     \
        const long long tnow = clock64();                                         \
        atomicAdd(A.dbg_cycles + tph, (unsigned long long)(tnow - tmark));        \
        tmark = tnow;                                                             \
      }                                                                           \
      tph++;                                                                      \
    } while (0)
#pragma unroll
    for (int k = 0; k < K; k++) {
      const int i = tid + k * nt;
      L[k] = __ldcg(gm + i);                            // L2 only: keep L1 for the lookup tables
      s_fft[i] = __ldcs(lf + i);
    }
#pragma unroll
    for (int k = 0; k < K; k++) {
      L[k] = add345(todB_dev(L[k]));                    // lib/mapping0.c:384-385
      __stcs(A.logmdct + (size_t)row * n + tid + k * nt, L[k]);
    }
#ifndef VB200_NO_PREFETCH
    {   // the next row of this CTA: HBM -> L2 while this one is worked on (128-byte lines)
      const int nrow = row0 + gridDim.x * R + half;
      if (nrow < nrows && tid < 2 * (n / 32)) {
        const float *src = tid < n / 32 ? A.mdct_in : A.logfft;
        prefetch_l2(src + (size_t)nrow * n + (tid & (n / 32 - 1)) * 32);
      }
    }
#endif
    __syncthreads();
    PHASE_MARK();   // 0 load
    dev_tone_runs3(P, s_fft, g, att, run_rec, tid);
    __syncthreads();
    PHASE_MARK();   // 1 runs
    dev_tone_scatter3(P, copies, tp, run_rec, tid);
    __syncthreads();
    PHASE_MARK();   // 2 scatter
    dev_chase3<DBG>(P, copies, tp, s_misc, tid, half == 0 ? A.dbg_cycles : nullptr);
    PHASE_MARK();   // 3 chase
    // max_seeds gather, first half: one minimum per static group (lib/psy.c:522-533)
    const float *seed = copies;
#pragma unroll 1
    for (int q = tid; q <= P.ngrp; q += nt) {
      float minV;
      if (q < P.ngrp) {
        const int4 gg = __ldg(P.grps + q);
        if (gg.y - gg.x > 16) continue;                // long fold: done by a whole warp below
        int pos = gg.x;
        minV = seed[pos];
        if (minV > P.tone_abs_limit) minV = P.tone_abs_limit;
#pragma unroll 1
        while (pos < gg.y) {
          pos++;
          const float s = seed[pos];
          if ((s > VB_NEGINF && s < minV) || minV == VB_NEGINF) minV = s;
        }
      } else {
        minV = seed[P.total - 1];                      // tail bins (lib/psy.c:540-544)
      }
      grp_min[q] = minV;
    }
    // long groups (the first few bins span tens of seed slots): the fold equals the minimum over
    // the non-NEGINF seeds of the range, joined by tone_abs_limit iff the first seed is not
    // NEGINF, and NEGINF if there is none - associative, so a warp reduces it with shuffles
#pragma unroll 1
    for (int li = tid >> 5; li < P.nlong; li += nt >> 5) {
      const int q = __ldg(P.long_grp + li);
      const int4 gg = __ldg(P.grps + q);
      float mn = 3.0e38f;
      int any = 0;
#pragma unroll 1
      for (int pos = gg.x + lane; pos <= gg.y; pos += 32) {
        const float s = seed[pos];
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
    // ---- noise mask: two passes of the same three steps (terms, sequential sums, windowed regressions), ONE copy
    // of the code (instruction fetch is a first-order cost in this kernel): pass 0 on logmdct with offset 140 and
    // the bark windows only -> p1, pass 1 on logmdct - p1 with offset 0 and bark + fixed windows -> p2
    // (lib/psy.c:706-726; logmdct - 0.f is logmdct exactly)
    const int *bark = P.bark;
    const int bfe = P.bark_first_extra, ffe = P.fixed_first_extra, fixedw = P.noisewindowfixed;
    float p2[K];
#pragma unroll
    for (int k = 0; k < K; k++) p1[k] = 0.f;
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
      const float off = pass ? 0.f : 140.f;
      const int fx = pass ? fixedw : -1;
#pragma unroll
      for (int k = 0; k < K; k++) dev_noise_term1(tid + k * nt, L[k] - p1[k], off, S, ns);
      __syncthreads();
      PHASE_MARK();   // 5 / 8 terms
      if (threadIdx.x < 5 * R) dev_noise_scan3(n, sm_cta + (threadIdx.x / 5) * row_floats + (threadIdx.x % 5) * ns);
      __syncthreads();
      PHASE_MARK();   // 6 / 9 scan
      if (K >= 2) {
#pragma unroll
        for (int k = 0; k + 1 < K; k += 2) {
          const float2 r = regress_pair<K * PSY3_THREADS + 4>(bark, bfe, ffe, S, tid + k * nt, tid + (k + 1) * nt, off, fx);
          p2[k] = r.x; p2[k + 1] = r.y;
        }
      } else {
#pragma unroll
        for (int k = 0; k < K; k++) p2[k] = regress_core<K * PSY3_THREADS + 4>(bark, bfe, ffe, S, tid + k * nt, off, fx);
      }
      if (pass == 0) {
#pragma unroll
        for (int k = 0; k < K; k++) p1[k] = p2[k];
        __syncthreads();                                 // the sums are overwritten by the second pass' terms
        PHASE_MARK();   // 7 regress 1
      }
    }
    MixConst MC;
    MC.noisemaxsupp = P.noisemaxsupp; MC.toneatt = P.tone_masteratt[1]; MC.m_val = P.m_val;
    MC.att = att;
    const float *noff = P.noiseoffset + n;             // offset_select 1
    const float *athp = P.ath, *compand = P.noisecompand;
    const short *bin_grp = P.bin_grp;
#pragma unroll
    for (int k = 0; k < K && !spare; k++) {
      const int i = tid + k * nt;
      const MixOut o = final_mix_val(p2[k], L[k], p1[k], __ldg(noff + i), __ldg(athp + i),
                                     grp_min[__ldg(bin_grp + i)], compand, MC, __ldcs(gm + i));
      __stcs(A.logmask + (size_t)row * n + i, o.logmask);
      __stcs(A.mdct_out + (size_t)row * n + i, o.m);
      if (DBG && A.tap_noise) A.tap_noise[(size_t)row * n + i] = o.nz;
      if (DBG && A.tap_tone) A.tap_tone[(size_t)row * n + i] = o.tn;
    }
    if (tid == 0 && (row % ch) == 0) A.ampmax_out[blk] = g;   // lib/mapping0.c:576
    __syncthreads();
    PHASE_MARK();   // 10 regress 2 + final + mix
#undef PHASE_MARK
  }
}

}  // namespace vb200
