// vb200_kernels.cuh — hand-written sm_90a kernels for the libvorbis per-block
// DSP path (window, MDCT, real FFT, log spectra, noise/tone masks, mix).
//
// Numerics contract: every output value is produced by the same sequence of
// IEEE-754 fp32 (and, where the reference promotes, fp64) operations as the
// reference C code, only scheduled in parallel.  The TU is compiled with
// -fmad=false (no FMA contraction), default -prec-div/-prec-sqrt, no fast-math,
// so results are bit-identical to the reference built with -ffp-contract=off.
// Each stage is a set of independent work items (see DESIGN.md); items are
// distributed over the threads of one CTA, data lives in shared memory.
//
// Reference citations are to the xiph/vorbis tree (libvorbis 1.3.7).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

namespace vb200 {

#define VB_C1 .92387953251128675613F   /* cos(pi/8),  lib/mdct.h:47 */
#define VB_C2 .70710678118654752441F   /* cos(2pi/8), lib/mdct.h:46 */
#define VB_C3 .38268343236508977175F   /* cos(3pi/8), lib/mdct.h:45 */
#define VB_NEGINF (-9999.f)            /* lib/psy.c:31 */

struct XformDev {
  int N, log2n, nst, nf;
  int fac[8];           // factors in drfti1 order (lib/smallft.c:37)
  int stage_off[8];     // float2 offsets into stage_tw
  float scale;          // 4/N
  const float  *trig;   // N + N/4
  const int    *bitrev; // N/4
  const float2 *stage_tw;
  const float  *win;    // N/2
  const float  *wa;     // N
};

struct WinDev {         // both half windows, for lW/nW selection (lib/window.c:2102)
  int N[2];
  const float *win[2];
};

struct PsyDev {
  int n, total, linesper, firstoc, shiftoc;
  int noisewindowfixed, bark_first_extra, fixed_first_extra;
  int nruns, ngrp, tail_lin0;
  float ath_adjatt, ath_maxatt, tone_abs_limit, noisemaxsupp, max_curve_dB, m_val;
  float tone_masteratt[3];
  const float *ath;          // [n]
  const int   *octave;       // [n]
  const int   *bark;         // [n]
  const float *tonecurves;   // [17][8][58]
  const float *noiseoffset;  // [3][n]
  const float *noisecompand; // [40]
  const int4  *runinfo;      // [nruns] (lo, hi, octave[hi]-firstoc, band)
  const int4  *grps;         // [ngrp]  (pos0,pos1,lin0,lin1)
  const int2  *cls_run;      // runs grouped by residue class, (run id, oc-firstoc), sorted by oc
  const int2  *slot_rng;     // [total] candidate range in cls_run for every seed slot
  int linesper_log2;
  const short *bin_grp;      // [n] group of every bin (ngrp = the tail bins)
  const int4  *runrec;       // [nruns] class-ordered: lo|hi<<16, oc-firstoc, band, bits(ath[hi])
  const int   *long_grp;     // [nlong] groups folded cooperatively
  int nlong;
  const int *cls_off;        // [L+1] (device) class c owns cls_run[cls_off[c] .. cls_off[c+1])
  int max_cls_len;           // longest class
};

// arguments of the fused psy kernels (k_phaseA_psy3 and the generic k_phaseA_psy)
struct PsyArgs {
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
  unsigned long long *dbg_cycles;   // optional [16]: per-phase SM cycles summed over rows (thread 0 of each CTA)
};

// ------------------------------------------------------------------------
__device__ __forceinline__ float todB_dev(float x) {           // lib/scales.h:43-51
  const unsigned int u = __float_as_uint(x) & 0x7fffffffu;
  return __uint2float_rn(u) * 7.17711438e-7f - 764.6161886f;
}
__device__ __forceinline__ float add345(float x) {             // "+ .345" is a double add
  return (float)((double)x + .345);
}

// 32-bit shared-window addressing: one cvta per array, then ld/st.shared with register offsets
// (keeps the compiler from re-deriving the shared base inside predicated hot loops)
#ifndef VB200_EMU
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float lds_f32(unsigned a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a)); return v; }
__device__ __forceinline__ int lds_s32(unsigned a) { int v; asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ int4 lds_v4(unsigned a) { int4 v; asm volatile("ld.shared.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)); return v; }
__device__ __forceinline__ float4 lds_f4(unsigned a) { float4 v; asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a)); return v; }
__device__ __forceinline__ void sts_f4(unsigned a, float4 v) { asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" :: "r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory"); }
__device__ __forceinline__ void sts_f32(unsigned a, float v) { asm volatile("st.shared.f32 [%0], %1;" :: "r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_s32(unsigned a, int v) { asm volatile("st.shared.s32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void named_bar_sync(int barid, int nt) { asm volatile("bar.sync %0, %1;" :: "r"(barid), "r"(nt) : "memory"); }
// predicated forms (the access is skipped, and `old` is returned, when p is false): keep data-dependent
// branches out of loops whose lanes would otherwise diverge on every iteration
__device__ __forceinline__ float lds_f32_if(unsigned a, float old, bool p) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q ld.shared.f32 %0, [%1];\n\t}" : "+f"(old) : "r"(a), "r"((int)p));
  return old;
}
__device__ __forceinline__ int lds_s32_if(unsigned a, int old, bool p) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q ld.shared.s32 %0, [%1];\n\t}" : "+r"(old) : "r"(a), "r"((int)p));
  return old;
}
__device__ __forceinline__ void sts_s32_if(unsigned a, int v, bool p) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q st.shared.s32 [%0], %1;\n\t}" :: "r"(a), "r"(v), "r"((int)p) : "memory");
}
__device__ __forceinline__ void sts_f32_if(unsigned a, float v, bool p) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q st.shared.f32 [%0], %1;\n\t}" :: "r"(a), "f"(v), "r"((int)p) : "memory");
}
// cp.async: 16 bytes global -> shared without passing through registers (SASS: LDGSTS)
__device__ __forceinline__ void cp_async16(unsigned dst, const void *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }
#else   // host emulation build (tools/cuemu, development aid): "shared addresses" are offsets into the CTA's buffer
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)((const unsigned char *)p - cuemu::dyn_smem()); }
__device__ __forceinline__ float lds_f32(unsigned a) { return *reinterpret_cast<const float *>(cuemu::dyn_smem() + a); }
__device__ __forceinline__ int lds_s32(unsigned a) { return *reinterpret_cast<const int *>(cuemu::dyn_smem() + a); }
__device__ __forceinline__ int4 lds_v4(unsigned a) { return *reinterpret_cast<const int4 *>(cuemu::dyn_smem() + a); }
__device__ __forceinline__ float4 lds_f4(unsigned a) { return *reinterpret_cast<const float4 *>(cuemu::dyn_smem() + a); }
__device__ __forceinline__ void sts_f4(unsigned a, float4 v) { *reinterpret_cast<float4 *>(cuemu::dyn_smem() + a) = v; }
__device__ __forceinline__ void sts_f32(unsigned a, float v) { *reinterpret_cast<float *>(cuemu::dyn_smem() + a) = v; }
__device__ __forceinline__ void sts_s32(unsigned a, int v) { *reinterpret_cast<int *>(cuemu::dyn_smem() + a) = v; }
__device__ __forceinline__ void named_bar_sync(int barid, int nt) { cuemu_named_barrier(barid, nt); }
__device__ __forceinline__ void prefetch_l2(const void *) {}
__device__ __forceinline__ void cp_async16(unsigned dst, const void *src) { memcpy(cuemu::dyn_smem() + dst, src, 16); }
__device__ __forceinline__ void cp_async_commit() {}
__device__ __forceinline__ void cp_async_wait_all() {}
__device__ __forceinline__ float lds_f32_if(unsigned a, float old, bool p) { return p ? lds_f32(a) : old; }
__device__ __forceinline__ void sts_f32_if(unsigned a, float v, bool p) { if (p) sts_f32(a, v); }
__device__ __forceinline__ int lds_s32_if(unsigned a, int old, bool p) { return p ? lds_s32(a) : old; }
__device__ __forceinline__ void sts_s32_if(unsigned a, int v, bool p) { if (p) sts_s32(a, v); }
#endif

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------
// MDCT pieces.  x points at n2 = N/2 floats in shared memory.

// mdct_butterflies (lib/mdct.c:316-336): radix-2 stages (butterfly_first /
// butterfly_generic, :216-314) then the fixed 32/16/8-point flies (:93-214),
// each level spread over all threads: level L has N/8 independent items.
// NC = block size as a compile-time constant (0: read it from X at run time).  With NC known
// every loop bound, shift and FFT pass shape below folds to a constant and the stage loops unroll.
template <int NC> struct XLog2 { static constexpr int v = 1 + XLog2<NC / 2>::v; };
template <> struct XLog2<1> { static constexpr int v = 0; };
template <> struct XLog2<0> { static constexpr int v = 0; };

// Padded index for the output of the last butterfly level when it goes to a separate buffer: the
// bit-reverse stage gathers float2 at strides of 32 floats and more (16-way bank conflicts on the
// plain layout); two extra floats per 32 and per 512 spread those gathers - and the level's own
// stores - over all banks (checked for n2 = 1024: both gathers and the stores are conflict free).
__device__ __forceinline__ int fly_pad(int a) { return a + 2 * (a >> 5) + 2 * (a >> 9); }

// mdct_butterfly_8 (lib/mdct.c:93-115) on registers: v0 = x0..x3, v1 = x4..x7
__device__ __forceinline__ void dev_fly8(const float4 v0, const float4 v1, float4 &o0, float4 &o1) {
  const float s62 = v1.z + v0.z, d62 = v1.z - v0.z;
  const float s40 = v1.x + v0.x, d40 = v1.x - v0.x;
  const float d51 = v1.y - v0.y, d73 = v1.w - v0.w;
  const float s51 = v1.y + v0.y, s73 = v1.w + v0.w;
  o1.z = s62 + s40;  o1.x = s62 - s40;
  o0.x = d62 + d51;  o0.z = d62 - d51;
  o0.w = d73 + d40;  o0.y = d73 - d40;
  o1.w = s73 + s51;  o1.y = s73 - s51;
}

// one radix-2 butterfly of mdct_butterfly_generic / _first (lib/mdct.c:216-314): hi <- hi + lo, lo <- (hi - lo) * t
__device__ __forceinline__ void fly_bf(float2 &hi, float2 &lo, float2 t) {
  const float r0 = hi.x - lo.x, r1 = hi.y - lo.y;
  hi = make_float2(hi.x + lo.x, hi.y + lo.y);
  lo = make_float2(r1 * t.y + r0 * t.x, r1 * t.x - r0 * t.y);
}

// The item of the 32-point fly's first level (lib/mdct.c:152-209; see the loop in dev_butterflies, which keeps its
// own copy so that the kernels without paired levels compile as before) on registers: hi = (30-2q), lo = (14-2q).
__device__ __forceinline__ void fly32_bf(float2 &hi, float2 &lo, int q) {
  const float dxp = hi.x - lo.x, dxn = lo.x - hi.x, dyp = hi.y - lo.y, dyn = lo.y - hi.y;
  const float r0 = q >= 5 ? dxn : dxp;
  const float r1 = q >= 4 ? dyn : dyp;
  // odd q: o0 = r0*k00 + r1*k01, o1 = r0*k10 + r1*k11
  const bool q15 = (q == 1) | (q == 7);                // k00 = k11 = C1 there, C3 for q = 3, 5
  const float k00 = q15 ? VB_C1 : VB_C3;
  const float k3 = q15 ? VB_C3 : VB_C1;                // the other constant, sign by case
  const float k01 = q < 4 ? -k3 : k3;
  const float k10 = q < 4 ? k3 : -k3;
  const float A0 = r0 * k00 + r1 * k01;
  const float A1 = r0 * k10 + r1 * k00;
  // q = 2: (r0 - r1)*C2, (r0 + r1)*C2;  q = 6: (r1 + r0)*C2, (r1 - r0)*C2
  const float B0 = (q == 2 ? r0 - r1 : r1 + r0) * VB_C2;
  const float B1 = (q == 2 ? r0 + r1 : r1 - r0) * VB_C2;
  // q = 0: r0, r1;  q = 4: r1, r0
  const float T0 = q == 0 ? r0 : r1, T1 = q == 0 ? r1 : r0;
  const bool odd = q & 1, triv = (q & 3) == 0;
  const float o0 = odd ? A0 : (triv ? T0 : B0);
  const float o1 = odd ? A1 : (triv ? T1 : B1);
  hi = make_float2(hi.x + lo.x, hi.y + lo.y);
  lo = make_float2(o0, o1);
}

// Levels s and s+1 of the butterflies in one shared-memory pass (NC > 0; level nst is the 32-point fly's first
// level).  Level s pairs (P-2-2q, P/2-2-2q) in a block of P values; level s+1 does the same in each half.  Level-s
// items q and q + P/8 touch exactly the four pairs that level s+1 item q touches in the two halves, so one thread
// takes those four pairs through both levels in registers.
template <int NC>
__device__ __forceinline__ void dev_fly_pair(const XformDev &X, float *x, int s, int tid, int nt) {
  constexpr int log2n = XLog2<NC>::v, nst = log2n - 6, n2 = NC >> 1;
  const int P = n2 >> s, e = P >> 3;
  const int sh = log2n - 4 - s;                  // log2(P/8)
  const float2 *tw = X.stage_tw + X.stage_off[s];
  for (int u = tid; u < (n2 >> 3); u += nt) {
    const int blk = u >> sh, q = u & (e - 1);
    float *xb = x + P * blk;
    float2 *pu1 = reinterpret_cast<float2 *>(xb + P - 2 - 2 * q);
    float2 *pl1 = reinterpret_cast<float2 *>(xb + (P >> 1) - 2 - 2 * q);
    float2 *pu2 = reinterpret_cast<float2 *>(xb + 3 * (P >> 2) - 2 - 2 * q);
    float2 *pl2 = reinterpret_cast<float2 *>(xb + (P >> 2) - 2 - 2 * q);
    float2 u1 = *pu1, l1 = *pl1, u2 = *pu2, l2 = *pl2;
    fly_bf(u1, l1, __ldg(tw + q));
    fly_bf(u2, l2, __ldg(tw + q + e));
    if (s + 1 < nst) {
      const float2 t = __ldg(X.stage_tw + X.stage_off[s + 1] + q);
      fly_bf(u1, u2, t);
      fly_bf(l1, l2, t);
    } else {
      fly32_bf(u1, u2, q);
      fly32_bf(l1, l2, q);
    }
    *pu1 = u1; *pl1 = l1; *pu2 = u2; *pl2 = l2;
  }
}

// PAIRED (NC > 0 only): the generic levels and the 32-point fly's first level two per pass (dev_fly_pair)
template <int NC, bool PAIRED = false>
__device__ __forceinline__ void dev_butterflies(const XformDev &X, float *x, int tid, int nt, float *padbuf = nullptr) {
  const int N = NC ? NC : X.N;
  const int log2n = NC ? XLog2<NC>::v : X.log2n;
  const int nst = log2n - 6;
  const int n2 = N >> 1;
  const int items = n2 >> 2;
  if constexpr (PAIRED) {
    static_assert(NC > 0, "paired butterflies need the block size at compile time");
#pragma unroll
    for (int s = 0; s + 1 <= nst; s += 2) {
      dev_fly_pair<NC>(X, x, s, tid, nt);
      __syncthreads();
    }
  } else {
#pragma unroll
  for (int s = 0; s < nst; s++) {
    const int P = n2 >> s;
    const int lq = P >> 2;                       // items per sub-block (power of two)
    const int sh = log2n - 3 - s;                // log2(lq)
    const float2 *tw = X.stage_tw + X.stage_off[s];
    for (int u = tid; u < items; u += nt) {
      const int blk = u >> sh, q = u & (lq - 1);
      float *xb = x + P * blk;
      const int a = P - 2 - 2 * q, b = (P >> 1) - 2 - 2 * q;
      const float2 t = __ldg(tw + q);
      const float2 hi = *reinterpret_cast<float2 *>(xb + a);
      const float2 lo = *reinterpret_cast<float2 *>(xb + b);
      const float r0 = hi.x - lo.x, r1 = hi.y - lo.y;
      *reinterpret_cast<float2 *>(xb + a) = make_float2(hi.x + lo.x, hi.y + lo.y);
      *reinterpret_cast<float2 *>(xb + b) = make_float2(r1 * t.y + r0 * t.x, r1 * t.x - r0 * t.y);
    }
    __syncthreads();
  }
  }
  if (!PAIRED || ((nst + 1) & 1)) {   // paired: an odd level count leaves the 32-point level on its own
  // 32-point fly, first level (lib/mdct.c:152-209): item q pairs (30-2q) with (14-2q).  The eight cases of
  // the reference differ in which difference they take (a-b or b-a: both are computed, x-x is +0 either way,
  // so one is not the negation of the other) and in the rotation: none (q=0,4), (r0 -/+ r1)*C2 (q=2,6), or
  // r0*k + r1*k' with signed constants (q odd; a - b*c == a + b*(-c) exactly).  All lanes run the three
  // forms and select: the eight-way switch on q cost eight serialised paths per warp.
  for (int u = tid; u < items; u += nt) {
    float *xc = x + 32 * (u >> 3);
    const int q = u & 7;
    const int a = 30 - 2 * q, b = 14 - 2 * q;
    const float2 hi = *reinterpret_cast<float2 *>(xc + a);
    const float2 lo = *reinterpret_cast<float2 *>(xc + b);
    const float dxp = hi.x - lo.x, dxn = lo.x - hi.x, dyp = hi.y - lo.y, dyn = lo.y - hi.y;
    const float r0 = q >= 5 ? dxn : dxp;
    const float r1 = q >= 4 ? dyn : dyp;
    // odd q: o0 = r0*k00 + r1*k01, o1 = r0*k10 + r1*k11
    const bool q15 = (q == 1) | (q == 7);                // k00 = k11 = C1 there, C3 for q = 3, 5
    const float k00 = q15 ? VB_C1 : VB_C3;
    const float k3 = q15 ? VB_C3 : VB_C1;                // the other constant, sign by case
    const float k01 = q < 4 ? -k3 : k3;
    const float k10 = q < 4 ? k3 : -k3;
    const float A0 = r0 * k00 + r1 * k01;
    const float A1 = r0 * k10 + r1 * k00;
    // q = 2: (r0 - r1)*C2, (r0 + r1)*C2;  q = 6: (r1 + r0)*C2, (r1 - r0)*C2
    const float B0 = (q == 2 ? r0 - r1 : r1 + r0) * VB_C2;
    const float B1 = (q == 2 ? r0 + r1 : r1 - r0) * VB_C2;
    // q = 0: r0, r1;  q = 4: r1, r0
    const float T0 = q == 0 ? r0 : r1, T1 = q == 0 ? r1 : r0;
    const bool odd = q & 1, triv = (q & 3) == 0;
    const float o0 = odd ? A0 : (triv ? T0 : B0);
    const float o1 = odd ? A1 : (triv ? T1 : B1);
    *reinterpret_cast<float2 *>(xc + a) = make_float2(hi.x + lo.x, hi.y + lo.y);
    *reinterpret_cast<float2 *>(xc + b) = make_float2(o0, o1);
  }
  __syncthreads();
  }
  // 16-point fly (lib/mdct.c:117-147) with its two 8-point flies (:93-115): one item per 16 values, all in
  // registers - one shared-memory round trip and one barrier instead of two, and no per-lane case split
  for (int u = tid; u < (n2 >> 4); u += nt) {
    float4 *p = reinterpret_cast<float4 *>(x + 16 * u);
    float4 v0 = p[0], v1 = p[1], v2 = p[2], v3 = p[3];   // x0..x3, x4..x7, x8..x11, x12..x15
    {
      const float a = v0.y - v2.y, b = v0.x - v2.x;      // x1-x9, x0-x8
      v2.x = v2.x + v0.x; v2.y = v2.y + v0.y;
      v0.x = (a + b) * VB_C2; v0.y = (a - b) * VB_C2;
    }
    {
      const float o0 = v0.w - v2.w, o1 = v2.z - v0.z;    // x3-x11, x10-x2
      v2.z = v2.z + v0.z; v2.w = v2.w + v0.w;
      v0.z = o0; v0.w = o1;
    }
    {
      const float a = v3.x - v1.x, b = v3.y - v1.y;      // x12-x4, x13-x5
      v3.x = v3.x + v1.x; v3.y = v3.y + v1.y;
      v1.x = (a - b) * VB_C2; v1.y = (a + b) * VB_C2;
    }
    {
      const float o0 = v3.z - v1.z, o1 = v3.w - v1.w;    // x14-x6, x15-x7
      v3.z = v3.z + v1.z; v3.w = v3.w + v1.w;
      v1.z = o0; v1.w = o1;
    }
    float4 o0, o1, o2, o3;
    dev_fly8(v0, v1, o0, o1);
    dev_fly8(v2, v3, o2, o3);
    if (padbuf) {
      float2 *q = reinterpret_cast<float2 *>(padbuf + fly_pad(16 * u));
      q[0] = make_float2(o0.x, o0.y); q[1] = make_float2(o0.z, o0.w);
      q[2] = make_float2(o1.x, o1.y); q[3] = make_float2(o1.z, o1.w);
      float2 *r = reinterpret_cast<float2 *>(padbuf + fly_pad(16 * u + 8));
      r[0] = make_float2(o2.x, o2.y); r[1] = make_float2(o2.z, o2.w);
      r[2] = make_float2(o3.x, o3.y); r[3] = make_float2(o3.z, o3.w);
    } else {
      p[0] = o0; p[1] = o1; p[2] = o2; p[3] = o3;
    }
  }
  __syncthreads();
}

// mdct_bitreverse (lib/mdct.c:346-394): item m reads two complex values of the
// upper half w[n2..N) through bitrev[] and writes four values of w[0..n2).
template <int NC>
__device__ __forceinline__ void dev_bitreverse(const XformDev &X, float *w, int tid, int nt, const float *padbuf = nullptr) {
  const int N = NC ? NC : X.N, n2 = N >> 1;
  const float2 *T = reinterpret_cast<const float2 *>(X.trig + N);
  const int2 *br = reinterpret_cast<const int2 *>(X.bitrev);
  const float *x = w + n2;
  for (int m = tid; m < (N >> 3); m += nt) {
    const int2 b = __ldg(br + m);
    const float2 t = __ldg(T + m);
    const float2 x0 = padbuf ? *reinterpret_cast<const float2 *>(padbuf + fly_pad(b.x)) : *reinterpret_cast<const float2 *>(x + b.x);
    const float2 x1 = padbuf ? *reinterpret_cast<const float2 *>(padbuf + fly_pad(b.y)) : *reinterpret_cast<const float2 *>(x + b.y);
    const float r0 = x0.y - x1.y;
    const float r1 = x0.x + x1.x;
    const float r2 = r1 * t.x + r0 * t.y;
    const float r3 = r1 * t.y - r0 * t.x;
    const float h0 = (x0.y + x1.y) * .5f;
    const float h1 = (x0.x - x1.x) * .5f;
    *reinterpret_cast<float2 *>(w + 2 * m) = make_float2(h0 + r2, h1 + r3);
    *reinterpret_cast<float2 *>(w + n2 - 2 * m - 2) = make_float2(h0 - r2, r3 - h1);
  }
  __syncthreads();
}

// Forward MDCT of the N samples at `in` (shared memory, read-only) using the N
// floats of scratch at `w`; writes N/2 coefficients to `out` (global or shared).
// mdct_forward, lib/mdct.c:492-562.
// padbuf: optional n2 + n2/16 + n2/256 + 8 floats of scratch (16-byte aligned) for the padded hand-over
// between the butterflies and the bit-reverse stage
// PAIRED: the butterflies two levels per pass (dev_butterflies), for the templated transform kernel
template <int NC, bool PAIRED = false>
__device__ __forceinline__ void dev_mdct_forward(const XformDev &X, const float *in, float *w,
                                                 float *out, int tid, int nt, float *padbuf = nullptr) {
  const int N = NC ? NC : X.N, n2 = N >> 1, n4 = N >> 2, n16 = N >> 4;
  float *w2 = w + n2;
  const float2 *Tf = reinterpret_cast<const float2 *>(X.trig);
  for (int p = tid; p < n4; p += nt) {
    const float2 t = __ldg(Tf + (n4 - 1 - p));     // trig[n2-2p-2], trig[n2-2p-1]
    float r0, r1;
    // x0[0],x0[2] and x1[0],x1[2] via two aligned 128-bit loads (x1 sits at an odd offset)
    if (p < n16) {
      const float4 a = *reinterpret_cast<const float4 *>(in + n2 + n4 - 4 * (p + 1));
      const float4 b = *reinterpret_cast<const float4 *>(in + n2 + n4 + 4 * p);
      r0 = a.z + b.y;
      r1 = a.x + b.w;
    } else if (p < n4 - n16) {
      const float4 a = *reinterpret_cast<const float4 *>(in + n2 + n4 - 4 * (p + 1));
      const float4 b = *reinterpret_cast<const float4 *>(in + 4 * (p - n16));
      r0 = a.z - b.y;
      r1 = a.x - b.w;
    } else {
      const float4 a = *reinterpret_cast<const float4 *>(in + N - 4 * (p - (n4 - n16) + 1));
      const float4 b = *reinterpret_cast<const float4 *>(in + 4 * (p - n16));
      r0 = -a.z - b.y;
      r1 = -a.x - b.w;
    }
    *reinterpret_cast<float2 *>(w2 + 2 * p) = make_float2(r1 * t.y + r0 * t.x, r1 * t.x - r0 * t.y);
  }
  __syncthreads();
  dev_butterflies<NC, PAIRED>(X, w2, tid, nt, padbuf);
  dev_bitreverse<NC>(X, w, tid, nt, padbuf);
  const float2 *Tp = reinterpret_cast<const float2 *>(X.trig + n2);
  const float scale = X.scale;
  for (int i = tid; i < n4; i += nt) {
    const float2 v = *reinterpret_cast<const float2 *>(w + 2 * i);
    const float2 t = __ldg(Tp + i);
    out[i]          = (v.x * t.x + v.y * t.y) * scale;
    out[n2 - 1 - i] = (v.x * t.y - v.y * t.x) * scale;
  }
}

// Inverse MDCT: N/2 coefficients at `in` (shared or global, read-only) -> N
// samples in the shared buffer `out` (N floats).  mdct_backward, lib/mdct.c:396-490.
// The result layout is [A | -rev(A) | rev(B) | B] (see DESIGN.md).
template <int NC>
__device__ __forceinline__ void dev_mdct_backward(const XformDev &X, const float *in, float *out,
                                                  int tid, int nt) {
  const int N = NC ? NC : X.N, n2 = N >> 1, n4 = N >> 2, n16 = N >> 4;
  const float *T = X.trig;
  for (int u = tid; u < 2 * n16; u += nt) {
    if (u < n16) {
      const int j = u;
      const float *iX = in + n2 - 7 - 8 * j;
      const float4 t = __ldg(reinterpret_cast<const float4 *>(T + n4 + 4 * j));
      float4 o;
      o.x = -iX[2] * t.w - iX[0] * t.z;
      o.y =  iX[0] * t.w - iX[2] * t.z;
      o.z = -iX[6] * t.y - iX[4] * t.x;
      o.w =  iX[4] * t.y - iX[6] * t.x;
      *reinterpret_cast<float4 *>(out + n2 + n4 - 4 * (j + 1)) = o;
    } else {
      const int j = u - n16;
      const float *iX = in + n2 - 8 - 8 * j;
      const float4 t = __ldg(reinterpret_cast<const float4 *>(T + n4 - 4 * (j + 1)));
      float4 o;
      o.x = iX[4] * t.w + iX[6] * t.z;
      o.y = iX[4] * t.z - iX[6] * t.w;
      o.z = iX[0] * t.y + iX[2] * t.x;
      o.w = iX[0] * t.x - iX[2] * t.y;
      *reinterpret_cast<float4 *>(out + n2 + n4 + 4 * j) = o;
    }
  }
  __syncthreads();
  dev_butterflies<NC>(X, out + n2, tid, nt);
  dev_bitreverse<NC>(X, out, tid, nt);
  const float2 *Tp = reinterpret_cast<const float2 *>(X.trig + n2);
  // item k: A[n4-1-k] = re*T1 - im*T0, B[k] = -(re*T0 + im*T1)
  for (int k = tid; k < n4; k += nt) {
    const float2 v = *reinterpret_cast<const float2 *>(out + 2 * k);
    const float2 t = __ldg(Tp + k);
    out[n2 + n4 - 1 - k] = v.x * t.y - v.y * t.x;
    out[n2 + n4 + k]     = -(v.x * t.x + v.y * t.y);
  }
  __syncthreads();
  for (int k = tid; k < n4; k += nt) {
    const float a = out[n2 + n4 - 1 - k];
    out[n4 - 1 - k] = a;
    out[n4 + k] = -a;
  }
  __syncthreads();
  for (int k = tid; k < n4; k += nt) out[n2 + n4 - 1 - k] = out[n2 + n4 + k];
  __syncthreads();
}

// ------------------------------------------------------------------------
// Real FFT forward (drftf1 + dradf4 + dradf2, lib/smallft.c:572-631, 168-268,
// 113-166).  One pass per factor, last factor first; each pass reads cc and
// writes ch.  Items: for every k<l1, the i=0 column, the twiddled interior
// pairs i=2,4,.., and the i=ido-1 column.
//
// Layout of the ping-pong buffers: logical element e of a pass output lives at float index
// fft_idx(e) = pad(e + 1), pad(a) = a + 2*(a >> 5).  The shift by one float puts FFTPACK's (re,im)
// pairs (2k-1,2k) on 8-byte boundaries (one 64-bit access per pair); the two spare floats per 32
// spread the stride-4*ido stores of the small-ido passes over the banks (tools/fft_bank_sim.py:
// 2344 -> 1315 wavefronts per N=2048 row).  Pairs never straddle a pad (they start on an even index).
// The very first pass reads the caller's plain, unshifted input.
__device__ __forceinline__ int fft_idx(int e) { const int a = e + 1; return a + 2 * (a >> 5); }
__host__ __device__ constexpr int fft_buf_floats(int N) { return N + (N >> 4) + 16; }

template <bool FIRST>
__device__ __forceinline__ int fft_rd(int e) { return FIRST ? e : fft_idx(e); }

template <bool FIRST>
__device__ __forceinline__ void dev_fft_pass4(int ido, int l1, const float *cc, float *ch,
                                              const float *w1, const float *w2, const float *w3,
                                              int tid, int nt) {
  const float hsqt2 = .70710678118654752f;
  const int t0 = l1 * ido;
  if (ido == 1) {
    for (int k = tid; k < l1; k += nt) {
      const float c0 = cc[fft_rd<FIRST>(k)], c1 = cc[fft_rd<FIRST>(k + t0)];
      const float c2 = cc[fft_rd<FIRST>(k + 2 * t0)], c3 = cc[fft_rd<FIRST>(k + 3 * t0)];
      const float tr1 = c1 + c3, tr2 = c0 + c2;
      const int o = 4 * k;
      ch[fft_idx(o)] = tr1 + tr2;                                                      // o[0]
      *reinterpret_cast<float2 *>(ch + fft_idx(o + 1)) = make_float2(c0 - c2, c3 - c1); // o[2*ido-1], o[2*ido]
      ch[fft_idx(o + 3)] = tr2 - tr1;                                                  // o[4*ido-1]
    }
    return;
  }
  // ido >= 4 here (ido runs 1, 4, 16, ..).  l1*ido/2 work items of eight reals each: the first l1 are the two
  // un-twiddled columns (i = 0 and i = ido-1) of one k, the others one twiddled pair (k, i).  With the
  // special columns on the leading threads a warp runs ONE of the two code paths whenever l1 >= 32.
  // Padded addresses: fft_idx(e + D) = fft_idx(e) + D + D/16 whenever 32 | D, so the four inputs of an item
  // (t0 apart) and the output pairs 2*ido apart share one index computation each.
  const int half = ido >> 1, hm1 = half - 1;
  const int T = l1 * half;
  const bool t0al = FIRST || (t0 & 31) == 0, idal = ((2 * ido) & 31) == 0;
  const int pt0 = FIRST ? t0 : t0 + (t0 >> 4), p2 = 2 * ido + ((2 * ido) >> 4);
  for (int v = tid; v < T; v += nt) {
    if (v < l1) {
      const int k = v;
      const int c0 = k * ido;
      const int o = 4 * k * ido;
      {
        const int r0 = fft_rd<FIRST>(c0);
        const int r1 = t0al ? r0 + pt0 : fft_idx(c0 + t0), r2 = t0al ? r1 + pt0 : fft_idx(c0 + 2 * t0);
        const int r3 = t0al ? r2 + pt0 : fft_idx(c0 + 3 * t0);
        const float a0 = cc[r0], a1 = cc[r1], a2 = cc[r2], a3 = cc[r3];
        const float tr1 = a1 + a3;
        const float tr2 = a0 + a2;
        ch[fft_idx(o)]               = tr1 + tr2;
        ch[fft_idx(o + 4 * ido - 1)] = tr2 - tr1;
        *reinterpret_cast<float2 *>(ch + fft_idx(o + 2 * ido - 1)) = make_float2(a0 - a2, a3 - a1);
      }
      {
        const int e = c0 + ido - 1;
        const int r0 = fft_rd<FIRST>(e);
        const int r1 = t0al ? r0 + pt0 : fft_idx(e + t0), r2 = t0al ? r1 + pt0 : fft_idx(e + 2 * t0);
        const int r3 = t0al ? r2 + pt0 : fft_idx(e + 3 * t0);
        const float a0 = cc[r0], a1 = cc[r1], a2 = cc[r2], a3 = cc[r3];
        const float ti1 = -hsqt2 * (a1 + a3);
        const float tr1 =  hsqt2 * (a1 - a3);
        const int s1 = fft_idx(o + ido - 1), s3 = idal ? s1 + p2 : fft_idx(o + 3 * ido - 1);
        *reinterpret_cast<float2 *>(ch + s1) = make_float2(tr1 + a0, ti1 - a2);   // o[ido-1], o[ido]
        *reinterpret_cast<float2 *>(ch + s3) = make_float2(a0 - tr1, ti1 + a2);   // o[3ido-1], o[3ido]
      }
    } else {
      const int g = v - l1;
      const int k = g / hm1, ii = 1 + g - k * hm1;     // hm1 is a compile-time constant in the templated kernels
      const int c0 = k * ido;
      const int o = 4 * k * ido;
      const int i = 2 * ii;
      const float wa1r = __ldg(w1 + i - 2), wa1i = __ldg(w1 + i - 1);
      const float wa2r = __ldg(w2 + i - 2), wa2i = __ldg(w2 + i - 1);
      const float wa3r = __ldg(w3 + i - 2), wa3i = __ldg(w3 + i - 1);
      const int r0 = fft_rd<FIRST>(c0 + i - 1);
      const int r1 = t0al ? r0 + pt0 : fft_idx(c0 + t0 + i - 1), r2 = t0al ? r1 + pt0 : fft_idx(c0 + 2 * t0 + i - 1);
      const int r3 = t0al ? r2 + pt0 : fft_idx(c0 + 3 * t0 + i - 1);
      const float2 a0 = *reinterpret_cast<const float2 *>(cc + r0);
      const float2 a1 = *reinterpret_cast<const float2 *>(cc + r1);
      const float2 a2 = *reinterpret_cast<const float2 *>(cc + r2);
      const float2 a3 = *reinterpret_cast<const float2 *>(cc + r3);
      const float cr2 = wa1r * a1.x + wa1i * a1.y;
      const float ci2 = wa1r * a1.y - wa1i * a1.x;
      const float cr3 = wa2r * a2.x + wa2i * a2.y;
      const float ci3 = wa2r * a2.y - wa2i * a2.x;
      const float cr4 = wa3r * a3.x + wa3i * a3.y;
      const float ci4 = wa3r * a3.y - wa3i * a3.x;
      const float tr1 = cr2 + cr4, tr4 = cr4 - cr2;
      const float ti1 = ci2 + ci4, ti4 = ci2 - ci4;
      const float ti2 = a0.y + ci3, ti3 = a0.y - ci3;
      const float tr2 = a0.x + cr3, tr3 = a0.x - cr3;
      const int ic = 2 * ido - i;
      const int o1 = fft_idx(o + i - 1), o2 = fft_idx(o + ic - 1);
      const int o3 = idal ? o1 + p2 : fft_idx(o + 2 * ido + i - 1), o4 = idal ? o2 + p2 : fft_idx(o + 2 * ido + ic - 1);
      *reinterpret_cast<float2 *>(ch + o1) = make_float2(tr1 + tr2, ti1 + ti2);
      *reinterpret_cast<float2 *>(ch + o2) = make_float2(tr3 - ti4, tr4 - ti3);
      *reinterpret_cast<float2 *>(ch + o3) = make_float2(ti4 + tr3, tr4 + ti3);
      *reinterpret_cast<float2 *>(ch + o4) = make_float2(tr2 - tr1, ti1 - ti2);
    }
  }
}

template <bool FIRST>
__device__ __forceinline__ void dev_fft_pass2(int ido, int l1, const float *cc, float *ch,
                                              const float *w1, int tid, int nt) {
  const int t0 = l1 * ido;
  if (ido == 1) {
    for (int k = tid; k < l1; k += nt) {
      const float a = cc[fft_rd<FIRST>(k)], b = cc[fft_rd<FIRST>(k + t0)];
      ch[fft_idx(2 * k)] = a + b;
      ch[fft_idx(2 * k + 1)] = a - b;
    }
    return;
  }
  const int half = ido >> 1;
  const int hsh = 31 - __clz(half);
  const int items = l1 * half;
  for (int v = tid; v < items; v += nt) {
    const int k = v >> hsh, ii = v & (half - 1);
    const int c0 = k * ido, c1 = c0 + t0;
    const int o = 2 * k * ido;
    if (ii == 0) {                                     // the two un-twiddled columns of this k
      const float a0 = cc[fft_rd<FIRST>(c0)], a1 = cc[fft_rd<FIRST>(c1)];
      ch[fft_idx(o)]               = a0 + a1;
      ch[fft_idx(o + 2 * ido - 1)] = a0 - a1;
      *reinterpret_cast<float2 *>(ch + fft_idx(o + ido - 1)) =
          make_float2(cc[fft_rd<FIRST>(c0 + ido - 1)], -cc[fft_rd<FIRST>(c1 + ido - 1)]);   // o[ido-1], o[ido]
    } else {
      const int i = 2 * ii;
      const float wr = __ldg(w1 + i - 2), wi = __ldg(w1 + i - 1);
      const int r0 = fft_rd<FIRST>(c0 + i - 1);
      const int r1 = FIRST ? r0 + t0 : ((t0 & 31) == 0 ? r0 + t0 + (t0 >> 4) : fft_idx(c1 + i - 1));
      const float2 a0 = *reinterpret_cast<const float2 *>(cc + r0);
      const float2 a1 = *reinterpret_cast<const float2 *>(cc + r1);
      const float tr2 = wr * a1.x + wi * a1.y;
      const float ti2 = wr * a1.y - wi * a1.x;
      const int ic = 2 * ido - i;
      *reinterpret_cast<float2 *>(ch + fft_idx(o + i - 1))  = make_float2(a0.x + tr2, a0.y + ti2);
      *reinterpret_cast<float2 *>(ch + fft_idx(o + ic - 1)) = make_float2(a0.x - tr2, ti2 - a0.y);
    }
  }
}

// ---- Two FFT levels per shared-memory pass (the power-of-two sizes with NC known at compile time).
// Level A is a dradf4 pass (ido = a, l1 = L); level B the pass after it (ido = 4a, l1 = L/4 for radix 4,
// L/2 for radix 2).  Level B reads element i' + 4a*k' + t0*j' (t0 = L*a = N/4), which level A writes as
// element i' of its output block k = k' + (L/4)*j' (radix-2 B: k = k' + (L/2)*j', j' < 2).  So the level-A
// items of one column i at those 4 (2) values of k produce exactly the inputs of 4 level-B items, which one
// thread runs from registers: one load and one store of every element per two levels, and one barrier.
// The butterflies below are those of dev_fft_pass4 / dev_fft_pass2, expression for expression.

// dradf4, column 0 (and the whole butterfly when ido = 1): o[0], (o[2ido-1], o[2ido]), o[4ido-1]
__device__ __forceinline__ void r4_col0(float a0, float a1, float a2, float a3, float &y0, float2 &y2, float &y4) {
  const float tr1 = a1 + a3;
  const float tr2 = a0 + a2;
  y0 = tr1 + tr2;
  y2 = make_float2(a0 - a2, a3 - a1);
  y4 = tr2 - tr1;
}
// dradf4, column ido-1: (o[ido-1], o[ido]), (o[3ido-1], o[3ido])
__device__ __forceinline__ void r4_colL(float a0, float a1, float a2, float a3, float2 &y1, float2 &y3) {
  const float hsqt2 = .70710678118654752f;
  const float ti1 = -hsqt2 * (a1 + a3);
  const float tr1 =  hsqt2 * (a1 - a3);
  y1 = make_float2(tr1 + a0, ti1 - a2);
  y3 = make_float2(a0 - tr1, ti1 + a2);
}
// dradf4, twiddled pair i (input pairs (i-1, i) of the four l1 blocks): the output pairs ending at
// i, 2ido-i, 2ido+i and 4ido-i
__device__ __forceinline__ void r4_tw(float2 a0, float2 a1, float2 a2, float2 a3, const float *w1, const float *w2,
                                      const float *w3, int i, float2 &y0, float2 &y1, float2 &y2, float2 &y3) {
  const float wa1r = __ldg(w1 + i - 2), wa1i = __ldg(w1 + i - 1);
  const float wa2r = __ldg(w2 + i - 2), wa2i = __ldg(w2 + i - 1);
  const float wa3r = __ldg(w3 + i - 2), wa3i = __ldg(w3 + i - 1);
  const float cr2 = wa1r * a1.x + wa1i * a1.y;
  const float ci2 = wa1r * a1.y - wa1i * a1.x;
  const float cr3 = wa2r * a2.x + wa2i * a2.y;
  const float ci3 = wa2r * a2.y - wa2i * a2.x;
  const float cr4 = wa3r * a3.x + wa3i * a3.y;
  const float ci4 = wa3r * a3.y - wa3i * a3.x;
  const float tr1 = cr2 + cr4, tr4 = cr4 - cr2;
  const float ti1 = ci2 + ci4, ti4 = ci2 - ci4;
  const float ti2 = a0.y + ci3, ti3 = a0.y - ci3;
  const float tr2 = a0.x + cr3, tr3 = a0.x - cr3;
  y0 = make_float2(tr1 + tr2, ti1 + ti2);
  y1 = make_float2(tr3 - ti4, tr4 - ti3);
  y2 = make_float2(ti4 + tr3, tr4 + ti3);
  y3 = make_float2(tr2 - tr1, ti1 - ti2);
}
// dradf2, twiddled pair i: the output pairs ending at i and 2ido-i
__device__ __forceinline__ void r2_tw(float2 a0, float2 a1, const float *w1, int i, float2 &y0, float2 &y1) {
  const float wr = __ldg(w1 + i - 2), wi = __ldg(w1 + i - 1);
  const float tr2 = wr * a1.x + wi * a1.y;
  const float ti2 = wr * a1.y - wi * a1.x;
  y0 = make_float2(a0.x + tr2, a0.y + ti2);
  y1 = make_float2(a0.x - tr2, ti2 - a0.y);
}
__device__ __forceinline__ void st_f2(float *p, int e, float2 v) { *reinterpret_cast<float2 *>(p + fft_idx(e)) = v; }
// padded index of e + D from r = fft_idx(e): one add when 32 | D (D is a compile-time constant in the fused passes),
// so the loads of an item share one index computation
__device__ __forceinline__ int fft_idx_add(int r, int e, int D) { return (D & 31) == 0 ? r + D + (D >> 4) : fft_idx(e + D); }
__device__ __forceinline__ float2 ld_f2(const float *p) { return *reinterpret_cast<const float2 *>(p); }

// level-B dradf4 (ido = ib) twiddled item i' of block k' from its four input pairs, stored
__device__ __forceinline__ void r4_tw_store(const float2 (&p)[4], const float *w1, const float *w2, const float *w3,
                                            int ip, int ib, int o, float *ch) {
  float2 y0, y1, y2, y3;
  r4_tw(p[0], p[1], p[2], p[3], w1, w2, w3, ip, y0, y1, y2, y3);
  const int e0 = o + ip - 1, e1 = o + 2 * ib - ip - 1;
  const int r0 = fft_idx(e0), r1 = fft_idx(e1);
  *reinterpret_cast<float2 *>(ch + r0) = y0;
  *reinterpret_cast<float2 *>(ch + r1) = y1;
  *reinterpret_cast<float2 *>(ch + fft_idx_add(r0, e0, 2 * ib)) = y2;
  *reinterpret_cast<float2 *>(ch + fft_idx_add(r1, e1, 2 * ib)) = y3;
}

// dradf4 (ido = a, l1 = L) then dradf4 (ido = 4a, l1 = L/4).  FIRST: level A reads the plain input (a = 1 only).
template <bool FIRST>
__device__ __forceinline__ void dev_fft_pass44(int a, int L, const float *cc, float *ch,
                                               const float *wa1, const float *wa2, const float *wa3,
                                               const float *wb1, const float *wb2, const float *wb3, int tid, int nt) {
  const int t0 = L * a, Lq = L >> 2, ib = 4 * a;
  if (a == 1) {
    // item k': the four one-column level-A butterflies of k = k' + Lq*j' give the 16 elements of level-B block k'
    for (int kp = tid; kp < Lq; kp += nt) {
      float y0[4], y3[4];
      float2 y12[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int k = kp + Lq * j;
        r4_col0(cc[fft_rd<FIRST>(k)], cc[fft_rd<FIRST>(k + t0)], cc[fft_rd<FIRST>(k + 2 * t0)],
                cc[fft_rd<FIRST>(k + 3 * t0)], y0[j], y12[j], y3[j]);
      }
      const int o = 16 * kp;
      float z0, z15;
      float2 z7, z3, z11;
      r4_col0(y0[0], y0[1], y0[2], y0[3], z0, z7, z15);
      ch[fft_idx(o)] = z0;
      st_f2(ch, o + 7, z7);
      ch[fft_idx(o + 15)] = z15;
      r4_colL(y3[0], y3[1], y3[2], y3[3], z3, z11);
      st_f2(ch, o + 3, z3);
      st_f2(ch, o + 11, z11);
      r4_tw_store(y12, wb1, wb2, wb3, 2, 4, o, ch);
    }
    return;
  }
  // a >= 4: Lq*a/2 items of 32 elements.  The first Lq are the two un-twiddled level-A columns of block k'
  // (giving level B's un-twiddled columns and its pairs i' = a, 2a, 3a), the others one twiddled level-A
  // column i (giving level B's pairs i' = i, 2a-i, 2a+i, 4a-i).
  const int hm1 = (a >> 1) - 1;
  const int items = Lq * (a >> 1);
  for (int v = tid; v < items; v += nt) {
    if (v < Lq) {
      const int kp = v;
      float s0[4], s1[4];
      float2 pa[3][4];                                     // [i' = a, 2a, 3a][j']
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int c0 = kp * a, e = c0 + a - 1, D = Lq * a * j;
        const int r = fft_idx(c0), q = fft_idx(e);
        r4_col0(cc[fft_idx_add(r, c0, D)], cc[fft_idx_add(r, c0, D + t0)], cc[fft_idx_add(r, c0, D + 2 * t0)],
                cc[fft_idx_add(r, c0, D + 3 * t0)], s0[j], pa[1][j], s1[j]);
        r4_colL(cc[fft_idx_add(q, e, D)], cc[fft_idx_add(q, e, D + t0)], cc[fft_idx_add(q, e, D + 2 * t0)],
                cc[fft_idx_add(q, e, D + 3 * t0)], pa[0][j], pa[2][j]);
      }
      const int o = 4 * kp * ib;
      float z0, zl;
      float2 zm, z1, z3;
      r4_col0(s0[0], s0[1], s0[2], s0[3], z0, zm, zl);
      ch[fft_idx(o)] = z0;
      st_f2(ch, o + 2 * ib - 1, zm);
      ch[fft_idx(o + 4 * ib - 1)] = zl;
      r4_colL(s1[0], s1[1], s1[2], s1[3], z1, z3);
      st_f2(ch, o + ib - 1, z1);
      st_f2(ch, o + 3 * ib - 1, z3);
#pragma unroll
      for (int m = 0; m < 3; m++) r4_tw_store(pa[m], wb1, wb2, wb3, (m + 1) * a, ib, o, ch);
    } else {
      const int g = v - Lq;
      const int kp = g / hm1, i = 2 * (1 + g - kp * hm1);
      const int e = kp * a + i - 1, r = fft_idx(e);
      float2 y[4][4];                                      // [i' = i, 2a-i, 2a+i, 4a-i][j']
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int D = Lq * a * j;
        r4_tw(ld_f2(cc + fft_idx_add(r, e, D)), ld_f2(cc + fft_idx_add(r, e, D + t0)),
              ld_f2(cc + fft_idx_add(r, e, D + 2 * t0)), ld_f2(cc + fft_idx_add(r, e, D + 3 * t0)), wa1, wa2, wa3, i,
              y[0][j], y[1][j], y[2][j], y[3][j]);
      }
      const int o = 4 * kp * ib;
      r4_tw_store(y[0], wb1, wb2, wb3, i, ib, o, ch);
      r4_tw_store(y[1], wb1, wb2, wb3, 2 * a - i, ib, o, ch);
      r4_tw_store(y[2], wb1, wb2, wb3, 2 * a + i, ib, o, ch);
      r4_tw_store(y[3], wb1, wb2, wb3, 4 * a - i, ib, o, ch);
    }
  }
}

// dradf4 (ido = a >= 4, l1 = L) then dradf2 (ido = 4a, l1 = L/2): items of 16 elements, as in dev_fft_pass44
__device__ __forceinline__ void dev_fft_pass42(int a, int L, const float *cc, float *ch,
                                               const float *wa1, const float *wa2, const float *wa3,
                                               const float *wb1, int tid, int nt) {
  const int t0 = L * a, Lh = L >> 1, ib = 4 * a;
  const int hm1 = (a >> 1) - 1;
  const int items = Lh * (a >> 1);
  for (int v = tid; v < items; v += nt) {
    if (v < Lh) {
      const int kp = v;
      float s0[2], s1[2];
      float2 pa[3][2];                                     // [i' = a, 2a, 3a][j']
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int c0 = kp * a, e = c0 + a - 1, D = Lh * a * j;
        const int r = fft_idx(c0), q = fft_idx(e);
        r4_col0(cc[fft_idx_add(r, c0, D)], cc[fft_idx_add(r, c0, D + t0)], cc[fft_idx_add(r, c0, D + 2 * t0)],
                cc[fft_idx_add(r, c0, D + 3 * t0)], s0[j], pa[1][j], s1[j]);
        r4_colL(cc[fft_idx_add(q, e, D)], cc[fft_idx_add(q, e, D + t0)], cc[fft_idx_add(q, e, D + 2 * t0)],
                cc[fft_idx_add(q, e, D + 3 * t0)], pa[0][j], pa[2][j]);
      }
      const int o = 2 * kp * ib;
      ch[fft_idx(o)]              = s0[0] + s0[1];
      ch[fft_idx(o + 2 * ib - 1)] = s0[0] - s0[1];
      st_f2(ch, o + ib - 1, make_float2(s1[0], -s1[1]));
#pragma unroll
      for (int m = 0; m < 3; m++) {
        const int ip = (m + 1) * a;
        float2 y0, y1;
        r2_tw(pa[m][0], pa[m][1], wb1, ip, y0, y1);
        st_f2(ch, o + ip - 1, y0);
        st_f2(ch, o + 2 * ib - ip - 1, y1);
      }
    } else {
      const int g = v - Lh;
      const int kp = g / hm1, i = 2 * (1 + g - kp * hm1);
      const int e = kp * a + i - 1, r = fft_idx(e);
      float2 y[4][2];                                      // [i' = i, 2a-i, 2a+i, 4a-i][j']
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int D = Lh * a * j;
        r4_tw(ld_f2(cc + fft_idx_add(r, e, D)), ld_f2(cc + fft_idx_add(r, e, D + t0)),
              ld_f2(cc + fft_idx_add(r, e, D + 2 * t0)), ld_f2(cc + fft_idx_add(r, e, D + 3 * t0)), wa1, wa2, wa3, i,
              y[0][j], y[1][j], y[2][j], y[3][j]);
      }
      const int o = 2 * kp * ib;
      const int ips[4] = {i, 2 * a - i, 2 * a + i, 4 * a - i};
#pragma unroll
      for (int m = 0; m < 4; m++) {
        float2 y0, y1;
        r2_tw(y[m][0], y[m][1], wb1, ips[m], y0, y1);
        st_f2(ch, o + ips[m] - 1, y0);
        st_f2(ch, o + 2 * ib - ips[m] - 1, y1);
      }
    }
  }
}

// the factor of pass k1 of a power-of-two N (see dev_drft_forward)
__host__ __device__ constexpr int fft_factor(int log2n, int k1) { return (k1 == ((log2n + 1) >> 1) - 1 && (log2n & 1)) ? 2 : 4; }

// dev_drft_forward for NC > 0: the passes from K1 on, two levels per pass where both exist and the first is radix 4
template <int NC, int K1, int L2, int IW>
__device__ __forceinline__ float *dev_drft_passes(const XformDev &X, float *src, float *dst, int tid, int nt) {
  constexpr int log2n = XLog2<NC>::v, nf = (log2n + 1) >> 1;
  if constexpr (K1 >= nf) {
    return src;
  } else {
    constexpr int ipA = fft_factor(log2n, K1), l1A = L2 / ipA, idoA = NC / L2, iwA = IW - (ipA - 1) * idoA;
    const float *wa = X.wa + iwA - 1;
    if constexpr (ipA == 4 && K1 + 1 < nf) {
      constexpr int ipB = fft_factor(log2n, K1 + 1), l1B = l1A / ipB, idoB = NC / l1A, iwB = iwA - (ipB - 1) * idoB;
      const float *wb = X.wa + iwB - 1;
      if constexpr (ipB == 4) {
        dev_fft_pass44<K1 == 0>(idoA, l1A, src, dst, wa, wa + idoA, wa + 2 * idoA, wb, wb + idoB, wb + 2 * idoB, tid, nt);
      } else {
        static_assert(K1 > 0, "the radix-2 pass is never second");
        dev_fft_pass42(idoA, l1A, src, dst, wa, wa + idoA, wa + 2 * idoA, wb, tid, nt);
      }
      __syncthreads();
      return dev_drft_passes<NC, K1 + 2, l1B, iwB>(X, dst, src, tid, nt);
    } else {
      if constexpr (ipA == 4) dev_fft_pass4<K1 == 0>(idoA, l1A, src, dst, wa, wa + idoA, wa + 2 * idoA, tid, nt);
      else dev_fft_pass2<K1 == 0>(idoA, l1A, src, dst, wa, tid, nt);
      __syncthreads();
      return dev_drft_passes<NC, K1 + 1, l1A, iwA>(X, dst, src, tid, nt);
    }
  }
}

// a: N plain input floats (16-byte aligned).  a and b must each have room for fft_buf_floats(N) floats:
// after the first pass `a` is reused as a padded ping-pong buffer.  Returns the buffer that holds the
// result; logical element e of it is at [fft_idx(e)].
template <int NC>
__device__ __forceinline__ float *dev_drft_forward(const XformDev &X, float *a, float *b,
                                                   int tid, int nt) {
  if constexpr (NC > 0) return dev_drft_passes<NC, 0, NC, NC>(X, a, b, tid, nt);
  const int N = NC ? NC : X.N;
  // power-of-two N: drfti1 stores 4,..,4 with a single 2 (odd log2) moved to the front, and the
  // passes run last factor first: radix 4 throughout, the radix-2 pass (if any) comes last
  const int log2n = NC ? XLog2<NC>::v : X.log2n;
  const int nf = (log2n + 1) >> 1;
  int l2 = N, iw = N;
  float *src = a, *dst = b;
#pragma unroll
  for (int k1 = 0; k1 < nf; k1++) {
    const int ip = (k1 == nf - 1 && (log2n & 1)) ? 2 : 4;
    const int l1 = l2 / ip, ido = N / l2;
    iw -= (ip - 1) * ido;
    if (k1 == 0) {
      if (ip == 4) dev_fft_pass4<true>(ido, l1, src, dst, X.wa + iw - 1, X.wa + iw + ido - 1, X.wa + iw + 2 * ido - 1, tid, nt);
      else dev_fft_pass2<true>(ido, l1, src, dst, X.wa + iw - 1, tid, nt);
    } else {
      if (ip == 4) dev_fft_pass4<false>(ido, l1, src, dst, X.wa + iw - 1, X.wa + iw + ido - 1, X.wa + iw + 2 * ido - 1, tid, nt);
      else dev_fft_pass2<false>(ido, l1, src, dst, X.wa + iw - 1, tid, nt);
    }
    __syncthreads();
    float *t = src; src = dst; dst = t;
    l2 = l1;
  }
  return src;
}

// _vorbis_apply_window (lib/window.c:2102-2135) fused into the load of one
// block from global memory: dst[i] = windowed src[i].
__device__ __forceinline__ float dev_window_gain(const WinDev &Wd, int W, int lW, int nW, int i,
                                                 bool &zero) {
  if (!W) { lW = 0; nW = 0; }
  const int n = Wd.N[W], ln = Wd.N[lW], rn = Wd.N[nW];
  const int leftbegin = n / 4 - ln / 4, leftend = leftbegin + ln / 2;
  const int rightbegin = n / 2 + n / 4 - rn / 4, rightend = rightbegin + rn / 2;
  zero = false;
  if (i < leftbegin || i >= rightend) { zero = true; return 0.f; }
  if (i < leftend) return __ldg(Wd.win[lW] + (i - leftbegin));
  if (i >= rightbegin) return __ldg(Wd.win[nW] + (rn / 2 - 1 - (i - rightbegin)));
  return 1.f;   // flat middle: sample is left untouched (x*1.0f is exact)
}

// The window regions all start on multiples of four samples (block sizes are powers of two >= 64), so a
// float4 never straddles two regions: one decision and at most one 128-bit table load per four samples.
__device__ __forceinline__ float4 dev_window4(const WinDev &Wd, int W, int lW, int nW, int i0, float4 x) {
  if (!W) { lW = 0; nW = 0; }
  const int n = Wd.N[W], ln = Wd.N[lW], rn = Wd.N[nW];
  const int leftbegin = n / 4 - ln / 4, leftend = leftbegin + ln / 2;
  const int rightbegin = n / 2 + n / 4 - rn / 4, rightend = rightbegin + rn / 2;
  if (i0 < leftbegin || i0 >= rightend) return make_float4(0.f, 0.f, 0.f, 0.f);
  if (i0 < leftend) {
    const float4 g = __ldg(reinterpret_cast<const float4 *>(Wd.win[lW] + (i0 - leftbegin)));
    return make_float4(x.x * g.x, x.y * g.y, x.z * g.z, x.w * g.w);
  }
  if (i0 >= rightbegin) {                           // the falling half reads the table backwards
    const float4 g = __ldg(reinterpret_cast<const float4 *>(Wd.win[nW] + (rn / 2 - 4 - (i0 - rightbegin))));
    return make_float4(x.x * g.w, x.y * g.z, x.z * g.y, x.w * g.x);
  }
  return x;                                         // flat middle: untouched (x*1.0f is exact)
}

// ------------------------------------------------------------------------
// Noise mask: bark_noise_hybridmp (lib/psy.c:547-704).
// S = 5 prefix arrays with row stride ns (ns = n+4 keeps the five sequential
// lanes on different banks for 128-bit accesses).
//
// The psy device functions are written for a *group* of threads that may be a
// subset of the CTA (warp specialisation): `tid`/`nt` are the rank and size of
// the group and group_sync() is a named barrier over exactly those threads.

__device__ __forceinline__ void group_sync(int barid, int nt) {
  if (nt == 32) __syncwarp();
  else named_bar_sync(barid, nt);
}

struct Abd { float A, B, D; };

__device__ __forceinline__ Abd dev_window_abd(int lo, int hi, const float *S, int ns) {
  const float *N = S, *X = S + ns, *XX = S + 2 * ns, *Y = S + 3 * ns, *XY = S + 4 * ns;
  // lo < 0 mirrors the window at 0 (lib/psy.c:608-624): N, XX, Y are ADDED there, X and XY subtracted as always.
  // x + y == x - (-y) exactly, so the mirrored case only flips the sign bit of three operands: one code path.
  const int a = lo < 0 ? -lo : lo;
  const unsigned flip = lo < 0 ? 0x80000000u : 0u;
  const float nN = __uint_as_float(__float_as_uint(N[a]) ^ flip);
  const float nXX = __uint_as_float(__float_as_uint(XX[a]) ^ flip);
  const float nY = __uint_as_float(__float_as_uint(Y[a]) ^ flip);
  const float tN = N[hi] - nN, tX = X[hi] - X[a], tXX = XX[hi] - nXX;
  const float tY = Y[hi] - nY, tXY = XY[hi] - XY[a];
  Abd r;
  r.A = tY * tXX - tX * tXY;
  r.B = tN * tXY - tX * tY;
  r.D = tN * tXX - tX * tX;
  return r;
}

// per-bin terms of the five running sums (lib/psy.c:565-596)
// f = a[i] (b == nullptr) or a[i] - b[i] (second pass: logmdct - first-pass mask, lib/psy.c:717)
__device__ __forceinline__ void dev_noise_terms(int n, const float *a, const float *b, float offset,
                                                float *S, int ns, int tid, int nt) {
  float *aN = S, *aX = S + ns, *aXX = S + 2 * ns, *aY = S + 3 * ns, *aXY = S + 4 * ns;
  for (int i = tid; i < n; i += nt) {
    const float f = b ? a[i] - b[i] : a[i];
    float y = f + offset;
    if (y < 1.f) y = 1.f;
    float w = y * y;
    if (i == 0) {
      w = w * .5f;
      aN[0] = w; aX[0] = w; aXX[0] = 0.f; aY[0] = w * y; aXY[0] = 0.f;
    } else {
      const float x = (float)i;
      const float wx = w * x;
      aN[i] = w; aX[i] = wx; aXX[i] = wx * x; aY[i] = w * y; aXY[i] = wx * y;
    }
  }
}

// The running sums are strictly sequential fp32 (order matters, SURVEY fact 8):
// five lanes, one array each, 16 values in flight per lane so that only the
// 4-cycle add chain is on the critical path.
__device__ __forceinline__ void dev_noise_scan(int n, float *S, int ns, int lane) {
  if (lane >= 5) return;
  float4 *a = reinterpret_cast<float4 *>(S + lane * ns);
  const int q = n >> 2;                   // float4 count (n is a multiple of 32)
  float t = 0.f;
  float4 v0 = a[0], v1 = a[1], v2 = a[2], v3 = a[3];
  for (int i = 0; i < q; i += 4) {
    float4 w0 = v0, w1 = v1, w2 = v2, w3 = v3;
    if (i + 4 < q) { v0 = a[i + 4]; v1 = a[i + 5]; v2 = a[i + 6]; v3 = a[i + 7]; }
    t += w0.x; w0.x = t; t += w0.y; w0.y = t; t += w0.z; w0.z = t; t += w0.w; w0.w = t;
    t += w1.x; w1.x = t; t += w1.y; w1.y = t; t += w1.z; w1.z = t; t += w1.w; w1.w = t;
    t += w2.x; w2.x = t; t += w2.y; w2.y = t; t += w2.z; w2.z = t; t += w2.w; w2.w = t;
    t += w3.x; w3.x = t; t += w3.y; w3.y = t; t += w3.z; w3.z = t; t += w3.w; w3.w = t;
    a[i] = w0; a[i + 1] = w1; a[i + 2] = w2; a[i + 3] = w3;
  }
}

// regression per bin (lib/psy.c:604-703); bins past first_extra reuse the last A,B,D
// If logmdct != nullptr this is the second pass and the final step of _vp_noisemask
// (lib/psy.c:722,745-750) is applied in place: noise[i] holds the first-pass mask p1 on entry.
__device__ __forceinline__ void dev_noise_regress(const PsyDev &P, float *noise, float offset, int fixed,
                                                  const float *S, int ns, int tid, int nt,
                                                  const float *logmdct) {
  const int n = P.n;
  const int bfe = P.bark_first_extra;
  const int ffe = P.fixed_first_extra;
  for (int i = tid; i < n; i += nt) {
    Abd cur; cur.A = 0.f; cur.B = 0.f; cur.D = 1.f;
    if (bfe > 0) {
      const int wb = i < bfe ? i : bfe - 1;
      const int bk = __ldg(P.bark + wb);
      cur = dev_window_abd(bk >> 16, bk & 0xffff, S, ns);
    }
    const float x = (float)i;
    float R = (cur.A + x * cur.B) / cur.D;
    if (R < 0.f) R = 0.f;
    float v = R - offset;
    if (fixed > 0) {
      if (ffe > 0) {
        const int wb = i < ffe ? i : ffe - 1;
        const int hi = wb + fixed / 2, lo = hi - fixed;
        cur = dev_window_abd(lo, hi, S, ns);
      } else if (bfe > 0 && i < bfe) {
        // no fixed window qualifies: A,B,D left by the bark loops' last bin
        const int bk = __ldg(P.bark + (bfe - 1));
        cur = dev_window_abd(bk >> 16, bk & 0xffff, S, ns);
      }
      const float R2 = (cur.A + x * cur.B) / cur.D;
      if (R2 - offset < v) v = R2 - offset;
    }
    if (logmdct) {
      const float l = logmdct[i];
      const float work = l - noise[i];               // logmdct - p1   (lib/psy.c:717)
      const float base = l - work;                   // logmdct - work (lib/psy.c:722)
      int dB = (int)((double)v + .5);
      if (dB >= VB200_COMPAND_LEVELS) dB = VB200_COMPAND_LEVELS - 1;
      if (dB < 0) dB = 0;
      v = base + __ldg(P.noisecompand + dB);
    }
    noise[i] = v;
  }
}

// single-bin form used by the register-resident kernel (vb200_psy3.cuh)
__device__ __forceinline__ void dev_noise_term1(int i, float f, float offset, float *S, int ns) {
  float *aN = S, *aX = S + ns, *aXX = S + 2 * ns, *aY = S + 3 * ns, *aXY = S + 4 * ns;
  float y = f + offset;
  if (y < 1.f) y = 1.f;
  float w = y * y;
  if (i == 0) {
    w = w * .5f;
    aN[0] = w; aX[0] = w; aXX[0] = 0.f; aY[0] = w * y; aXY[0] = 0.f;
  } else {
    const float x = (float)i;
    const float wx = w * x;
    aN[i] = w; aX[i] = wx; aXX[i] = wx * x; aY[i] = w * y; aXY[i] = wx * y;
  }
}

// _vp_noisemask (lib/psy.c:706-752): logmdct (smem) -> noise (smem).
// If terms_done, the pass-1 terms were already written to S by the caller.
__device__ __forceinline__ void dev_noisemask(const PsyDev &P, const float *logmdct, float *noise,
                                              float *S, int ns, int tid, int nt,
                                              int barid, bool terms_done) {
  const int n = P.n;
  if (!terms_done) { dev_noise_terms(n, logmdct, nullptr, 140.f, S, ns, tid, nt); group_sync(barid, nt); }
  if (tid < 32) dev_noise_scan(n, S, ns, tid);
  group_sync(barid, nt);
  dev_noise_regress(P, noise, 140.f, -1, S, ns, tid, nt, nullptr);
  group_sync(barid, nt);
  dev_noise_terms(n, logmdct, noise, 0.f, S, ns, tid, nt);
  group_sync(barid, nt);
  if (tid < 32) dev_noise_scan(n, S, ns, tid);
  group_sync(barid, nt);
  dev_noise_regress(P, noise, 0.f, P.noisewindowfixed, S, ns, tid, nt, logmdct);
  group_sync(barid, nt);
}

// ------------------------------------------------------------------------
// Tone mask: _vp_tonemask (lib/psy.c:754-777) with seed_loop/seed_curve
// (:417-452, :390-415), seed_chase (:454-508) and max_seeds (:512-545).
//
// seed_curve's scatter-max is evaluated owner-computes: a seed slot s can only
// be written by runs r with (s - oc_r + linesper/2) divisible by linesper, and
// only through curve point i = (s - oc_r + half)/linesper + 16.  The candidate
// runs of every slot are a static contiguous range of a per-residue run list,
// so each slot takes the max over its candidates: no atomics, and max is
// order-independent so the result is bit-identical to the sequential scatter.

struct ToneSmem {
  float *seed;      // [total]
  float *astk;      // [total]
  short *pstk;      // [total]
  int4  *run_rec;   // [nruns] in cls_run order: decoded run records (see dev_tone_runs)
  short *rec;       // [total] chase restart points; aliases run_rec (dead by then)
};

__device__ __forceinline__ float tone_att(const PsyDev &P, float lmax) {
  float att = lmax + P.ath_adjatt;
  if (att < P.ath_maxatt) att = P.ath_maxatt;
  return att;
}

// seed_loop: one item per run of equal octave[] (peak, audibility gate, curve choice).
// Items are visited in residue-class order (cls_run) and everything seed_curve needs is
// decoded here, once, into a 16-byte record at that index:
//   rec.x = peak (float bits)          rec.y = index of the first usable curve value
//   rec.z = seed slot of that value     rec.w = number of usable values (0: inactive)
// "usable" = curve points post0..post1-1 whose slot lies in (0,total) (lib/psy.c:405-413).
__device__ __forceinline__ void dev_tone_runs(const PsyDev &P, const float *logfft, float gmax, float lmax,
                                              const ToneSmem &T, int tid, int nt) {
  const float att = tone_att(P, lmax);
  const float dBoffset = P.max_curve_dB - gmax;
  const int L = P.linesper, half = L >> 1, total = P.total;
  for (int k = tid; k < P.nruns; k += nt) {
    const int4 rr = __ldg(P.runrec + k);             // lo|hi<<16, oc - firstoc, band, ath[hi]
    int4 ri; ri.x = rr.x & 0xffff; ri.y = rr.x >> 16; ri.z = rr.y; ri.w = rr.z;
    float mx = logfft[ri.x];
    for (int i = ri.x + 1; i <= ri.y; i++) { const float v = logfft[i]; if (v > mx) mx = v; }
    int4 rec = make_int4(__float_as_int(mx), 0, 0, 0);
    if (mx + 6.f > __int_as_float(rr.w) + att) {
      int choice = (int)((((double)(mx + dBoffset)) - 30.) * (double).1f);   // P_LEVEL_0 is a double
      if (choice < 0) choice = 0;
      if (choice > VB200_P_LEVELS - 1) choice = VB200_P_LEVELS - 1;
      const int cbase = (ri.w * VB200_P_LEVELS + choice) * (VB200_EHMER_MAX + 2);
      int post0 = (int)__ldg(P.tonecurves + cbase), post1 = (int)__ldg(P.tonecurves + cbase + 1);
      // clip to slots 1..total-1:  sp(i) = oc + (i-16)*L - half
      const int sp_at0 = ri.z - 16 * L - half;                   // slot of i = 0
      // smallest i with sp(i) > 0  and  smallest i with sp(i) >= total
      int ilo = sp_at0 > 0 ? 0 : (-sp_at0) / L + 1;
      int ihi = total - sp_at0 <= 0 ? 0 : (total - sp_at0 + L - 1) / L;
      if (post0 < ilo) post0 = ilo;
      if (post1 > ihi) post1 = ihi;
      if (post0 < post1) {
        rec.y = cbase + 2 + post0;
        rec.z = sp_at0 + post0 * L;
        rec.w = post1 - post0;
      }
    }
    T.run_rec[k] = rec;
  }
}

// seed_curve (lib/psy.c:390-415) for all runs, without atomics: a run with octave
// position oc only touches slots s = oc - L/2 (mod L), so runs of different residue
// classes never collide.  Each class is owned by a group of G = nt/L lanes (inside one
// warp) that walks the class' runs in order; within a run the G lanes update distinct
// slots; __syncwarp() orders the runs.  `max` is order-independent, so the result is
// bit-identical to the reference's sequential scatter.  Requires L in {4,8,16,32} and
// nt == 128 (G = 32,16,8,4 lanes); other L use dev_tone_slots_gather below.
__device__ __forceinline__ void dev_tone_slots_scatter(const PsyDev &P, const ToneSmem &T, int tid, int nt) {
  const int L = P.linesper, total = P.total;
  for (int s = tid; s < total; s += nt) T.seed[s] = VB_NEGINF;
  __syncthreads();
  const int G = nt >> P.linesper_log2;               // lanes per class (<= 32)
  const int cls = tid / G, g = tid - cls * G;
  const int k0 = __ldg(P.cls_off + cls), k1 = __ldg(P.cls_off + cls + 1);
  // every warp loops to the longest class it hosts so that __syncwarp() is convergent
  const int wfirst = (tid & ~31) / G, wlast = ((tid | 31)) / G;
  int len = 0;
  for (int c = wfirst; c <= wlast; c++) { const int l = __ldg(P.cls_off + c + 1) - __ldg(P.cls_off + c); if (l > len) len = l; }
  const int GL = G * L, gL = g * L;
  // software pipeline, two register sets: while run q is applied, run q+1's record and its first
  // two curve values (the only global reads, L2/L1 resident) are already in flight
  const unsigned a_seed = smem_u32(T.seed), a_rec = smem_u32(T.run_rec);
  const float *__restrict__ curves = P.tonecurves;
  struct Run { float mx, c0, c1; int ext, sp, ci; };
  auto fetch = [&](int k, Run &r) {
    r.ext = 0;
    if (k < k1) {
      const int4 v = lds_v4(a_rec + 16u * k);
      r.mx = __int_as_float(v.x);
      r.ci = v.y + g;
      r.sp = v.z + gL;
      r.ext = v.w - g;                               // > 0: values ci, ci+G, ... for this lane
      if (r.ext > 0) r.c0 = __ldg(curves + r.ci);
      if (r.ext > G) r.c1 = __ldg(curves + r.ci + G);
    }
  };
  auto apply = [&](const Run &r) {
    if (r.ext > 0) {
      const unsigned a0 = a_seed + 4u * r.sp;
      sts_f32(a0, fmaxf(lds_f32(a0), r.mx + r.c0));
      if (r.ext > G) {
        const unsigned a1 = a0 + 4u * GL;
        sts_f32(a1, fmaxf(lds_f32(a1), r.mx + r.c1));
        for (int t = 2; r.ext > t * G; t++) {
          const unsigned at = a0 + 4u * t * GL;
          sts_f32(at, fmaxf(lds_f32(at), r.mx + __ldg(curves + r.ci + t * G)));
        }
      }
    }
  };
  Run A, B;
  A.mx = A.c0 = A.c1 = 0.f; A.ext = A.sp = A.ci = 0; B = A;
  fetch(k0, A);
  for (int q = 0; q < len; q += 2) {
    fetch(k0 + q + 1, B);
    apply(A);
    __syncwarp();
    if (q + 1 < len) {
      fetch(k0 + q + 2, A);
      apply(B);
      __syncwarp();
    }
  }
}

// seed_curve, owner-computes (generic fallback): one item per seed slot
__device__ __forceinline__ void dev_tone_slots_gather(const PsyDev &P, const ToneSmem &T, int tid, int nt) {
  for (int s = tid; s < P.total; s += nt) {
    float m = VB_NEGINF;
    const int2 rg = __ldg(P.slot_rng + s);           // candidate range in cls_run (empty for s == 0)
    for (int k = rg.x; k < rg.y; k++) {
      const int4 rec = T.run_rec[k];                 // peak, first curve index, first slot, count
      const int d = s - rec.z;                       // multiple of L by construction of the class
      const int j = d >> P.linesper_log2;
      if (d >= 0 && j < rec.w) {
        const float lin = __int_as_float(rec.x) + __ldg(P.tonecurves + rec.y + j);
        if (m < lin) m = lin;
      }
    }
    T.seed[s] = m;
  }
}

__device__ __forceinline__ void dev_tone_slots(const PsyDev &P, const ToneSmem &T, int tid, int nt) {
  if (nt == 128 && P.linesper >= 4 && P.linesper <= 32) dev_tone_slots_scatter(P, T, tid, nt);
  else dev_tone_slots_gather(P, T, tid, nt);
}

// seed_chase + max_seeds gather, executed by ONE warp (lane = 0..31).
// tone: n floats (written).
//
// seed_chase (lib/psy.c:454-508) is a stack algorithm whose pop rule is not a
// sliding maximum (SURVEY §7), so it is emulated literally -- but not by one lane.
// Exact segmentation: at step i the entry left directly below the new entry i has
// position >= i-L+1 (a pop needs `i < pos[below]+L`).  Hence if seeds[i] is strictly
// greater than seeds[i-L+1..i-1] ("record"), entry i sits on a strictly smaller
// entry, can never satisfy the pop test `amp[top] <= amp[top-1]`, and freezes
// everything beneath it: the algorithm restarted at i with an empty stack evolves
// identically from there on.  The warp finds all records, splits them evenly over
// its 32 lanes, and every lane runs the unmodified stack algorithm on its own
// segment (up to and including the pop phase of the next lane's first record).
// The final stack is the concatenation of the lanes' stacks.  Worst case (no record,
// e.g. an all-NEGINF seed vector) degenerates to one lane doing all the work.
__device__ __forceinline__ void dev_tone_chase_gather(const PsyDev &P, float *tone, float lmax,
                                                      const ToneSmem &T, int lane) {
  const int n = P.n, total = P.total, linesper = P.linesper;
  float *seed = T.seed; short *pstk = T.pstk; float *astk = T.astk; short *rec = T.rec;
  const unsigned full = 0xffffffffu;
  // 1. records
  int m = 0;
  for (int base = 0; base < total; base += 32) {
    const int i = base + lane;
    // record <=> strictly greater than each of the previous linesper-1 seeds (branch free)
    bool r = i < total;
    {
      const float v = r ? seed[i] : 0.f;
      for (int d = 1; d < linesper; d++) {
        const int j = i - d;
        const float u = (r && j >= 0) ? seed[j] : 0.f;
        r = r && (j < 0 || v > u);
      }
    }
    const unsigned b = __ballot_sync(full, r);
    if (r) rec[m + __popc(b & ((1u << lane) - 1u))] = (short)i;
    m += __popc(b);
  }
  __syncwarp();
  // 2. this lane's segment [start, end]
  const int r0 = (lane * m) >> 5, r1 = ((lane + 1) * m) >> 5;
  int start = 0, end = 0, cnt = 0;
  if (r0 < r1) {
    start = rec[r0];
    end = r1 < m ? rec[r1] : total;
    // 3. the stack algorithm on seeds[start..end); entries stored at astk/pstk[start + depth].
    // Top three entries are cached in registers (a0 = top, l = pos + linesper, c = #valid).
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    int l0 = 0, l1 = 0, l2 = 0, c = 0, stack = 0;
    float s = seed[start];
    for (int i = start; i <= end && i < total; i++) {
      const float snext = i + 1 < total ? seed[i + 1] : 0.f;
      if (stack >= 2 && !(s < a0)) {
        for (;;) {
          if (c < 2) { a1 = astk[start + stack - 2]; l1 = pstk[start + stack - 2] + linesper; c = 2; }
          if (!(i < l0 && a0 <= a1 && i < l1)) break;
          stack--;                           // top is completely overlapped: drop it
          a0 = a1; l0 = l1; a1 = a2; l1 = l2; c--;
          if (stack < 2 || s < a0) break;    // the reference re-tests seeds[i] < new top
        }
      }
      if (i < end) {                         // i == end: only the pops belong to this lane
        astk[start + stack] = s; pstk[start + stack] = (short)i;
        a2 = a1; l2 = l1; a1 = a0; l1 = l0; a0 = s; l0 = i + linesper;
        stack++;
        c = c < 3 ? c + 1 : 3;
      }
      s = snext;
    }
    cnt = stack;
  }
  __syncwarp();
  // 4. fill (lib/psy.c:489-503): entry k is written from the running cursor to endpos_k
  {
    int M = 0;
    for (int j = 0; j < cnt; j++) {
      const float a = astk[start + j];
      int endpos;
      const int nx = j + 1 < cnt ? start + j + 1 : (end < total ? end : -1);
      if (nx >= 0 && astk[nx] > a) endpos = pstk[nx];
      else endpos = pstk[start + j] + linesper + 1;
      if (endpos > total) endpos = total;
      if (endpos > M) M = endpos;
    }
    int incl = M;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(full, incl, o);
      if (lane >= o && t > incl) incl = t;
    }
    int cursor = __shfl_up_sync(full, incl, 1);
    if (lane == 0) cursor = 0;
    __syncwarp();
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
  }
  __syncwarp();
  // gather (max_seeds second half): one item per static group; tone starts as ath+att
  const float att = tone_att(P, lmax);
  for (int g = lane; g < P.ngrp; g += 32) {
    const int4 gg = __ldg(P.grps + g);
    int pos = gg.x;
    float minV = seed[pos];
    if (minV > P.tone_abs_limit) minV = P.tone_abs_limit;
    while (pos < gg.y) {
      pos++;
      const float s = seed[pos];
      if ((s > VB_NEGINF && s < minV) || minV == VB_NEGINF) minV = s;
    }
    for (int i = gg.z; i < gg.w; i++) {
      float t = __ldg(P.ath + i) + att;
      if (t < minV) t = minV;
      tone[i] = t;
    }
  }
  {
    const float minV = seed[total - 1];
    for (int i = P.tail_lin0 + lane; i < n; i += 32) {
      float t = __ldg(P.ath + i) + att;
      if (t < minV) t = minV;
      tone[i] = t;
    }
  }
  __syncwarp();
}


// _vp_offset_and_mix for one bin (lib/psy.c:779-835); returns logmask, scales m.
__device__ __forceinline__ float dev_mix_bin(const PsyDev &P, int sel, float noise, float tone,
                                             float noff, float logmdct, float &m) {
  float val = noise + noff;
  if (val > P.noisemaxsupp) val = P.noisemaxsupp;
  const float t = tone + P.tone_masteratt[sel];
  const float logmask = val < t ? t : val;
  if (sel == 1) {
    const float coeffi = -17.2f;
    float de;
    val = val - logmdct;
    if (val > coeffi) {
      de = (float)(1.0 - ((double)(val - coeffi) * 0.005 * (double)P.m_val));
      if (de < 0.f) de = 0.0001f;
    } else {
      de = (float)(1.0 - ((double)(val - coeffi) * 0.0003 * (double)P.m_val));
    }
    m *= de;
  }
  return logmask;
}

}  // namespace vb200
