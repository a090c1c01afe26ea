// vb200_cqn.cuh — Phase B: _vp_couple_quantize_normalize (lib/psy.c:1014-1213) with
// flag_lossless (:924-935) and noise_normalize (:941-1010).
//
// Partitions are independent (noise_normalize resets its accumulator, :951), and inside
// a partition every line is independent except for (a) the fp32 sum of the pooled
// energies, taken in line order, and (b) the descending sort of the pooled lines.
// One warp owns 32 consecutive lines of one block for all channels: lane = line; a
// partition (8, 16 or 32 lines) is a sub-group of the warp and (a),(b) use shuffles of
// that width.  Per-channel working values live in shared memory columns owned by the lane.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

namespace vb200 {

struct CqnDev {
  int n, ch, partition, limit, sliding_lowpass, steps;
  int normal_p, normal_start;
  float prepoint, postpoint;
  double normal_thresh;
  const int *mag, *ang;        // [steps]
  const float *fromdB;         // [256] floor1_inverse_dB_table
};

// lib/psy.c:959-963: rint(sqrt(ve)) in double, then the sign.  For ve < 2^22 the result is computed
// without the fp64 square root: q0 = trunc(sqrtf(ve)) is floor(sqrt(ve)) or one more (only when ve is
// within an fp32 rounding of q0^2, where q0 is still the nearest integer), and the nearest integer
// is q0+1 exactly when ve > (q0+.5)^2 = q0^2+q0+.25, a comparison that is exact in fp64.  The
// correctly rounded double sqrt can only land on a tie k+.5 when ve == (k+.5)^2 exactly (ve has
// 24 significant bits), where rint rounds to even.
__device__ __forceinline__ int cqn_quant(float sign_src, float ve) {
  int q;
  if (ve < 4194304.f) {
    const int q0 = (int)sqrtf(ve);
    const double h = (double)(q0 * q0 + q0) + .25, vd = (double)ve;
    q = q0 + ((vd > h || (vd == h && (q0 & 1))) ? 1 : 0);
  } else {
    q = (int)rint(sqrt((double)ve));
  }
  return sign_src < 0.f ? -q : q;
}

// noise_normalize for the lane's line.  use_flags=false <=> flags==NULL in the reference.
__device__ __forceinline__ void cqn_normalize(const CqnDev &Q, float r, float &q, float f, bool use_flags,
                                              int flag, int i, int j, int &out, int width, int lane) {
  const unsigned full = 0xffffffffu;
  const int jn = Q.partition;
  int start = Q.normal_p ? Q.normal_start - i : jn;
  if (start > jn) start = jn;
  const bool skip = use_flags && flag;             // losslessly coupled: already quantised
  bool pooled = false;
  float ve = 0.f;
  if (!skip) {
    ve = q / f;
    if (j >= start && ve < .25f && (!use_flags || j >= Q.limit - i)) pooled = true;
    else {
      out = cqn_quant(r, ve);
      if (j >= start) q = out * out * f;
    }
  }
  // (a) acc += ve over the pooled lines in increasing line order (fp32, sequential)
  // (b) rank among pooled lines, descending by q, ties by line order (stable, as qsort here)
  // Only pooled lines take part, so the walk visits the set bits of the ballot: `offs` is the
  // union over the warp's partitions of the in-partition offsets that hold a pooled line.
  const unsigned bal = __ballot_sync(full, pooled);
  if (!bal) return;
  const int g0 = lane & ~(width - 1);
  const unsigned wmask = width == 32 ? full : ((1u << width) - 1u);
  const unsigned mine = (bal >> g0) & wmask;
  unsigned offs = 0;
  for (int g = 0; g < 32; g += width) offs |= (bal >> g) & wmask;
  float acc = 0.f;
  int rank = 0;
  const int any = mine != 0;
  for (unsigned m = offs; m; m &= m - 1) {
    const int t = __ffs(m) - 1;
    const float vt = __shfl_sync(full, ve, g0 + t);
    const float qt = __shfl_sync(full, q, g0 + t);
    if ((mine >> t) & 1) {
      acc += vt;
      if (qt > q || (qt == q && t < j)) rank++;
    }
  }
  if (any && pooled) {
    // lines are visited in rank order; each promotion costs 1.0 of acc (lib/psy.c:993-1006)
    float a = acc;
    bool ok = true;
    for (int u = 0; u < rank; u++) {
      if (!((double)a >= Q.normal_thresh)) { ok = false; break; }
      a -= 1.f;
    }
    if (ok && (double)a >= Q.normal_thresh) {
      out = (int)__int_as_float((__float_as_int(r) & 0x80000000) | 0x3f800000);   // unitnorm
      q = f;
    } else {
      out = 0;
      q = 0.f;
    }
  }
}

// field-wise select: a reference to one of two kernel-parameter structs would force both into
// local memory (dynamic indexing of the parameter space)
__device__ __forceinline__ CqnDev cqn_pick(const CqnDev &a, const CqnDev &b, bool second) {
  CqnDev q;
  q.n = a.n; q.ch = a.ch; q.steps = a.steps; q.mag = a.mag; q.ang = a.ang; q.fromdB = a.fromdB;
  q.partition = second ? b.partition : a.partition;
  q.limit = second ? b.limit : a.limit;
  q.sliding_lowpass = second ? b.sliding_lowpass : a.sliding_lowpass;
  q.normal_p = second ? b.normal_p : a.normal_p;
  q.normal_start = second ? b.normal_start : a.normal_start;
  q.prepoint = second ? b.prepoint : a.prepoint;
  q.postpoint = second ? b.postpoint : a.postpoint;
  q.normal_thresh = second ? b.normal_thresh : a.normal_thresh;
  return q;
}

// ---- register-resident version for 1 channel, or 2 channels with at most one coupling step
// (every stereo / mono setup of vorbisenc).  Lane = line as in k_cqn, but nothing goes through
// shared memory except the 256-entry floor table, and the next task's four loads are in flight
// while the current one is computed (the kernel is latency bound: two dependent global loads,
// two IEEE divisions and an fp64 sqrt per channel on the critical path).
//
// One (block, 32 lines) task of one curve: slot 0 = magnitude channel, slot 1 = angle channel.
template <int CH>
__device__ __forceinline__ void cqn_fast_lines(const CqnDev &Q, const float *s_fromdB, bool coupled, int line,
                                               int lane, const float (&mv)[CH], const int (&il)[CH],
                                               const int (&nzr)[CH], int (&out)[CH]) {
  const int width = Q.partition;
  const int i = line & ~(width - 1), j = line - i;
  float R[CH], Qe[CH], F[CH];
  int G[CH];
#pragma unroll
  for (int k = 0; k < CH; k++) {
    R[k] = 0.f; Qe[k] = 0.f; F[k] = 1e-10f; G[k] = 0; out[k] = 0;
    if (nzr[k]) {
      const float fl = s_fromdB[il[k] & 255];
      const float point = j >= Q.limit - i ? Q.postpoint : Q.prepoint;      // flag_lossless
      G[k] = (fabsf(mv[k]) / fl < point) ? 0 : 1;
      Qe[k] = R[k] = mv[k] * mv[k];
      if (mv[k] < 0.f) R[k] *= -1.f;
      F[k] = fl * fl;
      cqn_normalize(Q, R[k], Qe[k], F[k], false, 0, i, j, out[k], width, lane);
    }
  }
  if (CH == 2 && coupled && (nzr[0] || nzr[1])) {
    float reM = R[0], reA = R[1], qeM = Qe[0], qeA = Qe[1];
    int gM = G[0], gA = G[1], iM = out[0], iA = out[1];
    if (j < Q.sliding_lowpass - i) {
      if (gM || gA) {                                    // lossless: integer square-polar map
        const int A = iM, B = iA;
        reM = fabsf(reM) + fabsf(reA);
        qeM = qeM + qeA;
        gM = gA = 1;
        if (abs(A) > abs(B)) {
          iA = (A > 0 ? A - B : B - A);
        } else {
          iA = (B > 0 ? A - B : B - A);
          iM = B;
        }
        if (iA >= abs(iM) * 2) { iA = -iA; iM = -iM; }
      } else {                                           // point stereo
        if (j < Q.limit - i) {
          reM += reA;
          qeM = fabsf(reM);
        } else {
          const float e = fabsf(reM) + fabsf(reA);
          qeM = e;
          reM = (reM + reA < 0.f) ? -e : e;
        }
        reA = qeA = 0.f;
        gA = 1;
        iA = 0;
      }
    }
    const float fM = F[0] + F[1];
    cqn_normalize(Q, reM, qeM, fM, true, gM, i, j, iM, width, lane);
    out[0] = iM; out[1] = iA;
  }
}

template <int CH>
__global__ void __launch_bounds__(128)
k_cqn_fast(CqnDev Q0, CqnDev Q1, const vb200_block_desc *__restrict__ desc, int nblocks,
           const float *__restrict__ mdct, int *__restrict__ iwork, const int *__restrict__ nonzero) {
  __shared__ float s_fromdB[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_fromdB[i] = __ldg(Q0.fromdB + i);
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int n = Q0.n, csh = 31 - __clz(n >> 5);          // n is a power of two: chunks = 1 << csh
  const int tasks = nblocks << csh, stride = gridDim.x * wpb;   // the launcher keeps tasks < 2^31
  const bool coupled = CH == 2 && Q0.steps > 0;
  // slot 0 = magnitude channel, slot 1 = angle channel (channels are independent up to the coupling)
  const int c0 = coupled ? __ldg(Q0.mag) : 0, c1 = coupled ? __ldg(Q0.ang) : 1;
  float mv[CH], nmv[CH];
  int il[CH], nil[CH], nzr[CH], nnz[CH];
  auto fetch = [&](int t, float (&m_)[CH], int (&i_)[CH], int (&z_)[CH]) {
    const int blk = t >> csh, line = ((t & ((1 << csh) - 1)) << 5) + lane;
#pragma unroll
    for (int k = 0; k < CH; k++) {
      const int c = k == 0 ? c0 : c1;
      const size_t row = (size_t)blk * CH + c;
      z_[k] = __ldg(nonzero + row);
      m_[k] = __ldcs(mdct + row * n + line);
      i_[k] = __ldcs(iwork + row * n + line);
    }
  };
  int t = blockIdx.x * wpb + wid;
  if (t < tasks) fetch(t, nmv, nil, nnz);
  for (; t < tasks; t += stride) {
#pragma unroll
    for (int k = 0; k < CH; k++) { mv[k] = nmv[k]; il[k] = nil[k]; nzr[k] = nnz[k]; }
    if (t < tasks - stride) fetch(t + stride, nmv, nil, nnz);
    const int blk = t >> csh, line = ((t & ((1 << csh) - 1)) << 5) + lane;
    const CqnDev Q = cqn_pick(Q0, Q1, desc && desc[blk].blocktype);
    int out[CH];
    cqn_fast_lines<CH>(Q, s_fromdB, coupled, line, lane, mv, il, nzr, out);
    {
      int *iw = iwork + (size_t)blk * CH * n + line;
      __stcs(iw + (size_t)c0 * n, out[0]);
      if (CH == 2) __stcs(iw + (size_t)c1 * n, out[CH - 1]);
    }
  }
}

// ---- bitrate-managed mode: all VB200_PACKETBLOBS curves in one launch (same channel cases as k_cqn_fast).
// The curves share the MDCT and differ in the floor (iwork[k] holds curve k's ilogmask on entry), the
// nonzero flags and four parameters of the blob, kept per (blocktype, blob) in shared memory.  One warp owns
// 32 lines of one block for every curve: the MDCT lines are loaded once per task, and the next curve's (or
// the next task's first curve's) floor and flags are in flight while the current curve is computed.
struct CqnCurve {
  int limit, sliding_lowpass;   // coupling_pointlimit[blockflag][blob], sliding_lowpass[W][blob]
  float prepoint, postpoint;    // the coupling point amplitudes of the blob
};
struct CqnCurveTab { CqnCurve c[2][VB200_PACKETBLOBS]; };   // [blocktype][blob]

template <int CH>
__global__ void __launch_bounds__(128)
k_cqn_fast_curves(CqnDev Q0, CqnDev Q1, const __grid_constant__ CqnCurveTab T,
                  const vb200_block_desc *__restrict__ desc, int nblocks, long long blob_blocks,
                  const float *__restrict__ mdct, int *__restrict__ iwork, const int *__restrict__ nonzero) {
  constexpr int NB = VB200_PACKETBLOBS;
  __shared__ float s_fromdB[256];
  __shared__ CqnCurve s_cur[2 * NB];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_fromdB[i] = __ldg(Q0.fromdB + i);
  if (threadIdx.x < 2 * NB) s_cur[threadIdx.x] = (&T.c[0][0])[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int n = Q0.n, csh = 31 - __clz(n >> 5);          // n is a power of two: chunks = 1 << csh
  const int tasks = nblocks << csh, stride = gridDim.x * wpb;   // the launcher keeps tasks < 2^31
  const size_t brows = (size_t)blob_blocks * CH;         // rows between consecutive curves
  const bool coupled = CH == 2 && Q0.steps > 0;
  const int c0 = coupled ? __ldg(Q0.mag) : 0, c1 = coupled ? __ldg(Q0.ang) : 1;
  float mv[CH], nmv[CH];
  int il[CH], nil[CH], nzr[CH], nnz[CH];
  // curve k's floor and flags of task t; with curve 0 also the task's MDCT lines
  auto fetch = [&](int t, int k) {
    const int blk = t >> csh, line = ((t & ((1 << csh) - 1)) << 5) + lane;
#pragma unroll
    for (int s = 0; s < CH; s++) {
      const size_t row = (size_t)blk * CH + (s == 0 ? c0 : c1), crow = (size_t)k * brows + row;
      nnz[s] = __ldg(nonzero + crow);
      nil[s] = __ldcs(iwork + crow * n + line);
      if (k == 0) nmv[s] = __ldcs(mdct + row * n + line);
    }
  };
  int t = blockIdx.x * wpb + wid;
  if (t < tasks) fetch(t, 0);
  for (; t < tasks; t += stride) {
    const int blk = t >> csh, line = ((t & ((1 << csh) - 1)) << 5) + lane;
    const int bt = desc && desc[blk].blocktype ? 1 : 0;
    CqnDev Q = cqn_pick(Q0, Q1, bt);
#pragma unroll
    for (int s = 0; s < CH; s++) mv[s] = nmv[s];
#pragma unroll 1
    for (int k = 0; k < NB; k++) {
#pragma unroll
      for (int s = 0; s < CH; s++) { il[s] = nil[s]; nzr[s] = nnz[s]; }
      if (k + 1 < NB) fetch(t, k + 1);
      else if (t < tasks - stride) fetch(t + stride, 0);
      const CqnCurve cv = s_cur[bt * NB + k];
      Q.limit = cv.limit; Q.sliding_lowpass = cv.sliding_lowpass; Q.prepoint = cv.prepoint; Q.postpoint = cv.postpoint;
      int out[CH];
      cqn_fast_lines<CH>(Q, s_fromdB, coupled, line, lane, mv, il, nzr, out);
      int *iw = iwork + ((size_t)k * brows + (size_t)blk * CH) * n + line;
      __stcs(iw + (size_t)c0 * n, out[0]);
      if (CH == 2) __stcs(iw + (size_t)c1 * n, out[CH - 1]);
    }
  }
}

// smem per warp: raw, quant, floor (float), flag and quantised value (int): CQN_COLS * ch * 32 words
#define CQN_COLS 5
__global__ void __launch_bounds__(128)
k_cqn(CqnDev Q0, CqnDev Q1, const vb200_block_desc *__restrict__ desc, int nblocks,
      const float *__restrict__ mdct, int *__restrict__ iwork, const int *__restrict__ nonzero) {
  // desc == NULL: every block uses Q0; else block b uses the psy look of its blocktype
  // (b->psy + blocktype + (W?2:0), lib/mapping0.c:250), Q0 / Q1
  extern __shared__ __align__(16) float sm[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int n = Q0.n, ch = Q0.ch;
  float *raw = sm + (size_t)wid * CQN_COLS * ch * 32;
  float *quant = raw + ch * 32, *flr = quant + ch * 32;
  int *flag = reinterpret_cast<int *>(flr + ch * 32);
  int *iq = flag + ch * 32;
  int *nz = reinterpret_cast<int *>(sm + (size_t)wpb * CQN_COLS * ch * 32) + wid * ch;   // [ch] per warp
  const int chunks = n >> 5;
  const long tasks = (long)nblocks * chunks;
  for (long t = (long)blockIdx.x * wpb + wid; t < tasks; t += (long)gridDim.x * wpb) {
    const int blk = (int)(t / chunks), line = (int)(t % chunks) * 32 + lane;
    const CqnDev Q = cqn_pick(Q0, Q1, desc && desc[blk].blocktype);
    const int width = Q.partition;
    const int i = line & ~(width - 1), j = line - i;       // partition start, index inside it
    const float *m = mdct + (size_t)blk * ch * n;
    int *iw = iwork + (size_t)blk * ch * n;
    for (int k = lane; k < ch; k += 32) nz[k] = nonzero[(size_t)blk * ch + k];
    __syncwarp();
    for (int k = 0; k < ch; k++) {
      int out = 0;
      float R = 0.f, Qe = 0.f, F = 1e-10f; int G = 0;
      if (nz[k]) {
        const float mv = m[(size_t)k * n + line];
        const float fl = __ldg(Q.fromdB + iw[(size_t)k * n + line]);
        const float point = j >= Q.limit - i ? Q.postpoint : Q.prepoint;      // flag_lossless
        G = (fabsf(mv) / fl < point) ? 0 : 1;
        Qe = R = mv * mv;
        if (mv < 0.f) R *= -1.f;
        F = fl * fl;
        cqn_normalize(Q, R, Qe, F, false, 0, i, j, out, width, lane);
      }
      raw[k * 32 + lane] = R; quant[k * 32 + lane] = Qe; flr[k * 32 + lane] = F; flag[k * 32 + lane] = nz[k] ? G : 0;
      iq[k * 32 + lane] = out;
      // note: flag_lossless results are kept for the coupling below; a zero channel has flag 0
    }
    for (int step = 0; step < Q.steps; step++) {
      const int Mi = Q.mag[step], Ai = Q.ang[step];
      if (!(nz[Mi] || nz[Ai])) continue;
      __syncwarp();
      if (lane == 0) { nz[Mi] = 1; nz[Ai] = 1; }
      __syncwarp();
      float reM = raw[Mi * 32 + lane], reA = raw[Ai * 32 + lane];
      float qeM = quant[Mi * 32 + lane], qeA = quant[Ai * 32 + lane];
      float fM = flr[Mi * 32 + lane], fA = flr[Ai * 32 + lane];
      int gM = flag[Mi * 32 + lane], gA = flag[Ai * 32 + lane];
      int iM = iq[Mi * 32 + lane], iA = iq[Ai * 32 + lane];
      if (j < Q.sliding_lowpass - i) {
        if (gM || gA) {                                    // lossless: integer square-polar map
          const int A = iM, B = iA;
          reM = fabsf(reM) + fabsf(reA);
          qeM = qeM + qeA;
          gM = gA = 1;
          if (abs(A) > abs(B)) {
            iA = (A > 0 ? A - B : B - A);
          } else {
            iA = (B > 0 ? A - B : B - A);
            iM = B;
          }
          if (iA >= abs(iM) * 2) { iA = -iA; iM = -iM; }
        } else {                                           // point stereo
          if (j < Q.limit - i) {
            reM += reA;
            qeM = fabsf(reM);
          } else {
            const float e = fabsf(reM) + fabsf(reA);
            qeM = e;
            reM = (reM + reA < 0.f) ? -e : e;
          }
          reA = qeA = 0.f;
          gA = 1;
          iA = 0;
        }
      }
      fM = fA = fM + fA;
      cqn_normalize(Q, reM, qeM, fM, true, gM, i, j, iM, width, lane);
      raw[Mi * 32 + lane] = reM; raw[Ai * 32 + lane] = reA;
      quant[Mi * 32 + lane] = qeM; quant[Ai * 32 + lane] = qeA;
      flr[Mi * 32 + lane] = fM; flr[Ai * 32 + lane] = fA;
      flag[Mi * 32 + lane] = gM; flag[Ai * 32 + lane] = gA;
      iq[Mi * 32 + lane] = iM; iq[Ai * 32 + lane] = iA;
    }
    for (int k = 0; k < ch; k++) iw[(size_t)k * n + line] = iq[k * 32 + lane];
    __syncwarp();
  }
}

// nonzero[] propagation over coupling steps (lib/psy.c:1203-1212); runs after k_cqn.  blockIdx.y = curve,
// curve y's flags start blob_blocks blocks after curve y-1's (one curve: gridDim.y = 1)
__global__ void k_cqn_nonzero(int nblocks, int ch, int steps, const int *__restrict__ mag,
                              const int *__restrict__ ang, int *__restrict__ nonzero, long long blob_blocks) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  int *nz = nonzero + ((size_t)blockIdx.y * (size_t)blob_blocks + b) * ch;
  for (int s = 0; s < steps; s++)
    if (nz[mag[s]] || nz[ang[s]]) { nz[mag[s]] = 1; nz[ang[s]] = 1; }
}

}  // namespace vb200
