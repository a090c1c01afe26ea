// vb200_lpc.cuh — the LPC extrapolation of vorbis_analysis_wrote (lib/block.c:426-529, lib/lpc.c) on the device, for
// the raw-PCM calls (vb200_encode_pcm_packets[_managed]) and the stage call vb200_lpc_extrapolate.
//
//   k_lpc_filter<M>     one warp per job (a window of one channel): the autocorrelation of vorbis_lpc_from_data with
//                       one lane per lag (lane 0 also takes lag 32 when M = 32), each a sequential double sum over i
//                       ascending, the window staged through shared memory in tiles; then lane 0 runs Levinson-Durbin,
//                       the .99^k damping and the conversion to float.  Writes the M coefficients and the M prime
//                       samples (the window's last M, where vorbis_lpc_predict starts).
//   k_pcm_timeline<T>   T = false: one CTA per (stream, channel) writes the planar float timeline up to eof: the input
//                       (int16 converted as encoder_example does), and the preamble part by a serial replay of
//                       vorbis_lpc_predict from the carried order-16 filter.  T = true: one thread per (stream,
//                       channel) writes the tail part by a serial replay of the carried order-32 filter.
//   k_lpc_predict<M>    one thread per row: vorbis_lpc_predict from k_lpc_filter's coefficients and prime (stage call)
// Every sum runs in the reference's order; the TU is compiled with -fmad=false, so nothing is contracted.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

constexpr int LPC_PRE = 16, LPC_TAIL = 32;                      // the orders of lib/block.c:428 and :475
constexpr int LPC_FILTER_FLOATS = 2 * (LPC_PRE + LPC_TAIL);     // per channel: pre coef, pre prime, tail coef, prime
constexpr int LPC_WARPS = 4, LPC_TILE = 1024;

// window sample i of one job: the float at off + i * step of src, or the int16 there / 32768.f
struct LpcJob {
  const void *src;
  long long off, step, n;    // n: the window length
  int s16, pad;
  float *coef, *prime;       // [M] each
};

__device__ __forceinline__ float lpc_at(const LpcJob &J, long long i) {
  const long long k = J.off + i * J.step;
  return J.s16 ? (float)((const short *)J.src)[k] / 32768.f : ((const float *)J.src)[k];
}

// guard: the `> order*2` safety of lib/block.c:434 and :494 (n <= 2M: zero coefficients and prime, which replay as
// exact zeros, as the reference's untouched or memset samples are)
template <int M>
__global__ void __launch_bounds__(32 * LPC_WARPS) k_lpc_filter(const LpcJob *__restrict__ jobs, int njobs, int guard) {
  static_assert(M <= 32, "one lane per lag");
  __shared__ float s_w[LPC_WARPS][32 + LPC_TILE];
  __shared__ double s_aut[LPC_WARPS][M + 1], s_lpc[LPC_WARPS][M];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float *w = s_w[wid] + 32;  // w[k]: window sample t0 + k; w[-32 .. -1]: the 32 before it
  for (int j = blockIdx.x * LPC_WARPS + wid; j < njobs; j += gridDim.x * LPC_WARPS) {
    const LpcJob J = jobs[j];
    const long long n = J.n;
    if (guard && n <= 2 * M) {
      if (lane < M) { J.coef[lane] = 0.f; J.prime[lane] = 0.f; }
      continue;
    }
    // lib/lpc.c:68-73: aut[lag] = sum over i = lag .. n-1 ascending of (double)data[i] * data[i-lag]
    double d = 0., d32 = 0.;
    const bool mine = lane <= M && lane < 32, hi = M == 32 && lane == 0;
    for (long long t0 = 0; t0 < n; t0 += LPC_TILE) {
      const int cnt = (int)min((long long)LPC_TILE, n - t0);
      __syncwarp();
      if (t0) w[lane - 32] = w[LPC_TILE - 32 + lane];     // every tile before the last is full
      __syncwarp();
      for (int k = lane; k < cnt; k += 32) w[k] = lpc_at(J, t0 + k);
      __syncwarp();
      if (mine)
        for (int k = (int)max(0LL, lane - t0); k < cnt; k++) d += (double)w[k] * (double)w[k - lane];
      if (hi)
        for (int k = (int)max(0LL, 32 - t0); k < cnt; k++) d32 += (double)w[k] * (double)w[k - 32];
    }
    if (mine) s_aut[wid][lane] = d;
    if (hi) s_aut[wid][32 % (M + 1)] = d32;
    if (lane < M) J.prime[lane] = lpc_at(J, n - M + lane);
    __syncwarp();
    if (lane == 0) {
      // lib/lpc.c:77-124: Levinson-Durbin in double with the -100 dB floor, the damping, then float
      const double *aut = s_aut[wid];
      double *lpc = s_lpc[wid];
      double error = aut[0] * (1. + 1e-10);
      const double epsilon = 1e-9 * aut[0] + 1e-10;
      int i = 0;
      for (; i < M; i++) {
        double r = -aut[i + 1];
        if (error < epsilon) break;
        for (int k = 0; k < i; k++) r -= lpc[k] * aut[i - k];
        r /= error;
        lpc[i] = r;
        int k = 0;
        for (; k < i / 2; k++) {
          const double tmp = lpc[k];
          lpc[k] += r * lpc[i - 1 - k];
          lpc[i - 1 - k] += r * tmp;
        }
        if (i & 1) lpc[k] += lpc[k] * r;
        error *= 1. - r * r;
      }
      for (; i < M; i++) lpc[i] = 0.;
      double damp = .99;
      for (int k = 0; k < M; k++) {
        lpc[k] *= damp;
        damp *= .99;
      }
      for (int k = 0; k < M; k++) J.coef[k] = (float)lpc[k];
    }
    __syncwarp();
  }
}

// vorbis_lpc_predict (lib/lpc.c:132-159) from coef [M] and prime [M]: emit(k, y) for the outputs k < count, in order
template <int M, class F>
__device__ __forceinline__ void lpc_replay(const float *coef, const float *prime, long long count, F &&emit) {
  float c[M], wk[M];
#pragma unroll
  for (int j = 0; j < M; j++) { c[j] = coef[j]; wk[j] = prime[j]; }
  for (long long k = 0; k < count; k++) {
    float y = 0.f;
#pragma unroll
    for (int j = 0; j < M; j++) y -= wk[j] * c[M - 1 - j];
#pragma unroll
    for (int j = 0; j < M - 1; j++) wk[j] = wk[j + 1];
    wk[M - 1] = y;
    emit(k, y);
  }
}

// one stream of a raw-PCM call as the host planned it
struct PcmStream {
  long long base;       // the timeline sample at arena column 0 (the encode carry's base)
  long long raw_base;   // the input sample at index 0 of the caller's buffer
  long long len;        // arena columns this call passes (0: no preamble yet, or done)
  long long eof;        // the timeline eof (preamble + samples written) once ended, else 0
};

struct PcmTimelineArgs {
  const void *in;            // the caller's buffer: VB200_PCM_F32_PLANAR or VB200_PCM_S16_INTERLEAVED
  int s16, ch, half;         // half = blocksizes[1]/2, where the input starts on the timeline
  long long in_stride, tl_stride;
  const PcmStream *st;
  const float *filt;         // [nstreams][ch][LPC_FILTER_FLOATS]
  float *tl;                 // [nstreams][ch][tl_stride], column 0 = timeline sample st.base
  int nstreams;
};

template <bool TAIL>
__global__ void __launch_bounds__(256) k_pcm_timeline(PcmTimelineArgs A) {
  const long long pairs = (long long)A.nstreams * A.ch;
  if constexpr (!TAIL) {
    for (long long q = blockIdx.x; q < pairs; q += gridDim.x) {
      const int s = (int)(q / A.ch), c = (int)(q % A.ch);
      const PcmStream P = A.st[s];
      if (!P.len) continue;
      float *dst = A.tl + q * A.tl_stride - P.base;          // dst[t]: timeline sample t
      const long long lim = P.eof ? P.eof : P.base + P.len;
      const bool pre = P.base < A.half;
      if (pre && threadIdx.x == 0) {
        // _preextrapolate_helper (lib/block.c:455-461): output k lands on timeline sample half - 1 - k
        const float *f = A.filt + q * LPC_FILTER_FLOATS;
        lpc_replay<LPC_PRE>(f, f + LPC_PRE, A.half - P.base, [&](long long k, float y) { dst[A.half - 1 - k] = y; });
      }
      const int first = pre ? 1 : 0, nth = blockDim.x - first;
      if ((int)threadIdx.x < first) continue;
      for (long long t = max(P.base, (long long)A.half) + threadIdx.x - first; t < lim; t += nth) {
        const long long i = t - A.half - P.raw_base;
        dst[t] = A.s16 ? (float)((const short *)A.in)[((long long)s * A.in_stride + i) * A.ch + c] / 32768.f
                       : ((const float *)A.in)[q * A.in_stride + i];
      }
    }
  } else {
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < pairs; q += (long long)gridDim.x * blockDim.x) {
      const PcmStream P = A.st[q / A.ch];
      if (!P.len || !P.eof) continue;
      float *dst = A.tl + q * A.tl_stride - P.base;
      const float *f = A.filt + q * LPC_FILTER_FLOATS + 2 * LPC_PRE;
      // lib/block.c:504-505: output k lands on timeline sample eof + k
      lpc_replay<LPC_TAIL>(f, f + LPC_TAIL, P.base + P.len - P.eof, [&](long long k, float y) {
        if (P.eof + k >= P.base) dst[P.eof + k] = y;
      });
    }
  }
}

template <int M>
__global__ void k_lpc_predict(int nrows, const float *__restrict__ coef, const float *__restrict__ prime, int count,
                              float *out, long long out_stride) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nrows) return;
  float *o = out + (long long)r * out_stride;
  lpc_replay<M>(coef + (long long)r * M, prime + (long long)r * M, count, [&](long long k, float y) { o[k] = y; });
}
