// vb200_env.cuh — envelope / block-switch detector (SURVEY §8 f2): lib/envelope.c.
//
// k_env_spectrum   item = (stream, channel, step): squared-sine window, mdct_forward(128)
//                  (lib/envelope.c:113-118), the near-DC energy `temp` (:125) and the 32 half-dB
//                  pair powers (:147-149).  Independent items: one warp each, 4 warps per CTA.
// k_env_spectrum_var  the same with a first step and a step count per stream (carried streams)
// k_env_filter     everything of _ve_amp that carries state (near-DC running sum :124-145, spreading
//                  and limiting :150-157, band amplitudes and the 17-deep amplitude history :162-203,
//                  triggers :206-210) plus the stretch logic of _ve_envelope_search (:239-266).
//                  Sequential over steps, channels coupled through `stretch`: one warp per stream,
//                  lane = spectral pair for the spreading, lane = band for the history.
// The state lives in global memory in the reference's own envelope_filter_state layout.
#pragma once
#include "vb200_kernels.cuh"

namespace vb200 {

struct EnvDev {
  XformDev X;                 // mdct_init(128)
  const float *win;           // [128] sin^2 window, lib/envelope.c:47-50
  const float *bwin;          // [VE_BANDS][8] band windows, :63-66
  float total[VB200_VE_BANDS];
  int begin[VB200_VE_BANDS], end[VB200_VE_BANDS];
  float preecho[VB200_VE_BANDS], postecho[VB200_VE_BANDS];
  float stretch_penalty, minenergy;
};

constexpr int ENV_N = 128, ENV_STEP = 64, ENV_AMP = 17, ENV_NEARDC = 15;
constexpr int ENV_WARPS = 4;

struct EnvSrc { const void *base; int fmt; long long stride; int ch; };

// VAR: stream s analyses steps first_ps[s] + first_step + j for j < count_ps[s] - first_step (first_step is the
// chunk's offset then); items past a stream's count read its first samples and write nothing.
template <bool VAR>
__device__ __forceinline__ void env_spectrum_body(const EnvDev &E, const EnvSrc &src, int nstreams, int first_step,
                                                  int nsteps, float *__restrict__ temps, float *__restrict__ vals,
                                                  const int *__restrict__ first_ps, const int *__restrict__ count_ps) {
  __shared__ __align__(16) float s_in[ENV_WARPS][ENV_N];
  __shared__ __align__(16) float s_w[ENV_WARPS][ENV_N];
  __shared__ __align__(16) float s_out[ENV_WARPS][ENV_N / 2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long items = (long)nstreams * src.ch * nsteps;
  const long stride = (long)gridDim.x * ENV_WARPS;
  // every warp runs the same number of iterations: dev_mdct_forward synchronises the whole CTA
  const long iters = (items + stride - 1) / stride;
  for (long it = 0; it < iters; it++) {
    long item = (long)blockIdx.x * ENV_WARPS + wid + it * stride;
    const bool valid = item < items;
    if (!valid) item = items - 1;
    const int j = (int)(item % nsteps);
    const long sc = item / nsteps;                       // stream * ch + c
    long s0 = (long)ENV_STEP * (first_step + j);
    bool store = valid;
    if (VAR) {
      const long sst = sc / src.ch;
      store = valid && first_step + j < count_ps[sst];
      s0 = store ? (long)ENV_STEP * (first_ps[sst] + first_step + j) : 0;
    }
    // a stride-bounded step range (the raw-PCM calls): a CTA whose warps all lie past their streams' counts has
    // nothing to compute
    if (VAR && !__syncthreads_or(store)) continue;
    if (src.fmt == VB200_PCM_S16_INTERLEAVED) {
      const long st = sc / src.ch; const int c = (int)(sc - st * src.ch);
      const short *p = reinterpret_cast<const short *>(src.base) + ((long long)st * src.stride + s0) * src.ch + c;
      for (int i = lane; i < ENV_N; i += 32) s_in[wid][i] = ((float)__ldg(p + (long long)i * src.ch) / 32768.f) * __ldg(E.win + i);
    } else {
      const float *p = reinterpret_cast<const float *>(src.base) + sc * src.stride + s0;
      for (int i = lane; i < ENV_N; i += 32) s_in[wid][i] = __ldg(p + i) * __ldg(E.win + i);
    }
    __syncthreads();
    dev_mdct_forward<ENV_N>(E.X, s_in[wid], s_w[wid], s_out[wid], lane, 32);
    __syncthreads();
    if (VAR ? store : valid) {
      const float2 v = *reinterpret_cast<const float2 *>(&s_out[wid][2 * lane]);
      const float pw = v.x * v.x + v.y * v.y;
      vals[item * 32 + lane] = todB_dev(pw) * .5f;
      if (lane == 0) {
        const float v0 = s_out[wid][0], v1 = s_out[wid][1], v2 = s_out[wid][2];
        // vec[0]*vec[0]+.7*vec[1]*vec[1]+.2*vec[2]*vec[2]: the first product is fp32, the rest fp64
        temps[item] = (float)(((double)(v0 * v0) + (.7 * (double)v1) * (double)v1) + (.2 * (double)v2) * (double)v2);
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(32 * ENV_WARPS)
k_env_spectrum(EnvDev E, EnvSrc src, int nstreams, int first_step, int nsteps,
               float *__restrict__ temps, float *__restrict__ vals) {
  env_spectrum_body<false>(E, src, nstreams, first_step, nsteps, temps, vals, nullptr, nullptr);
}

__global__ void __launch_bounds__(32 * ENV_WARPS)
k_env_spectrum_var(EnvDev E, EnvSrc src, int nstreams, int j0, int nsteps, float *__restrict__ temps,
                   float *__restrict__ vals, const int *__restrict__ first_ps, const int *__restrict__ count_ps) {
  env_spectrum_body<true>(E, src, nstreams, j0, nsteps, temps, vals, first_ps, count_ps);
}

__global__ void __launch_bounds__(32 * ENV_WARPS)
k_env_filter(EnvDev E, int nstreams, int ch, int nsteps, int ret_stride, int ret_off,
             const float *__restrict__ temps, const float *__restrict__ vals,
             int *__restrict__ state, unsigned char *__restrict__ ret, const int *__restrict__ steps_per_stream) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int st = blockIdx.x * ENV_WARPS + (threadIdx.x >> 5);
  if (st >= nstreams) return;
  int *sw = state + (size_t)st * VB200_VE_STATE_WORDS(ch);
  int stretch_state = sw[0];
  const int band = lane < VB200_VE_BANDS ? lane : 0;
  const int bbegin = E.begin[band], bend = lane < VB200_VE_BANDS ? E.end[band] : 0;
  const float btotal = E.total[band], pre_t = E.preecho[band], post_t = E.postecho[band];
  float bw[8];
#pragma unroll
  for (int i = 0; i < 8; i++) bw[i] = __ldg(E.bwin + band * 8 + i);
  // streams may have different amounts of new data: stream st only runs its first steps_per_stream[st] steps
  int lim = steps_per_stream ? steps_per_stream[st] - ret_off : nsteps;
  if (lim > nsteps) lim = nsteps;
  for (int j = 0; j < lim; j++) {
    stretch_state++;                                            // lib/envelope.c:242-244
    if (stretch_state > 24) stretch_state = 24;
    const int half = stretch_state / 2;
    const int stretch = half > 2 ? half : 2;                    // :103
    float penalty = E.stretch_penalty - (float)(half - 2);      // :104-106
    if (penalty < 0.f) penalty = 0.f;
    if (penalty > E.stretch_penalty) penalty = E.stretch_penalty;
    unsigned r = 0;
    for (int c = 0; c < ch; c++) {
      const size_t item = ((size_t)st * ch + c) * nsteps + j;
      const float val = __ldcs(vals + item * 32 + lane);
      int *f0 = sw + 1 + (size_t)c * VB200_VE_BANDS * VB200_VE_FILTER_WORDS;
      float decay = 0.f;
      if (lane == 0) {                                          // near-DC spreading, :124-145
        const float temp = __ldcs(temps + item);
        float *nearDC = reinterpret_cast<float *>(f0 + 18);
        float *acc = reinterpret_cast<float *>(f0 + 33), *part = reinterpret_cast<float *>(f0 + 34);
        const int ptr = f0[35];
        if (ptr == 0) {
          decay = *part + temp; *acc = decay; *part = temp;
        } else {
          decay = *acc + temp; *acc = decay; *part = *part + temp;
        }
        *acc = *acc - nearDC[ptr];
        nearDC[ptr] = temp;
        decay = decay * .0625f;                                 // *(1./16): exact either way
        f0[35] = ptr + 1 >= ENV_NEARDC ? 0 : ptr + 1;
        decay = (float)((double)todB_dev(decay) * .5 - (double)15.f);
      }
      decay = __shfl_sync(full, decay, 0);
      // spreading and limiting (:150-157): lane k sees decay after k subtractions of 8 (each one
      // rounds to fp32, so they are replayed, not multiplied)
#pragma unroll 1
      for (int t = 0; t < 31; t++) if (t < lane) decay = decay - 8.f;
      float v = val;
      if (v < decay) v = decay;
      if (v < E.minenergy) v = E.minenergy;
      // band amplitude (:167-170): lane = band
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const float x = __shfl_sync(full, v, (bbegin + i) & 31);
        if (i < bend) acc = acc + x * bw[i];
      }
      acc = acc * btotal;
      if (lane < VB200_VE_BANDS) {                              // amplitude history, :173-203
        int *fb = f0 + lane * VB200_VE_FILTER_WORDS;
        float *ampbuf = reinterpret_cast<float *>(fb);
        const int cur = fb[17];
        int p = cur - 1; if (p < 0) p += ENV_AMP;
        const float prev = ampbuf[p];
        const float postmax = acc < prev ? prev : acc, postmin = acc > prev ? prev : acc;
        float premax = -99999.f, premin = 99999.f;
        for (int i = 0; i < stretch; i++) {
          p--; if (p < 0) p += ENV_AMP;
          const float a = ampbuf[p];
          premax = premax < a ? a : premax;
          premin = premin > a ? a : premin;
        }
        const float valmin = postmin - premin, valmax = postmax - premax;
        ampbuf[cur] = acc;
        fb[17] = cur + 1 >= ENV_AMP ? 0 : cur + 1;
        if (valmax > pre_t + penalty) r |= 5u;                   // :206-210
        if (valmin < post_t - penalty) r |= 2u;
      }
      __syncwarp();
    }
    r = __reduce_or_sync(full, r);
    if (lane == 0) ret[(size_t)st * ret_stride + ret_off + j] = (unsigned char)r;
    if (r & 4) stretch_state = -1;                              // :266
  }
  if (lane == 0) sw[0] = stretch_state;
}

}  // namespace vb200
