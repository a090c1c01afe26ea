// vb200_floor1.cuh — floor 1 on the device (SURVEY §8 f1).
//
// k_floor1_fit     floor1_fit            lib/floor1.c:576-729
//                    accumulate_fit      :406-454   per-gap integer sums, all lanes per gap + redux
//                    fit_line            :456-521   fp64 chains over per-gap terms computed once per row,
//                                                   one lane per chain (12 lanes for the two fits of a
//                                                   split, one fit per half-warp), summed in gap order
//                    inspect_error       :523-566   lanes over x; the Bresenham line in closed form at a lane's first x,
//                                                   then 32 abscissae per step with an integer error term; integer
//                                                   compares when maxover / maxunder are whole numbers
//                    post prediction     :702-727   one dependency level per step (lvl_*), one lane per post
//                    greedy splitting    :627-700   warp-uniform control flow, state in shared memory
// k_floor1_render  floor1_encode minus the bit packing  :765-832 (quantise, predict/flag), :919-945
//                    (render_line0 :376-403 into ilogmask)
//
// One warp per (block, channel) row.  All values are integers except vorbis_dBquant (fp32,
// :278-283) and the line fit (fp64); the library is built -fmad=false so every expression rounds
// where the C source rounds.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

struct Floor1Dev {                     // vorbis_look_floor1 (lib/codec_internal.h:138-155) in 16-bit
  int posts, n, mult, pad;
  float maxover, maxunder, maxerr, twofitweight, twofitatten;
  short postlist[VB200_VIF_POSIT + 3], sorted[VB200_VIF_POSIT + 3];
  short fwd[VB200_VIF_POSIT + 3], rev[VB200_VIF_POSIT + 3];
  short lo[VB200_VIF_POSIT + 1], hi[VB200_VIF_POSIT + 1];
  float prcp[VB200_VIF_POSIT + 1];     // 1 / (postlist[hi[i]] - postlist[lo[i]])
  // posts 2..P-1 ordered by dependency level (a post is predicted from its two neighbours lo[], hi[], which have
  // smaller indices): level 0 needs only posts 0 and 1, level k only levels < k.  lvl_start[k]..lvl_start[k+1]
  // index lvl_order[]; the prediction passes run one level per step, one lane per post
  int nlevels;
  int int_thresh, maxover_i, maxunder_i;   // maxover / maxunder as integers when they are whole numbers (inspect_error)
  unsigned char lvl_order[VB200_VIF_POSIT + 1], lvl_start[VB200_VIF_POSIT + 5];
};
static_assert(sizeof(Floor1Dev) % 4 == 0, "Floor1Dev is copied as words");
static_assert((sizeof(Floor1Dev) * VB200_MAX_SUBMAPS) % 8 == 0, "the per-warp fp64 terms follow the floor table in shared memory");

struct Floor1Args {
  const Floor1Dev *floors;             // [VB200_MAX_SUBMAPS] of this block size
  const unsigned char *chmux;          // [channels]
  int channels, floor_sel, nrows, n;   // n = spectral lines per row (row stride)
};

#define F1_WARPS 8
#define F1_ACC 12                      // xa ya x2a y2a xya an | xb yb x2b y2b xyb bn
#define F1_STATE (3 * (VB200_VIF_POSIT + 2) + 3 * ((VB200_VIF_POSIT + 2 + 1) / 2))   // A, B, out int; lon, hin, memo short

__host__ __device__ inline size_t floor1_fit_smem_per_warp(int n) {
  return ((sizeof(unsigned short) * (size_t)n + 7) & ~(size_t)7) + sizeof(int) * ((VB200_VIF_POSIT + 1) * F1_ACC + F1_STATE);
}

__device__ __forceinline__ int f1_dBquant(float x) {               // lib/floor1.c:278-283
  int i = (int)(x * 7.3142857f + 1023.5f);
  return i > 1023 ? 1023 : (i < 0 ? 0 : i);
}

// render_point (lib/floor1.c:362-374).  rcp = 1/(x1-x0) as fp32: ady*(x-x0) < 2^22 is exact in
// fp32, the quotient estimate is off by at most one and the remainder test makes it exact
__device__ __forceinline__ int f1_point(int x0, int x1, int y0, int y1, int x, float rcp) {
  y0 &= 0x7fff; y1 &= 0x7fff;
  const int dy = y1 - y0, adx = x1 - x0, ady = abs(dy);
  const int num = ady * (x - x0);
  int off = __float2int_rz((float)num * rcp);
  const int r = num - off * adx;
  if (r < 0) off--;
  else if (r >= adx) off++;
  return dy < 0 ? y0 - off : y0 + off;
}

// the integer line of render_line0 / inspect_error: after k steps the error term has wrapped
// floor(k*ady/adx) times, each wrap adding (sy - base)
struct F1Line {
  int x0, y0, adx, base, ady, step;
  float rcp;
  __device__ __forceinline__ F1Line(int x0_, int x1, int y0_, int y1) {
    x0 = x0_; y0 = y0_;
    const int dy = y1 - y0;
    adx = x1 - x0;
    base = dy / adx;
    step = dy < 0 ? -1 : 1;
    ady = abs(dy) - abs(base * adx);
    rcp = 1.f / (float)adx;
  }
  // floor(k*ady/adx) without the integer-division sequence: k*ady < 2^22 is exact in fp32, the
  // estimate is off by at most one, and the remainder test makes it exact
  __device__ __forceinline__ int at(int x) const {
    const int k = x - x0, num = k * ady;
    int q = __float2int_rz((float)num * rcp);
    const int r = num - q * adx;
    if (r < 0) q--;
    else if (r >= adx) q++;
    return y0 + k * base + q * step;
  }
};

__device__ __forceinline__ int f1_postY(const int *A, const int *B, int pos) {
  const int a = A[pos], b = B[pos];
  if (a < 0) return b;
  if (b < 0) return a;
  return (a + b) >> 1;
}

// inspect_error: 1 = this line is not good enough.  q[x] = dBquant(mask[x]) | (audible << 15)
__device__ __forceinline__ int f1_inspect(const Floor1Dev &F, const unsigned short *q, int x0, int x1,
                                          int y0, int y1, int lane) {
  const F1Line L(x0, x1, y0, y1);
  int mse = 0, viol = 0;
  int x = x0 + lane;
  if (x < x1) {
    // the line at this lane's first x in closed form, then 32 abscissae per step: the error term advances by
    // (32*ady) mod adx and wraps at most once more than floor(32*ady / adx) times
    int y = L.at(x);
    int r = (x - x0) * L.ady;
    { int qq = __float2int_rz((float)r * L.rcp); int t = r - qq * L.adx; if (t < 0) t += L.adx; else if (t >= L.adx) t -= L.adx; r = t; }
    const int n32 = 32 * L.ady;
    int d32 = __float2int_rz((float)n32 * L.rcp);
    int m32 = n32 - d32 * L.adx;
    if (m32 < 0) { d32--; m32 += L.adx; } else if (m32 >= L.adx) { d32++; m32 -= L.adx; }
    const int ystep = 32 * L.base + d32 * L.step;
    const bool ith = F.int_thresh != 0;                // maxover / maxunder are whole numbers: integer compares are exact
    for (; x < x1; x += 32) {
      const int v = q[x];
      const int val = v & 0x7fff;
      mse += (y - val) * (y - val);
      if ((v & 0x8000) && (x == x0 || val)) {
        if (ith) {
          if (y + F.maxover_i < val) viol = 1;
          if (y - F.maxunder_i > val) viol = 1;
        } else {
          if ((float)y + F.maxover < (float)val) viol = 1;
          if ((float)y - F.maxunder > (float)val) viol = 1;
        }
      }
      r += m32;
      y += ystep;
      if (r >= L.adx) { r -= L.adx; y += L.step; }
    }
  }
  if (__any_sync(0xffffffffu, viol)) return 1;
  mse = __reduce_add_sync(0xffffffffu, mse);
  const int cnt = x1 - x0;
  if (F.maxover * F.maxover / (float)cnt > F.maxerr) return 0;
  if (F.maxunder * F.maxunder / (float)cnt > F.maxerr) return 0;
  if ((float)(mse / cnt) > F.maxerr) return 1;
  return 0;
}

// fit_line (lib/floor1.c:456-521) for up to two runs of gaps at once.  term[gap*6 + f] holds what
// the reference adds to chain f (xb yb x2b y2b xyb bn) for that gap, a[i].Xb + a[i].Xa * weight, in
// fp64 exactly as the C expression evaluates; it does not depend on the run, so it is computed once
// per row.  Lane 16*s + f sums chain f of side s in gap order (the order the reference adds in),
// then the lanes of a side finish that side's fit.  y[2*s], y[2*s+1] receive the fitted ends,
// return bit s = fit s was degenerate (reference ret 1).  The reference's "*y0 >= 0" endpoint terms
// never fire on this path (every call passes -200).
__device__ __forceinline__ int f1_fit_lines(const Floor1Dev &F, const double *term, int start0, int cnt0,
                                            int start1, int cnt1, int lane, int y[4]) {
  const unsigned full = 0xffffffffu;
  const int side = lane >> 4, f = lane & 15;
  const int start = side ? start1 : start0;
  const int ct = side ? cnt1 : cnt0;
  double sum = 0.0;
  if (f < 6) {
    const double *tp = term + start * 6 + f;
    for (int t = 0; t < ct; t++) sum += tp[t * 6];
  }
  const int sb = lane & 16;
  const double xb = __shfl_sync(full, sum, sb + 0), yb = __shfl_sync(full, sum, sb + 1);
  const double x2b = __shfl_sync(full, sum, sb + 2);
  const double xyb = __shfl_sync(full, sum, sb + 4), bn = __shfl_sync(full, sum, sb + 5);
  const int x0 = F.sorted[start], x1 = F.sorted[start + ct];
  const double denom = bn * x2b - xb * xb;
  int a0 = 0, a1 = 0, bad = 1;
  if (ct > 0 && denom > 0.) {
    const double A = (yb * x2b - xyb * xb) / denom;
    const double B = (bn * xyb - xb * yb) / denom;
    a0 = (int)rint(A + B * (double)x0);
    a1 = (int)rint(A + B * (double)x1);
    a0 = a0 > 1023 ? 1023 : (a0 < 0 ? 0 : a0);
    a1 = a1 > 1023 ? 1023 : (a1 < 0 ? 0 : a1);
    bad = 0;
  }
  y[0] = __shfl_sync(full, a0, 0); y[1] = __shfl_sync(full, a1, 0);
  y[2] = __shfl_sync(full, a0, 16); y[3] = __shfl_sync(full, a1, 16);
  return __shfl_sync(full, bad, 0) | (__shfl_sync(full, bad, 16) << 1);
}

__global__ void __launch_bounds__(32 * F1_WARPS)
k_floor1_fit(Floor1Args a, const float *__restrict__ logmdct, const float *__restrict__ logmask,
             int32_t *__restrict__ posts_out, int32_t *__restrict__ fit_nonzero) {
  extern __shared__ __align__(16) unsigned char f1_smem[];
  Floor1Dev *sF = reinterpret_cast<Floor1Dev *>(f1_smem);
  {
    const int words = (int)(sizeof(Floor1Dev) * VB200_MAX_SUBMAPS / 4);
    const int *src = reinterpret_cast<const int *>(a.floors);
    int *dst = reinterpret_cast<int *>(sF);
    for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char *wbase = f1_smem + sizeof(Floor1Dev) * VB200_MAX_SUBMAPS + floor1_fit_smem_per_warp(a.n) * warp;
  double *term = reinterpret_cast<double *>(wbase);          // [gaps][6], same bytes as 12 ints per gap
  int *A = reinterpret_cast<int *>(wbase) + (VB200_VIF_POSIT + 1) * F1_ACC;
  int *B = A + (VB200_VIF_POSIT + 2), *out = B + (VB200_VIF_POSIT + 2);
  short *lon = reinterpret_cast<short *>(out + (VB200_VIF_POSIT + 2));
  short *hin = lon + 2 * ((VB200_VIF_POSIT + 2 + 1) / 2), *memo = hin + 2 * ((VB200_VIF_POSIT + 2 + 1) / 2);
  unsigned short *q = reinterpret_cast<unsigned short *>(memo + 2 * ((VB200_VIF_POSIT + 2 + 1) / 2));

  for (long row = (long)blockIdx.x * F1_WARPS + warp; row < a.nrows; row += (long)gridDim.x * F1_WARPS) {
    const int sel = a.floor_sel >= 0 ? a.floor_sel : a.chmux[row % a.channels];
    const Floor1Dev &F = sF[sel];
    const int P = F.posts, n = F.n;
    const float *md = logmdct + (size_t)row * a.n, *mk = logmask + (size_t)row * a.n;
    int32_t *po = posts_out + (size_t)row * VB200_FLOOR1_STRIDE;
    __syncwarp();
    for (int x = lane; x < n; x += 32) {
      const float m = mk[x];
      const int v = f1_dBquant(m);
      q[x] = (unsigned short)(v | ((md[x] + F.twofitatten >= m) ? 0x8000 : 0));
    }
    for (int i = lane; i < P; i += 32) { A[i] = -200; B[i] = -200; lon[i] = 0; hin[i] = 1; memo[i] = -1; }
    __syncwarp();
    // accumulate_fit: one accumulator per gap, both ends inclusive
    int nonzero = 0;
    for (int j = 0; j < P - 1; j++) {
      const int x0 = F.sorted[j];
      int x1 = F.sorted[j + 1];
      if (x1 >= n) x1 = n - 1;
      int s[F1_ACC];
#pragma unroll
      for (int k = 0; k < F1_ACC; k++) s[k] = 0;
      for (int x = x0 + lane; x <= x1; x += 32) {
        const int v = q[x], val = v & 0x7fff;
        if (val) {
          if (v & 0x8000) { s[0] += x; s[1] += val; s[2] += x * x; s[3] += val * val; s[4] += x * val; s[5]++; }
          else            { s[6] += x; s[7] += val; s[8] += x * x; s[9] += val * val; s[10] += x * val; s[11]++; }
        }
      }
#pragma unroll
      for (int k = 0; k < F1_ACC; k++) s[k] = __reduce_add_sync(0xffffffffu, s[k]);
      if (lane < F1_ACC) {                               // raw sums; turned into fit_line's terms below
        int v = s[0];
#pragma unroll
        for (int k = 1; k < F1_ACC; k++) if (lane == k) v = s[k];
        reinterpret_cast<int *>(term)[j * F1_ACC + lane] = v;
      }
      nonzero += s[5];
    }
    __syncwarp();
    // what fit_line adds for a gap, chain f: (double)Xb + (double)Xa * weight (lib/floor1.c:465-474).  One
    // lane per gap turns its 12 ints into the 6 doubles in place (same 48 bytes, private to the lane).
    for (int g = lane; g < P - 1; g += 32) {
      int a[F1_ACC];
      const int *src = reinterpret_cast<const int *>(term) + g * F1_ACC;
#pragma unroll
      for (int k = 0; k < F1_ACC; k++) a[k] = src[k];
      const double w = (double)((float)(a[11] + a[5]) * F.twofitweight / (float)(a[5] + 1)) + 1.0;
#pragma unroll
      for (int f = 0; f < 6; f++) term[g * 6 + f] = (double)a[6 + f] + (double)a[f] * w;
    }
    __syncwarp();
    if (!nonzero) {                                      // the reference returns NULL
      for (int i = lane; i < VB200_FLOOR1_STRIDE; i += 32) po[i] = 0;
      if (lane == 0) fit_nonzero[row] = 0;
      continue;
    }
    int y[4];
    f1_fit_lines(F, term, 0, P - 1, 0, 0, lane, y);
    if (lane == 0) { A[0] = y[0]; B[0] = y[0]; A[1] = y[1]; B[1] = y[1]; }
    __syncwarp();
    for (int i = 2; i < P; i++) {
      const int sortpos = F.rev[i];
      const int ln = lon[sortpos], hn = hin[sortpos];
      if (memo[ln] == hn) continue;                      // this span was already judged
      const int lsortpos = F.rev[ln], hsortpos = F.rev[hn];
      const int lx = F.postlist[ln], hx = F.postlist[hn];
      const int ly = f1_postY(A, B, ln), hy = f1_postY(A, B, hn);
      __syncwarp();
      if (lane == 0) memo[ln] = (short)hn;
      if (f1_inspect(F, q, lx, hx, ly, hy, lane)) {
        const int ret = f1_fit_lines(F, term, lsortpos, sortpos - lsortpos, sortpos, hsortpos - sortpos, lane, y);
        int ly0 = y[0], ly1 = y[1], hy0 = y[2], hy1 = y[3];
        if (ret & 1) { ly0 = ly; ly1 = hy0; }
        if (ret & 2) { hy0 = ly1; hy1 = hy; }
        if (lane == 0) {
          if (ret == 3) {
            A[i] = -200; B[i] = -200;
          } else {
            B[ln] = ly0;
            if (ln == 0) A[ln] = ly0;
            A[i] = ly1; B[i] = hy0;
            A[hn] = hy1;
            if (hn == 1) B[hn] = hy1;
            if (ly1 >= 0 || hy0 >= 0) {
              for (int j = sortpos - 1; j >= 0; j--) { if (hin[j] == hn) hin[j] = (short)i; else break; }
              for (int j = sortpos + 1; j < P; j++) { if (lon[j] == ln) lon[j] = (short)i; else break; }
            }
          }
        }
      } else if (lane == 0) {
        A[i] = -200; B[i] = -200;
      }
      __syncwarp();
    }
    // posts as the reference returns them: fitted value, or predicted | 0x8000 when unused
    if (lane == 0) {
      out[0] = f1_postY(A, B, 0);
      out[1] = f1_postY(A, B, 1);
      fit_nonzero[row] = 1;
    }
    __syncwarp();
    for (int lv = 0; lv < F.nlevels; lv++) {             // out[i] depends on out[lo], out[hi] only: level by level
      for (int t = F.lvl_start[lv] + lane; t < F.lvl_start[lv + 1]; t += 32) {
        const int i = F.lvl_order[t];
        const int ln = F.lo[i - 2], hn = F.hi[i - 2];
        const int predicted = f1_point(F.postlist[ln], F.postlist[hn], out[ln], out[hn], F.postlist[i], F.prcp[i - 2]);
        const int vx = f1_postY(A, B, i);
        out[i] = (vx >= 0 && predicted != vx) ? vx : (predicted | 0x8000);
      }
      __syncwarp();
    }
    for (int i = lane; i < VB200_FLOOR1_STRIDE; i += 32) po[i] = i < P ? out[i] : 0;
  }
}

// blockIdx.y = curve: rows a.nrows of every curve, curve y's arrays start blob_rows rows after curve y-1's
// (bitrate-managed mode renders its 15 curves in one launch; one curve: gridDim.y = 1)
__global__ void __launch_bounds__(32 * F1_WARPS)
k_floor1_render(Floor1Args a, int32_t *__restrict__ posts, const int32_t *__restrict__ fit_nonzero,
                int32_t *__restrict__ ilogmask, int32_t *__restrict__ nonzero, long long blob_rows) {
  {
    const size_t b = (size_t)blockIdx.y * (size_t)blob_rows;
    posts += b * VB200_FLOOR1_STRIDE; fit_nonzero += b; ilogmask += b * a.n; nonzero += b;
  }
  __shared__ Floor1Dev sF[VB200_MAX_SUBMAPS];
  __shared__ int s_post[F1_WARPS][VB200_VIF_POSIT + 2];
  __shared__ short s_segx[F1_WARPS][VB200_VIF_POSIT + 3];
  __shared__ short s_segy[F1_WARPS][VB200_VIF_POSIT + 3];
  {
    const int words = (int)(sizeof(Floor1Dev) * VB200_MAX_SUBMAPS / 4);
    const int *src = reinterpret_cast<const int *>(a.floors);
    int *dst = reinterpret_cast<int *>(sF);
    for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int *post = s_post[warp];
  short *segx = s_segx[warp], *segy = s_segy[warp];
  for (long row = (long)blockIdx.x * F1_WARPS + warp; row < a.nrows; row += (long)gridDim.x * F1_WARPS) {
    int32_t *il = ilogmask + (size_t)row * a.n;
    if (!fit_nonzero[row]) {
      for (int x = lane; x < a.n; x += 32) il[x] = 0;
      if (lane == 0) nonzero[row] = 0;
      continue;
    }
    const int sel = a.floor_sel >= 0 ? a.floor_sel : a.chmux[row % a.channels];
    const Floor1Dev &F = sF[sel];
    const int P = F.posts;
    int32_t *pr = posts + (size_t)row * VB200_FLOOR1_STRIDE;
    __syncwarp();
    for (int i = lane; i < P; i += 32) {                 // quantise to the multiplier, :765-783
      const int p = pr[i];
      int val = p & 0x7fff;
      switch (F.mult) {
        case 1: val >>= 2; break;
        case 2: val >>= 3; break;
        case 3: val /= 12; break;
        case 4: val >>= 4; break;
      }
      post[i] = val | (p & 0x8000);
    }
    __syncwarp();
    // prediction / flag pass, :788-832, one dependency level per step.  A post reads its neighbours' VALUES (final
    // since their level) and its own flag (only posts of later levels clear it); several lanes may clear the same
    // neighbour's flag (the "used" bit, read after the pass), hence the atomic AND.
    for (int lv = 0; lv < F.nlevels; lv++) {
      for (int t = F.lvl_start[lv] + lane; t < F.lvl_start[lv + 1]; t += 32) {
        const int i = F.lvl_order[t];
        const int ln = F.lo[i - 2], hn = F.hi[i - 2];
        const int predicted = f1_point(F.postlist[ln], F.postlist[hn], post[ln], post[hn], F.postlist[i], F.prcp[i - 2]);
        if ((post[i] & 0x8000) || predicted == post[i]) {
          post[i] = predicted | 0x8000;
        } else {
          atomicAnd(post + ln, 0x7fff);
          atomicAnd(post + hn, 0x7fff);
        }
      }
      __syncwarp();
    }
    for (int i = lane; i < P; i += 32) pr[i] = post[i];
    // the posts that carry a value, in abscissa order
    int nseg = 0;
    if (lane == 0) { segx[0] = 0; segy[0] = (short)(post[0] * F.mult); }
    for (int j0 = 1; j0 < P; j0 += 32) {
      const int j = j0 + lane;
      int used = 0, cur = 0;
      if (j < P) { cur = F.fwd[j]; used = !(post[cur] & 0x8000); }
      const unsigned m = __ballot_sync(0xffffffffu, used);
      if (used) {
        const int k = nseg + __popc(m & ((1u << lane) - 1)) + 1;
        segx[k] = F.postlist[cur];
        segy[k] = (short)(post[cur] * F.mult);
      }
      nseg += __popc(m);
    }
    __syncwarp();
    for (int k = 0; k < nseg; k++) {                     // render_line0 clipped at the row length
      const int lx = segx[k], hx = segx[k + 1];
      const F1Line L(lx, hx, segy[k], segy[k + 1]);
      const int lim = hx < a.n ? hx : a.n;
      for (int x = lx + lane; x < lim; x += 32) il[x] = L.at(x);
    }
    {
      const int hx = segx[nseg], ly = segy[nseg];
      for (int x = hx + lane; x < a.n; x += 32) il[x] = ly;
    }
    if (lane == 0) nonzero[row] = 1;
  }
}

// ---- decode side: floor1_inverse2 (lib/floor1.c:1041-1086): the curve through the posts that
// carry a value (fit_value[] as floor1_inverse1 leaves it: unused posts have bit 15 set), rendered
// with render_line (:337-360, the same integer line as the encoder's render_line0) and multiplied
// into the spectrum through FLOOR1_fromdB_LOOKUP; out-of-range values are clamped to 0..255 as
// the reference guards them (:1056-1064).  One warp per (block, channel) row, in place.
__device__ __forceinline__ void dev_floor1_inverse2_row(const Floor1Dev &F, const int32_t *__restrict__ fit,
                                                        bool present, float *__restrict__ d, int n,
                                                        const float *__restrict__ fromdB,
                                                        short *segx, short *segy, int lane) {
  if (!present) {                                        // memo == NULL: the channel is silent, :1084
    for (int x = lane; x < n; x += 32) d[x] = 0.f;
    return;
  }
  const int P = F.posts;
  int nseg = 0;
  __syncwarp();
  if (lane == 0) {
    int ly = fit[0] * F.mult;
    ly = ly < 0 ? 0 : (ly > 255 ? 255 : ly);
    segx[0] = 0; segy[0] = (short)ly;
  }
  for (int j0 = 1; j0 < P; j0 += 32) {
    const int j = j0 + lane;
    int used = 0, cur = 0, hy = 0;
    if (j < P) {
      cur = F.fwd[j];
      const int fv = fit[cur];
      hy = fv & 0x7fff;
      used = hy == fv;
    }
    const unsigned m = __ballot_sync(0xffffffffu, used);
    if (used) {
      const int k = nseg + __popc(m & ((1u << lane) - 1)) + 1;
      hy *= F.mult;
      hy = hy < 0 ? 0 : (hy > 255 ? 255 : hy);
      segx[k] = F.postlist[cur];
      segy[k] = (short)hy;
    }
    nseg += __popc(m);
  }
  __syncwarp();
  for (int k = 0; k < nseg; k++) {
    const int lx = segx[k], hx = segx[k + 1];
    const F1Line L(lx, hx, segy[k], segy[k + 1]);
    const int lim = hx < n ? hx : n;
    for (int x = lx + lane; x < lim; x += 32) d[x] = d[x] * __ldg(fromdB + L.at(x));
  }
  {
    const int hx = segx[nseg];
    const float f = __ldg(fromdB + segy[nseg]);
    for (int x = hx + lane; x < n; x += 32) d[x] = d[x] * f;
  }
}

__global__ void __launch_bounds__(32 * F1_WARPS)
k_floor1_inverse2(Floor1Args a, const int32_t *__restrict__ posts, const int32_t *__restrict__ present,
                  float *__restrict__ data, const float *__restrict__ fromdB) {
  __shared__ Floor1Dev sF[VB200_MAX_SUBMAPS];
  __shared__ short s_segx[F1_WARPS][VB200_VIF_POSIT + 3];
  __shared__ short s_segy[F1_WARPS][VB200_VIF_POSIT + 3];
  {
    const int words = (int)(sizeof(Floor1Dev) * VB200_MAX_SUBMAPS / 4);
    const int *src = reinterpret_cast<const int *>(a.floors);
    int *dst = reinterpret_cast<int *>(sF);
    for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long row = (long)blockIdx.x * F1_WARPS + warp; row < a.nrows; row += (long)gridDim.x * F1_WARPS) {
    const int sel = a.floor_sel >= 0 ? a.floor_sel : a.chmux[row % a.channels];
    dev_floor1_inverse2_row(sF[sel], posts + (size_t)row * VB200_FLOOR1_STRIDE, present[row] != 0,
                            data + (size_t)row * a.n, a.n, fromdB, s_segx[warp], s_segy[warp], lane);
  }
}

#include "vb200_entropy.cuh"

// ---- decode, fused front half of mapping0_inverse for packed mixed-size streams: one CTA per
// (stream, block): channel de-coupling (lib/mapping0.c:754-779, last step first) then the floor
// multiply of every channel (:781-790), in place on the residue vectors; k_synthesis follows.
struct DecodePrepArgs {
  const Floor1Dev *floors[2];          // per block size
  const unsigned char *chmux[2];
  const int *mag[2], *ang[2];
  int steps[2], n[2];
  int ch, nblk;
  long nitems;                         // nstreams * nblk
};

// the packets of the ENTROPY instances: item it is data[off[it] .. off[it] + bytes[it])
struct DecodePackets {
  const long long *off;
  const int *bytes;
  const unsigned char *data;
};

// COUNTED (vb200_decode_dsp_resume): item it = (stream it / nblk, block it % nblk) is skipped when the block
// lies past count[stream]
// ENTROPY (vb200_decode_packets_resume): the CTA zero-fills the block's rows, one thread decodes its packet
// (ent_block) with the posts and presence in shared memory, then the de-coupling and floor multiply read them
// from there; posts / present are not read.  Dynamic shared memory: entropy_smem(E).
template <bool COUNTED, bool ENTROPY = false>
__device__ __forceinline__ void
decode_prepare_body(const DecodePrepArgs &A, const int *__restrict__ Wseq, const long long *__restrict__ coef_off,
                    float *__restrict__ res, const int32_t *__restrict__ posts, const int32_t *__restrict__ present,
                    const float *__restrict__ fromdB, const int *__restrict__ count,
                    const EntDev *E = nullptr, DecodePackets P = DecodePackets{}) {
  __shared__ Floor1Dev sF[2][VB200_MAX_SUBMAPS];
  __shared__ short s_segx[4][VB200_VIF_POSIT + 3];
  __shared__ short s_segy[4][VB200_VIF_POSIT + 3];
  for (int w = 0; w < 2; w++) {
    const int words = (int)(sizeof(Floor1Dev) * VB200_MAX_SUBMAPS / 4);
    const int *src = reinterpret_cast<const int *>(A.floors[w]);
    int *dst = reinterpret_cast<int *>(sF[w]);
    for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long it = blockIdx.x; it < A.nitems; it += gridDim.x) {
    if constexpr (COUNTED)
      if ((int)it % A.nblk >= count[(int)it / A.nblk]) continue;   // nitems fits an int (grid_for)
    const int W = Wseq[it] ? 1 : 0, n = A.n[W];
    float *base = res + coef_off[it];
    if constexpr (ENTROPY) {
      extern __shared__ __align__(16) unsigned char ent_smem[];
      int32_t *s_posts = reinterpret_cast<int32_t *>(ent_smem), *s_present = s_posts + A.ch * VB200_FLOOR1_STRIDE;
      for (int j = threadIdx.x; j < A.ch * n; j += blockDim.x) base[j] = 0.f;
      for (int j = threadIdx.x; j < A.ch * VB200_FLOOR1_STRIDE; j += blockDim.x) s_posts[j] = 0;
      __syncthreads();
      if (threadIdx.x == 0) {
        unsigned char *nz = reinterpret_cast<unsigned char *>(s_present + A.ch);
        ent_block(*E, sF[W], W, P.data + P.off[it], P.bytes[it], base, s_posts, s_present, nz, nz + A.ch,
                  nz + 2 * A.ch);
      }
      __syncthreads();
    }
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      for (int s = A.steps[W] - 1; s >= 0; s--) {
        float *pM = base + (size_t)A.mag[W][s] * n + j, *pA = base + (size_t)A.ang[W][s] * n + j;
        const float m = *pM, a = *pA;
        if (m > 0.f) {
          if (a > 0.f) { *pM = m; *pA = m - a; }
          else         { *pA = m; *pM = m + a; }
        } else {
          if (a > 0.f) { *pM = m; *pA = m + a; }
          else         { *pA = m; *pM = m - a; }
        }
      }
    }
    __syncthreads();
    for (int c = warp; c < A.ch; c += 4) {
      if constexpr (ENTROPY) {
        extern __shared__ __align__(16) unsigned char ent_smem[];
        const int32_t *s_posts = reinterpret_cast<const int32_t *>(ent_smem);
        dev_floor1_inverse2_row(sF[W][A.chmux[W][c]], s_posts + (size_t)c * VB200_FLOOR1_STRIDE,
                                s_posts[A.ch * VB200_FLOOR1_STRIDE + c] != 0, base + (size_t)c * n, n, fromdB,
                                s_segx[warp], s_segy[warp], lane);
      } else {
        const size_t row = (size_t)it * A.ch + c;
        dev_floor1_inverse2_row(sF[W][A.chmux[W][c]], posts + row * VB200_FLOOR1_STRIDE, present[row] != 0,
                                base + (size_t)c * n, n, fromdB, s_segx[warp], s_segy[warp], lane);
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(128)
k_decode_prepare(DecodePrepArgs A, const int *__restrict__ Wseq, const long long *__restrict__ coef_off,
                 float *__restrict__ res, const int32_t *__restrict__ posts, const int32_t *__restrict__ present,
                 const float *__restrict__ fromdB) {
  decode_prepare_body<false>(A, Wseq, coef_off, res, posts, present, fromdB, nullptr);
}

__global__ void __launch_bounds__(128)
k_decode_prepare_counted(DecodePrepArgs A, const int *__restrict__ Wseq, const long long *__restrict__ coef_off,
                         float *__restrict__ res, const int32_t *__restrict__ posts,
                         const int32_t *__restrict__ present, const float *__restrict__ fromdB,
                         const int *__restrict__ count) {
  decode_prepare_body<true>(A, Wseq, coef_off, res, posts, present, fromdB, count);
}

// vb200_decode_packets_resume: the entropy decode of each block's packet in front of the same body
template <bool COUNTED>
__global__ void __launch_bounds__(128)
k_decode_packets(DecodePrepArgs A, EntDev E, DecodePackets P, const int *__restrict__ Wseq,
                 const long long *__restrict__ coef_off, float *__restrict__ res, const float *__restrict__ fromdB,
                 const int *__restrict__ count) {
  decode_prepare_body<COUNTED, true>(A, Wseq, coef_off, res, nullptr, nullptr, fromdB, count, &E, P);
}

// vb200_decode_entropy: the entropy decode alone, into the staging rows of vb200_decode_dsp; one CTA per block
__global__ void __launch_bounds__(32)
k_decode_entropy(EntDev E, const Floor1Dev *__restrict__ floors0, const Floor1Dev *__restrict__ floors1,
                 DecodePackets P, int nblocks, const int *__restrict__ Wseq, const long long *__restrict__ coef_off,
                 float *__restrict__ res, int32_t *__restrict__ posts, int32_t *__restrict__ present) {
  extern __shared__ __align__(16) unsigned char ent_smem[];
  for (int it = blockIdx.x; it < nblocks; it += gridDim.x) {
    const int W = Wseq[it] ? 1 : 0, n = E.n[W], ch = E.ch;
    float *base = res + coef_off[it];
    int32_t *po = posts + (size_t)it * ch * VB200_FLOOR1_STRIDE;
    for (int j = threadIdx.x; j < ch * n; j += blockDim.x) base[j] = 0.f;
    for (int j = threadIdx.x; j < ch * VB200_FLOOR1_STRIDE; j += blockDim.x) po[j] = 0;
    __syncthreads();
    if (threadIdx.x == 0)
      ent_block(E, W ? floors1 : floors0, W, P.data + P.off[it], P.bytes[it], base, po, present + (size_t)it * ch,
                ent_smem, ent_smem + ch, ent_smem + 2 * ch);
    __syncthreads();
  }
}
