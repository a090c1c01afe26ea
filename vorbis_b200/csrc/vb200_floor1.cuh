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
// k_floor1_fit's register bound: 4 CTAs (32 warps) per SM.  The fit is bound by instruction issue rather than by
// latency: on an H100 forcing 5 or 6 CTAs per SM (48 or 40 registers, a few spills) made it 1-2 % slower, not faster
#define F1_FIT_CTAS 4
#define F1_ACC 12                      // xa ya x2a y2a xya an | xb yb x2b y2b xyb bn

struct F1Post {                        // the split loop's state of one post (fitA, fitB, loneighbor, hineighbor, memo)
  int A, B, out;
  signed char lon, hin, memo, pad;     // post indices (< VB200_VIF_POSIT + 2) or -1
};
static_assert(sizeof(F1Post) % 8 == 0 && VB200_VIF_POSIT + 2 <= 127,
              "every warp's area in k_floor1_fit starts 8-byte aligned (its fp64 terms come first)");

// a warp's shared memory in k_floor1_fit, for floors of at most `posts` posts and rows of n lines: the fit terms
// (12 ints or 6 doubles per gap), the per-post state, the quantised row
__host__ __device__ inline size_t floor1_fit_smem_per_warp(int n, int posts) {
  return sizeof(int) * F1_ACC * (size_t)(posts - 1) + sizeof(F1Post) * (size_t)posts +
         ((sizeof(unsigned short) * (size_t)n + 7) & ~(size_t)7);
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

__device__ __forceinline__ int f1_postY(const F1Post *st, int pos) {
  const int a = st[pos].A, b = st[pos].B;
  if (a < 0) return b;
  if (b < 0) return a;
  return (a + b) >> 1;
}

// inspect_error's closing tests (lib/floor1.c:558-563) without a division per call.  fl(fl(maxover*maxover)/cnt) >
// maxerr cannot turn from false to true as cnt grows (correctly rounded division is monotone), nor can the maxunder
// test, so "either holds" is exactly cnt < skip for the smallest failing cnt, found by bisection.  (float)k > maxerr is
// monotone in the integer k, so with kerr the smallest k for which it holds, (float)(mse / cnt) > maxerr is exactly
// mse / cnt >= kerr, i.e. mse >= kerr * cnt (mse >= 0, cnt >= 1).  Computed once per floor per CTA.
struct F1Tests { int skip, kerr; };
__device__ inline F1Tests f1_inspect_tests(const Floor1Dev &F) {
  const auto either = [&](int cnt) {
    return F.maxover * F.maxover / (float)cnt > F.maxerr || F.maxunder * F.maxunder / (float)cnt > F.maxerr;
  };
  F1Tests t;
  if (!either(1)) {
    t.skip = 1;
  } else {                                             // either(lo) holds; cnt never reaches hi = 2^20
    int lo = 1, hi = 1 << 20;
    while (hi - lo > 1) { const int mid = lo + (hi - lo) / 2; if (either(mid)) lo = mid; else hi = mid; }
    t.skip = hi;
  }
  if ((float)0 > F.maxerr) {
    t.kerr = 0;
  } else {                                             // (float)lo > maxerr fails; hi = INT_MAX stands for "never"
    int lo = 0, hi = 0x7fffffff;
    while (hi - lo > 1) { const int mid = lo + (hi - lo) / 2; if ((float)mid > F.maxerr) hi = mid; else lo = mid; }
    t.kerr = hi;
  }
  return t;
}

// inspect_error's scan over one lane's abscissae x, x + 32, ... < x1, y = the line at x.  ITH: maxover / maxunder are
// whole numbers (F.int_thresh), so the integer compares are exact; the thresholds are hoisted out of the loop and the
// body is branch-free
template <bool ITH>
__device__ __forceinline__ void f1_scan(const Floor1Dev &F, const unsigned short *q, int x, int x0, int x1, int y,
                                        int r, int m32, int ystep, int adx, int step, int &mse, int &viol) {
  const int mo_i = F.maxover_i, mu_i = F.maxunder_i;
  const float mo = F.maxover, mu = F.maxunder;
  for (; x < x1; x += 32) {
    const int v = q[x];
    const int val = v & 0x7fff;
    mse += (y - val) * (y - val);
    bool over;
    if (ITH) over = (y + mo_i < val) | (y - mu_i > val);
    else     over = ((float)y + mo < (float)val) | ((float)y - mu > (float)val);
    viol |= (int)(over & ((v & 0x8000) != 0) & ((x == x0) | (val != 0)));
    r += m32;
    y += ystep;
    if (r >= adx) { r -= adx; y += step; }
  }
}

// inspect_error: 1 = this line is not good enough.  q[x] = dBquant(mask[x]) | (audible << 15)
__device__ __forceinline__ int f1_inspect(const Floor1Dev &F, F1Tests T, const unsigned short *q, int x0, int x1,
                                          int y0, int y1, int lane) {
  int mse = 0, viol = 0;
  int x = x0 + lane;
  if (x < x1) {
    // F1Line's integer line in closed form at this lane's first x, then 32 abscissae per step: the error term
    // advances by (32*ady) mod adx and wraps at most once more than floor(32*ady / adx) times.  Every quotient
    // here is floor(num / adx) with 0 <= num < 2^24 (exact in fp32) and num / adx < 2^12 (|dy| < 1224, k < n <= 4096,
    // ady < adx): from an approximate reciprocal (relative error < 2^-21) the estimate is off by at most one, and
    // the remainder test makes it exact
    const int adx = x1 - x0, dy = y1 - y0, step = dy < 0 ? -1 : 1;
    const float rcp = __fdividef(1.f, (float)adx);
    const auto qr = [&](int num, int &rem) {
      int qq = __float2int_rz((float)num * rcp), t = num - qq * adx;
      if (t < 0) { qq--; t += adx; } else if (t >= adx) { qq++; t -= adx; }
      rem = t;
      return qq;
    };
    int ady, r, m32;
    const int b = qr(abs(dy), ady);                    // |dy / adx|; ady = |dy| - |base| * adx
    const int base = dy < 0 ? -b : b;
    const int k = x - x0;
    const int y = y0 + k * base + qr(k * ady, r) * step;
    const int ystep = 32 * base + qr(32 * ady, m32) * step;
    if (F.int_thresh) f1_scan<true>(F, q, x, x0, x1, y, r, m32, ystep, adx, step, mse, viol);
    else              f1_scan<false>(F, q, x, x0, x1, y, r, m32, ystep, adx, step, mse, viol);
  }
  if (__any_sync(0xffffffffu, viol)) return 1;
  mse = __reduce_add_sync(0xffffffffu, mse);
  const int cnt = x1 - x0;
  if (cnt < T.skip) return 0;
  return (long long)mse >= (long long)T.kerr * cnt;
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

// DBG = true: the instance with per-phase clock marks and per-row counters (tools/floor1_phase_timing.py).  Every
// warp sums its own marks and lane 0 adds them into dbg[F1_DBG_SLOTS] once, at the end: the production instance
// (DBG = false) carries none of it.
enum { F1_T_Q, F1_T_ACC, F1_T_TERMS, F1_T_FIT0, F1_T_INSPECT, F1_T_FIT, F1_T_SPLIT, F1_T_OUT,
       F1_C_INSPECT, F1_C_FIT, F1_C_NULL, F1_C_ROWS, F1_DBG_SLOTS };

template <bool DBG>
__global__ void __launch_bounds__(32 * F1_WARPS, DBG ? 1 : F1_FIT_CTAS)
k_floor1_fit(Floor1Args a, int pcap, const float *__restrict__ logmdct, const float *__restrict__ logmask,
             int32_t *__restrict__ posts_out, int32_t *__restrict__ fit_nonzero, unsigned long long *dbg) {
  unsigned dsum[F1_DBG_SLOTS] = {};          // per-warp sums: a warp's rows take far fewer than 2^32 cycles
  long long tmark = 0;
#define F1_MARK(slot)                                                            \
  do {                                                                           \
    if (DBG) { const long long t_ = clock64(); dsum[slot] += (unsigned)(t_ - tmark); tmark = t_; } \
  } while (0)
#define F1_COUNT(slot) do { if (DBG) dsum[slot]++; } while (0)
  extern __shared__ __align__(16) unsigned char f1_smem[];
  Floor1Dev *sF = reinterpret_cast<Floor1Dev *>(f1_smem);
  {
    const int words = (int)(sizeof(Floor1Dev) * VB200_MAX_SUBMAPS / 4);
    const int *src = reinterpret_cast<const int *>(a.floors);
    int *dst = reinterpret_cast<int *>(sF);
    for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
  }
  __shared__ F1Tests sT[VB200_MAX_SUBMAPS];
  if (threadIdx.x < VB200_MAX_SUBMAPS) sT[threadIdx.x] = f1_inspect_tests(a.floors[threadIdx.x]);
  __syncthreads();
  if (DBG) tmark = clock64();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char *wbase = f1_smem + sizeof(Floor1Dev) * VB200_MAX_SUBMAPS + floor1_fit_smem_per_warp(a.n, pcap) * warp;
  double *term = reinterpret_cast<double *>(wbase);          // [gaps][6], same bytes as 12 ints per gap
  F1Post *st = reinterpret_cast<F1Post *>(wbase + sizeof(int) * F1_ACC * (pcap - 1));
  unsigned short *q = reinterpret_cast<unsigned short *>(st + pcap);

  for (int row = blockIdx.x * F1_WARPS + warp; row < a.nrows; row += gridDim.x * F1_WARPS) {   // grid_for: no overflow
    const int sel = a.floor_sel >= 0 ? a.floor_sel : a.chmux[row % a.channels];
    const Floor1Dev &F = sF[sel];
    const int P = F.posts, n = F.n;
    const float *md = logmdct + (size_t)row * a.n, *mk = logmask + (size_t)row * a.n;
    int32_t *po = posts_out + (size_t)row * VB200_FLOOR1_STRIDE;
    __syncwarp();
    F1_COUNT(F1_C_ROWS);
    const float att = F.twofitatten;
    const auto qv = [att](float d, float m) { return (unsigned)f1_dBquant(m) | ((d + att >= m) ? 0x8000u : 0u); };
    if ((n & 3) == 0 && (((uintptr_t)md | (uintptr_t)mk) & 15) == 0) {   // four lines per load and store
      for (int x = 4 * lane; x < n; x += 128) {
        const float4 d = *reinterpret_cast<const float4 *>(md + x), m = *reinterpret_cast<const float4 *>(mk + x);
        *reinterpret_cast<uint2 *>(q + x) = make_uint2(qv(d.x, m.x) | qv(d.y, m.y) << 16, qv(d.z, m.z) | qv(d.w, m.w) << 16);
      }
    } else {
      for (int x = lane; x < n; x += 32) q[x] = (unsigned short)qv(md[x], mk[x]);
    }
    for (int i = lane; i < P; i += 32) { st[i].A = -200; st[i].B = -200; st[i].lon = 0; st[i].hin = 1; st[i].memo = -1; }
    __syncwarp();
    F1_MARK(F1_T_Q);
    // accumulate_fit: one accumulator per gap, both ends inclusive
    int nonzero = 0;
    for (int j = 0; j < P - 1; j++) {
      const int x0 = F.sorted[j];
      int x1 = F.sorted[j + 1];
      if (x1 >= n) x1 = n - 1;
      int s[F1_ACC];
#pragma unroll
      for (int k = 0; k < F1_ACC; k++) s[k] = 0;
      // a warp-uniform trip count (every gap holds at least one line): no zero-trip path to set up twice
      const int iters = (x1 - x0 + 32) >> 5;
      int x = x0 + lane, it = 0;
      do {
        const int v = x <= x1 ? q[x] : 0, val = v & 0x7fff;
        const bool ua = val != 0 && (v & 0x8000), ub = val != 0 && !(v & 0x8000);   // predicated, no branch
        if (ua) { s[0] += x; s[1] += val; s[2] += x * x; s[3] += val * val; s[4] += x * val; s[5]++; }
        if (ub) { s[6] += x; s[7] += val; s[8] += x * x; s[9] += val * val; s[10] += x * val; s[11]++; }
        x += 32;
      } while (++it < iters);
#pragma unroll
      for (int k = 0; k < F1_ACC; k++) s[k] = __reduce_add_sync(0xffffffffu, s[k]);
      if (lane == 0) {                                   // raw sums; turned into fit_line's terms below
        int2 *dst = reinterpret_cast<int2 *>(term + j * (F1_ACC / 2));
#pragma unroll
        for (int k = 0; k < F1_ACC / 2; k++) dst[k] = make_int2(s[2 * k], s[2 * k + 1]);
      }
      nonzero += s[5];
    }
    __syncwarp();
    F1_MARK(F1_T_ACC);
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
    F1_MARK(F1_T_TERMS);
    if (!nonzero) {                                      // the reference returns NULL
      for (int i = lane; i < VB200_FLOOR1_STRIDE; i += 32) po[i] = 0;
      if (lane == 0) fit_nonzero[row] = 0;
      F1_COUNT(F1_C_NULL);
      F1_MARK(F1_T_OUT);
      continue;
    }
    int y[4];
    f1_fit_lines(F, term, 0, P - 1, 0, 0, lane, y);
    if (lane == 0) { st[0].A = y[0]; st[0].B = y[0]; st[1].A = y[1]; st[1].B = y[1]; }
    __syncwarp();
    F1_MARK(F1_T_FIT0);
    for (int i = 2; i < P; i++) {
      const int sortpos = F.rev[i];
      const int ln = st[sortpos].lon, hn = st[sortpos].hin;
      if (st[ln].memo == hn) continue;                      // this span was already judged
      const int lsortpos = F.rev[ln], hsortpos = F.rev[hn];
      const int lx = F.postlist[ln], hx = F.postlist[hn];
      const int ly = f1_postY(st, ln), hy = f1_postY(st, hn);
      __syncwarp();
      if (lane == 0) st[ln].memo = (signed char)hn;
      F1_MARK(F1_T_SPLIT);
      const int bad = f1_inspect(F, sT[sel], q, lx, hx, ly, hy, lane);
      F1_COUNT(F1_C_INSPECT);
      F1_MARK(F1_T_INSPECT);
      if (bad) {
        const int ret = f1_fit_lines(F, term, lsortpos, sortpos - lsortpos, sortpos, hsortpos - sortpos, lane, y);
        F1_COUNT(F1_C_FIT);
        F1_MARK(F1_T_FIT);
        int ly0 = y[0], ly1 = y[1], hy0 = y[2], hy1 = y[3];
        if (ret & 1) { ly0 = ly; ly1 = hy0; }
        if (ret & 2) { hy0 = ly1; hy1 = hy; }
        if (lane == 0) {
          if (ret == 3) {
            st[i].A = -200; st[i].B = -200;
          } else {
            st[ln].B = ly0;
            if (ln == 0) st[ln].A = ly0;
            st[i].A = ly1; st[i].B = hy0;
            st[hn].A = hy1;
            if (hn == 1) st[hn].B = hy1;
            if (ly1 >= 0 || hy0 >= 0) {
              for (int j = sortpos - 1; j >= 0; j--) { if (st[j].hin == hn) st[j].hin = (signed char)i; else break; }
              for (int j = sortpos + 1; j < P; j++) { if (st[j].lon == ln) st[j].lon = (signed char)i; else break; }
            }
          }
        }
      } else if (lane == 0) {
        st[i].A = -200; st[i].B = -200;
      }
      __syncwarp();
    }
    F1_MARK(F1_T_SPLIT);
    // posts as the reference returns them: fitted value, or predicted | 0x8000 when unused
    if (lane == 0) {
      st[0].out = f1_postY(st, 0);
      st[1].out = f1_postY(st, 1);
      fit_nonzero[row] = 1;
    }
    __syncwarp();
    for (int lv = 0; lv < F.nlevels; lv++) {             // out[i] depends on out[lo], out[hi] only: level by level
      for (int t = F.lvl_start[lv] + lane; t < F.lvl_start[lv + 1]; t += 32) {
        const int i = F.lvl_order[t];
        const int ln = F.lo[i - 2], hn = F.hi[i - 2];
        const int predicted = f1_point(F.postlist[ln], F.postlist[hn], st[ln].out, st[hn].out, F.postlist[i],
                                       F.prcp[i - 2]);
        const int vx = f1_postY(st, i);
        st[i].out = (vx >= 0 && predicted != vx) ? vx : (predicted | 0x8000);
      }
      __syncwarp();
    }
    for (int i = lane; i < VB200_FLOOR1_STRIDE; i += 32) po[i] = i < P ? st[i].out : 0;
    F1_MARK(F1_T_OUT);
  }
  if (DBG && lane == 0)
    for (int k = 0; k < F1_DBG_SLOTS; k++) atomicAdd(dbg + k, (unsigned long long)dsum[k]);
#undef F1_MARK
#undef F1_COUNT
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

// undo channel coupling, lib/mapping0.c:754-779 (square polar -> L/R), in place: one step's pair of bins
__device__ __forceinline__ void dev_decouple(float *pM, float *pA) {
  const float m = *pM, a = *pA;
  if (m > 0.f) {
    if (a > 0.f) { *pM = m; *pA = m - a; }
    else         { *pA = m; *pM = m + a; }
  } else {
    if (a > 0.f) { *pM = m; *pA = m + a; }
    else         { *pA = m; *pM = m - a; }
  }
}

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
    for (int j = threadIdx.x; j < n; j += blockDim.x)
      for (int s = A.steps[W] - 1; s >= 0; s--)
        dev_decouple(base + (size_t)A.mag[W][s] * n + j, base + (size_t)A.ang[W][s] * n + j);
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

template <bool COUNTED>
__global__ void __launch_bounds__(128)
k_decode_prepare(DecodePrepArgs A, const int *__restrict__ Wseq, const long long *__restrict__ coef_off,
                 float *__restrict__ res, const int32_t *__restrict__ posts, const int32_t *__restrict__ present,
                 const float *__restrict__ fromdB, const int *__restrict__ count) {
  decode_prepare_body<COUNTED>(A, Wseq, coef_off, res, posts, present, fromdB, count);
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
