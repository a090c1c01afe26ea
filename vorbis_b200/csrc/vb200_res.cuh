// vb200_res.cuh — residue partition classification (SURVEY §8 f3): res1_class / res2_class
// (lib/res0.c:745-778) -> _01class (:412-474) / _2class (:479-532), per submap as mapping0_forward
// calls them (lib/mapping0.c:660-672).  Integer max / sum reductions over `grouping` samples and a
// first-match search over the class metrics: one warp per (block, submap), lane = partition.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

namespace vb200 {

struct ResDev {
  int type, begin, end, grouping, partitions, partvals;
  float scale;                         // 100./grouping as fp32 (lib/res0.c:426)
  int pad;
  int cm1[64], cm2[64];
};

struct ResArgs {
  const ResDev *res;                   // [VB200_MAX_SUBMAPS] of this block size
  const unsigned char *chmux;          // [channels]
  int ch, n, submaps, nblocks, stride;
};

constexpr int RES_WARPS = 4;

// CURVES = false: nblocks blocks, rows blk*ch.  CURVES = true (bitrate-managed): the VB200_PACKETBLOBS curves of
// nblocks blocks; block b of curve k reads iwork / nonzero row k*curve_rows + b*ch (only rows < nblocks of each
// curve) and writes classes row (k*nblocks + b)*ch.
// (the kernels' pointers are __restrict__; restating it here would change the existing kernel's code)
template <bool CURVES>
__device__ __forceinline__ void residue_classify_body(const ResArgs &A, long long curve_rows, const int *iwork,
                                                      const int *nonzero, int *classes) {
  __shared__ unsigned char s_chan[RES_WARPS][256];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned char *chan = s_chan[wid];
  const long tasks = CURVES ? (long)VB200_PACKETBLOBS * A.nblocks * A.submaps : (long)A.nblocks * A.submaps;
  for (long t = (long)blockIdx.x * RES_WARPS + wid; t < tasks; t += (long)gridDim.x * RES_WARPS) {
    const int blk = (int)(t / A.submaps), sm = (int)(t - (long)blk * A.submaps);
    const ResDev &R = A.res[sm];
    if (R.type < 0) continue;
    const int *in = iwork + (size_t)blk * A.ch * A.n;
    const int *nz = nonzero + (size_t)blk * A.ch;
    if constexpr (CURVES) {                                // blk = curve * nblocks + block
      const int curve = blk / A.nblocks;
      const size_t row0 = (size_t)curve * curve_rows + (size_t)(blk - curve * A.nblocks) * A.ch;
      in = iwork + row0 * A.n;
      nz = nonzero + row0;
    }
    // the submap's channels in order, and whether any of them is in use
    __syncwarp();
    int cib = 0, used = 0;
    for (int j0 = 0; j0 < A.ch; j0 += 32) {
      const int j = j0 + lane;
      const bool mine = j < A.ch && A.chmux[j] == sm;
      const unsigned m = __ballot_sync(0xffffffffu, mine);
      if (mine) {
        chan[cib + __popc(m & ((1u << lane) - 1))] = (unsigned char)j;
        if (nz[j]) used = 1;
      }
      cib += __popc(m);
    }
    used = __any_sync(0xffffffffu, used);
    __syncwarp();
    if (!used || cib == 0) continue;                       // res1_class / res2_class return 0
    if (R.type == 2) {                                     // _2class: one vector for the bundle
      int *dst = classes + ((size_t)blk * A.ch + chan[0]) * A.stride;
      const int per = (R.grouping + cib - 1) / cib;        // l advances once per `ch` samples
      for (int i = lane; i < R.partvals; i += 32) {
        int l = R.begin / cib + i * per;
        int magmax = 0, angmax = 0;
        for (int j = 0; j < per; j++, l++) {
          const int a = abs(in[(size_t)chan[0] * A.n + l]);
          if (a > magmax) magmax = a;
          for (int k = 1; k < cib; k++) {
            const int v = abs(in[(size_t)chan[k] * A.n + l]);
            if (v > angmax) angmax = v;
          }
        }
        int j = 0;
        for (; j < R.partitions - 1; j++)
          if (magmax <= R.cm1[j] && angmax <= R.cm2[j]) break;
        dst[i] = j;
      }
    } else {                                               // _01class on every used channel
      for (int u = 0; u < cib; u++) {
        const int c = chan[u];
        if (!nz[c]) continue;
        const int *v = in + (size_t)c * A.n;
        int *dst = classes + ((size_t)blk * A.ch + c) * A.stride;
        for (int i = lane; i < R.partvals; i += 32) {
          const int offset = i * R.grouping + R.begin;
          int mx = 0, ent = 0;
          for (int k = 0; k < R.grouping; k++) {
            const int a = abs(v[offset + k]);
            if (a > mx) mx = a;
            ent += a;
          }
          ent = (int)((float)ent * R.scale);               // ent*=scale
          int k = 0;
          for (; k < R.partitions - 1; k++)
            if (mx <= R.cm1[k] && (R.cm2[k] < 0 || ent < R.cm2[k])) break;
          dst[i] = k;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(32 * RES_WARPS)
k_residue_classify(ResArgs A, const int *__restrict__ iwork, const int *__restrict__ nonzero,
                   int *__restrict__ classes) {
  residue_classify_body<false>(A, 0, iwork, nonzero, classes);
}

__global__ void __launch_bounds__(32 * RES_WARPS)
k_residue_classify_curves(ResArgs A, long long curve_rows, const int *__restrict__ iwork,
                          const int *__restrict__ nonzero, int *__restrict__ classes) {
  residue_classify_body<true>(A, curve_rows, iwork, nonzero, classes);
}

}  // namespace vb200
