// vb200_managed.cuh — the extra steps of bitrate-managed mode (SURVEY §8 a12; lib/mapping0.c:507-573):
//
//  k_mix_select          _vp_offset_and_mix (lib/psy.c:779-835) with offset_select 0 or 2 on a batch whose blocks
//                        carry their own psy look (blocktype): only the mask changes, the MDCT adjustment belongs
//                        to select 1 (done inside the psy kernel)
//  k_floor1_interpolate  floor1_interpolate_fit (lib/floor1.c:731-757) for the twelve intermediate curves, plus
//                        the NULL rules of mapping0_forward: the low / high fits exist only where the middle fit
//                        does (:506), an interpolated curve only where both of its ends do (:736)
//
// Posts are blob-major: posts[k][row][VB200_FLOOR1_STRIDE]; a missing curve is an all-zero row with present = 0,
// as everywhere else in this library.
#pragma once
#include "vb200_kernels.cuh"

namespace vb200 {

__global__ void __launch_bounds__(256)
k_mix_select(PsyDev P0, PsyDev P1, const vb200_block_desc *__restrict__ desc, int ch, long long total, int sel,
             const float *__restrict__ noise, const float *__restrict__ tone, const float *__restrict__ logmdct,
             float *__restrict__ logmask) {
  const int n = P0.n;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = e / n;
    const int i = (int)(e - row * n);
    const PsyDev &P = desc[row / ch].blocktype ? P1 : P0;
    float m = 0.f;                                       // select != 1 leaves the MDCT alone
    logmask[e] = dev_mix_bin(P, sel, noise[e], tone[e], __ldg(P.noiseoffset + (size_t)sel * n + i), logmdct[e], m);
  }
}

// one thread per (row, post slot); present[k][row] for all VB200_PACKETBLOBS curves.  Curve k of posts and
// present starts k * blob_rows rows in (blob_rows >= rows).
__global__ void __launch_bounds__(256)
k_floor1_interpolate(long long rows, long long blob_rows, int32_t *__restrict__ posts, const int32_t *__restrict__ fz_lo,
                     const int32_t *__restrict__ fz_mid, const int32_t *__restrict__ fz_hi,
                     int32_t *__restrict__ present) {
  constexpr int NB = VB200_PACKETBLOBS, MID = VB200_PACKETBLOBS / 2, S = VB200_FLOOR1_STRIDE;
  const long long total = rows * S;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = e / S;
    const int i = (int)(e - row * S);
    const int mid = fz_mid[row] != 0, lo = mid && fz_lo[row] != 0, hi = mid && fz_hi[row] != 0;
    const size_t blob = (size_t)blob_rows * S;
    int32_t *p = posts + (size_t)row * S + i;
    const int a = lo ? p[0] : 0, b = mid ? p[(size_t)MID * blob] : 0, c = hi ? p[(size_t)(NB - 1) * blob] : 0;
    p[0] = a; p[(size_t)(NB - 1) * blob] = c;
    for (int k = 1; k < MID; k++) {
      const int del = k * 65536 / MID;
      int v = 0;
      if (lo) {                                          // (mid holds whenever lo does)
        v = ((65536 - del) * (a & 0x7fff) + del * (b & 0x7fff) + 32768) >> 16;
        if ((a & 0x8000) && (b & 0x8000)) v |= 0x8000;
      }
      p[(size_t)k * blob] = v;
    }
    for (int k = MID + 1; k < NB - 1; k++) {
      const int del = (k - MID) * 65536 / MID;
      int v = 0;
      if (hi) {
        v = ((65536 - del) * (b & 0x7fff) + del * (c & 0x7fff) + 32768) >> 16;
        if ((b & 0x8000) && (c & 0x8000)) v |= 0x8000;
      }
      p[(size_t)k * blob] = v;
    }
    if (i == 0) {
      for (int k = 0; k < NB; k++)
        present[(size_t)k * blob_rows + row] = k < MID ? lo : (k == MID ? mid : hi);
    }
  }
}

}  // namespace vb200
