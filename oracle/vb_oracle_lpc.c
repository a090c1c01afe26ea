/* vb_oracle_lpc.c — the LPC extrapolation of vorbis_analysis_wrote restated in plain C.  TEST INFRASTRUCTURE ONLY
 * (oracle/lpc.py builds and binds it; it is the CPU counterpart of vorbis_b200/csrc/vb200_lpc.cuh).
 *
 *   vbo_lpc_filter   the coefficients of an order-m linear predictor fitted to x[0 .. n): the lag-k autocorrelations
 *                    as sequential double sums over ascending i, the Levinson-Durbin recursion in double with a
 *                    -100 dB floor (stop once the residual energy falls below 1e-9 of the signal's plus 1e-10), each
 *                    coefficient k damped by 0.99^(k+1), then rounded to float
 *   vbo_lpc_run      count predicted samples continuing a window whose last m samples are prime: each output is
 *                    0 minus the m products of the latest m samples with the coefficients in reverse, subtracted
 *                    one by one in float, and becomes the newest sample
 * Compiled with the parity flags of oracle/Makefile (no contraction), as the device kernels run with -fmad=false. */
#include <stdlib.h>
#include <string.h>

void vbo_lpc_filter(const float *x, long n, int m, float *coef){
  double r[33], a[32];
  double e, floor_e;
  int k, i, j;
  for(k = 0; k <= m; k++){
    double acc = 0.;
    long t;
    for(t = k; t < n; t++) acc += (double)x[t] * (double)x[t - k];
    r[k] = acc;
  }
  e = r[0] * (1. + 1e-10);
  floor_e = 1e-9 * r[0] + 1e-10;
  for(i = 0; i < m; i++) a[i] = 0.;
  for(i = 0; i < m; i++){
    double g;
    if(e < floor_e) break;
    g = -r[i + 1];
    for(j = 0; j < i; j++) g -= a[j] * r[i - j];
    g /= e;
    a[i] = g;
    for(j = 0; j < i / 2; j++){
      const double lo = a[j], hi = a[i - 1 - j];
      a[j] = lo + g * hi;
      a[i - 1 - j] = hi + g * lo;
    }
    if(i & 1) a[j] = a[j] + a[j] * g;
    e *= 1. - g * g;
  }
  {
    double w = .99;
    for(i = 0; i < m; i++){ a[i] *= w; w *= .99; }
  }
  for(i = 0; i < m; i++) coef[i] = (float)a[i];
}

void vbo_lpc_run(const float *coef, const float *prime, int m, float *out, long count){
  float hist[32];
  long k;
  int j;
  memcpy(hist, prime, sizeof(float) * m);
  for(k = 0; k < count; k++){
    float y = 0.f;
    for(j = 0; j < m; j++) y -= hist[j] * coef[m - 1 - j];
    memmove(hist, hist + 1, sizeof(float) * (m - 1));
    hist[m - 1] = y;
    out[k] = y;
  }
}
