/* vb_oracle_halfrate.c — CPU oracle for half-rate decode (vorbis_synthesis_halfrate, lib/synthesis.c:166-174).
 *
 * TEST INFRASTRUCTURE ONLY (see vb_oracle.h).  The restatement of vb_oracle.c is compiled into this unit
 * unchanged (#include below) and reused stage by stage; what half-rate decode changes is restated here:
 *   - _vds_shared_init builds the inverse MDCTs at blocksizes[W]>>1 (lib/block.c:182,197-198), so
 *     mapping0_inverse's mdct_backward (lib/mapping0.c:792-795) reads the first blocksizes[W]/4 lines of
 *     each channel's residue vector (still blocksizes[W]/2 long) and writes blocksizes[W]/2 samples;
 *   - vorbis_synthesis_blockin overlaps with the windows of the halved sizes, n0 = blocksizes[0]>>2,
 *     n1 = blocksizes[1]>>2 (lib/block.c:755-823), so block k finishes (bs[lW]/4 + bs[W]/4) >> 1 samples;
 *   - de-coupling and the floor multiply still cover all n lines (lib/mapping0.c:754-790).
 * The overlap-add of vb_oracle_b.inc is written against a context's two transforms, so a second context
 * whose transforms are those of the halved sizes gives exactly the half-rate overlap-add.
 * Built by oracle/Makefile with the flags of its libvb_oracle.so.
 */
#include "vb_oracle.c"

typedef struct vbohs {
  vbo_ctx *full;                  /* the full-rate lookups: de-coupling, floor multiply, spectra layout */
  vbo_ctx  half;                  /* x[w] = mdct_init(blocksizes[w]/2) and the half window of that size */
} vbohs;

/* NULL where vorbis_synthesis_halfrate returns -1 (blocksizes[0] <= 64).  window[w]: blocksizes[w]/4 floats,
 * what _vorbis_window_get(b->window[w]-1) returns; window or window[w] NULL = closed form (doc/04-codec.tex:320) */
vbohs *vbohs_create(const vb200_setup *setup, const float *const window[2]){
  vbohs *h;
  int w;
  if(setup->blocksizes[0] <= 64) return NULL;
  h = (vbohs*)calloc(1, sizeof(*h));
  h->full = vbo_create(setup);
  h->half.setup = *setup;
  for(w = 0; w < 2; w++){
    xform_init_mdct(&h->half.x[w], setup->blocksizes[w] / 2);
    xform_init_window(&h->half.x[w], window ? window[w] : NULL);
  }
  return h;
}

void vbohs_destroy(vbohs *h){
  int w;
  if(!h) return;
  for(w = 0; w < 2; w++){ free(h->half.x[w].trig); free(h->half.x[w].bitrev); free(h->half.x[w].win); }
  vbo_destroy(h->full);
  free(h);
}

/* mdct_backward at N = blocksizes[W]/2: in [nvec][N/2] -> out [nvec][N] */
void vbohs_mdct_backward(vbohs *h, int W, int nvec, const float *in, float *out){
  const vbo_xform *X = &h->half.x[W];
  int N = X->N, v;
  for(v = 0; v < nvec; v++) mdct_backward1(X, in + (size_t)v*(N/2), out + (size_t)v*N);
}

/* vbo_synthesis in half-rate mode: same spectra layout (channel cc of a block at coef_off + cc*blocksizes[W]/2),
 * pcm_off / pcm_stride in half-rate samples */
void vbohs_synthesis(vbohs *h, int nstreams, int nblk, const int32_t *Wseq,
                     const int64_t *coef_off, const float *coef,
                     const int64_t *pcm_off, float *pcm, int64_t pcm_stride){
  const vbo_ctx *hc = &h->half;
  int ch = hc->setup.channels, Nmax = hc->x[1].N, st, k, cc;
  float *cur = (float*)malloc(sizeof(float)*Nmax);
  float *prev = (float*)malloc(sizeof(float)*Nmax);
  for(st = 0; st < nstreams; st++){
    for(cc = 0; cc < ch; cc++){
      float *dst = pcm + ((size_t)st*ch + cc)*pcm_stride;
      for(k = 0; k < nblk; k++){
        int W = Wseq[(size_t)st*nblk + k];
        int N = hc->x[W].N;                       /* blocksizes[W]/2; a channel's residue vector is N long */
        const float *src = coef + coef_off[(size_t)st*nblk + k] + (size_t)cc*N;
        mdct_backward1(&hc->x[W], src, cur);
        if(k > 0){
          int lW = Wseq[(size_t)st*nblk + k - 1];
          overlap_pair(hc, lW, W, prev, cur, dst + pcm_off[(size_t)st*nblk + k]);
        }
        memcpy(prev, cur + N/2, sizeof(float)*(N/2));
      }
    }
  }
  free(cur); free(prev);
}

/* vbo_decode_dsp in half-rate mode: de-coupling and floor multiply at full size, in place on res */
void vbohs_decode_dsp(vbohs *h, int nstreams, int nblk, const int32_t *Wseq, const int64_t *coef_off,
                      float *res, const int32_t *posts, const int32_t *present,
                      const int64_t *pcm_off, float *pcm, int64_t pcm_stride){
  int ch = h->full->setup.channels;
  long i;
  for(i = 0; i < (long)nstreams*nblk; i++){
    int W = Wseq[i] ? 1 : 0;
    vbo_decouple(h->full, W, 1, res + coef_off[i]);
    vbo_floor1_inverse2(h->full, W, -1, ch, posts + (size_t)i*ch*VB200_FLOOR1_STRIDE, present + (size_t)i*ch,
                        res + coef_off[i]);
  }
  vbohs_synthesis(h, nstreams, nblk, Wseq, coef_off, res, pcm_off, pcm, pcm_stride);
}
