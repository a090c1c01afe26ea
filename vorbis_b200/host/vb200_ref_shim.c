/* vb200_ref_shim.c — the reference-side binding: libvorbis' own hot-path functions,
 * with libvorbis' own signatures, implemented by calls into the CUDA library.
 *
 * A libvorbis maintainer drops this file into lib/ and compiles lib/mapping0.c with
 *   -Dmdct_forward=vb200shim_mdct_forward -Dmdct_backward=vb200shim_mdct_backward
 *   -D_vorbis_apply_window=vb200shim_apply_window -Ddrft_forward=vb200shim_drft_forward
 *   -D_vp_noisemask=vb200shim_noisemask -D_vp_tonemask=vb200shim_tonemask
 *   -D_vp_offset_and_mix=vb200shim_offset_and_mix
 *   -D_vp_couple_quantize_normalize=vb200shim_couple_quantize_normalize
 *   -Dfloor1_fit=vb200shim_floor1_fit
 * and lib/block.c with
 *   -D_ve_envelope_search=vb200shim_envelope_search
 * (or renames the callees in place); nothing else in libvorbis changes.  Every function
 * below has exactly the prototype of the reference function it replaces (cited), and
 * the same argument meaning, in-place behaviour and (absence of) error returns; a CUDA
 * failure is reported on stderr and the block is left untouched rather than aborting.
 *
 * This is the per-function (stage-level) binding: one host<->device round trip per
 * call, so it demonstrates bit-exact drop-in behaviour, not speed.  The batched
 * entry points of include/vorbis_b200.h (vb200_analysis_phaseA etc.) are the fast path;
 * INTEGRATION.md shows how mapping0_forward hands whole batches to them.
 *
 * Compiled against the reference's internal headers (codec_internal.h, psy.h, mdct.h,
 * smallft.h) - like any libvorbis-internal backend - by oracle/Makefile target `dropin`.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "codec_internal.h"
#include "mdct.h"
#include "smallft.h"
#include "window.h"
#include "psy.h"
#include "envelope.h"

#include "vorbis_b200.h"
#include "vb200_vorbis_setup.h"

int vb200shim_attach_new(vorbis_dsp_state *vd, int device);
/* Bindings: one device context per codec setup (vorbis_info.codec_setup), shared by every vorbis_dsp_state
 * initialised from it - the device tables are read-only, so all streams of one configuration use the same
 * context (SURVEY §8b "ownership").  vb200shim_attach() finds or creates the binding of a state and makes it
 * the calling thread's current one; the stage-level shims below have the reference's own prototypes, which
 * carry no state pointer, so they act on that current binding (the reference is single threaded per
 * vorbis_dsp_state; concurrent states on different threads each attach in their own thread).  The block-level
 * seam (vb200_mapping0.c) never uses the current binding: it looks the binding up from vb->vd.
 * A CUDA failure latches binding->error (sticky) - vb200shim_error() - and vorbis_analysis reports
 * OV_EFAULT through the block-level seam; the stage shims leave the data untouched as before.          */
#define VB200_MAX_BINDINGS 64
typedef struct vb200_binding {
  vb200_ctx *ctx;
  void *setup_key;                       /* vd->vi->codec_setup */
  vorbis_dsp_state *vd;                  /* a state of this setup (for the lookups) */
  int analysisp, refs, error;
  int32_t *octave[4], *bark[4];
  float *tonecurves[4], *noiseoffset[4];
  float *fscratch; size_t fscratch_cap;  /* grow-only host scratch of the stage shims (no malloc per call) */
  int32_t *iscratch; size_t iscratch_cap;
} vb200_binding;
static vb200_binding g_bind[VB200_MAX_BINDINGS];
static __thread vb200_binding *g_cur;
#define g (*g_cur)

static void shim_warn(const char *what, int rc){
  if(g_cur && !g_cur->error) g_cur->error = rc;
  fprintf(stderr, "vb200 shim: %s failed (%d): %s\n", what, rc, vb200_last_error());
}
int vb200shim_error(void){ return g_cur ? g_cur->error : 0; }

vb200_binding *vb200shim_binding(vorbis_dsp_state *vd){
  int i;
  for(i = 0; i < VB200_MAX_BINDINGS; i++)
    if(g_bind[i].ctx && g_bind[i].setup_key == (void*)vd->vi->codec_setup && g_bind[i].analysisp == vd->analysisp) return &g_bind[i];
  return NULL;
}
vb200_ctx *vb200shim_ctx(vb200_binding *b){ return b ? b->ctx : NULL; }
void vb200shim_set_error(vb200_binding *b, int rc){ if(b && !b->error) b->error = rc; }
static float *bind_fscratch(size_t n){
  if(g.fscratch_cap < n){ free(g.fscratch); g.fscratch = (float*)malloc(sizeof(float)*n); g.fscratch_cap = g.fscratch ? n : 0; }
  return g.fscratch;
}
static int32_t *bind_iscratch(size_t n){
  if(g.iscratch_cap < n){ free(g.iscratch); g.iscratch = (int32_t*)malloc(sizeof(int32_t)*n); g.iscratch_cap = g.iscratch ? n : 0; }
  return g.iscratch;
}

/* vorbis_synthesis_halfrate (lib/synthesis.c:166-174) as _vds_shared_init saw it when it built vd's lookups
 * (lib/block.c:182,197-198): the decode shims then run at the halved sizes with the windows of those sizes */
static int bind_halfrate(vorbis_dsp_state *vd){
  codec_setup_info *ci = (codec_setup_info*)vd->vi->codec_setup;
  private_state *b = (private_state*)vd->backend_state;
  const float *win[2];
  int rc;
  if(!ci->halfrate_flag) return vb200_synthesis_halfrate(g.ctx, 0, NULL);
  win[0] = _vorbis_window_get(b->window[0] - 1);
  win[1] = _vorbis_window_get(b->window[1] - 1);
  rc = vb200_synthesis_halfrate(g.ctx, 1, win);
  if(rc) fprintf(stderr, "vb200 shim: vb200_synthesis_halfrate failed (%d): %s\n", rc, vb200_last_error());
  return rc;
}

/* Build the device context from the lookups _vds_shared_init made (lib/block.c:170-294). */
int vb200shim_attach(vorbis_dsp_state *vd, int device){
  vorbis_info *vi = vd->vi;
  vb200_binding *found = vb200shim_binding(vd);
  if(found){ found->refs++; g_cur = found; return bind_halfrate(vd); }   /* another state of the same setup: share the context */
  {
    int slot;
    for(slot = 0; slot < VB200_MAX_BINDINGS && g_bind[slot].ctx; slot++);
    if(slot == VB200_MAX_BINDINGS){ fprintf(stderr, "vb200 shim: too many codec setups attached\n"); return VB200_EINVAL; }
    memset(&g_bind[slot], 0, sizeof(g_bind[slot]));
    g_cur = &g_bind[slot];
  }
  return vb200shim_attach_new(vd, device);
}
static void bind_release(vb200_binding *b){
  int i;
  if(b->ctx) vb200_ctx_destroy(b->ctx);
  for(i = 0; i < 4; i++){ free(b->octave[i]); free(b->bark[i]); free(b->tonecurves[i]); free(b->noiseoffset[i]); }
  free(b->fscratch); free(b->iscratch);
  memset(b, 0, sizeof(*b));
}
int vb200shim_attach_new(vorbis_dsp_state *vd, int device){
  vorbis_info *vi = vd->vi;
  codec_setup_info *ci = (codec_setup_info*)vi->codec_setup;
  private_state *b = (private_state*)vd->backend_state;
  vorbis_info_psy_global *gi = &ci->psy_g_param;
  vb200_setup s;
  int i, j, k, w, rc;
  memset(&s, 0, sizeof(s));
  s.channels = vi->channels;
  s.rate = (int32_t)vi->rate;
  s.blocksizes[0] = (int32_t)ci->blocksizes[0];
  s.blocksizes[1] = (int32_t)ci->blocksizes[1];
  s.n_psy = (vd->analysisp && ci->psys == 4) ? 4 : 0;
  for(i = 0; i < s.n_psy; i++){
    vorbis_look_psy *p = b->psy + i;
    vorbis_info_psy *pi = p->vi;
    vb200_psy_setup *o = &s.psy[i];
    int n = p->n;
    o->n = n; o->blockflag = pi->blockflag;
    o->ath_adjatt = pi->ath_adjatt; o->ath_maxatt = pi->ath_maxatt;
    for(j = 0; j < P_NOISECURVES; j++) o->tone_masteratt[j] = pi->tone_masteratt[j];
    o->tone_abs_limit = pi->tone_abs_limit; o->noisemaxsupp = pi->noisemaxsupp;
    o->noisewindowfixed = pi->noisewindowfixed;
    for(j = 0; j < NOISE_COMPAND_LEVELS; j++) o->noisecompand[j] = pi->noisecompand[j];
    o->max_curve_dB = pi->max_curve_dB;
    o->normal_p = pi->normal_p; o->normal_start = pi->normal_start;
    o->normal_partition = pi->normal_partition; o->normal_thresh = pi->normal_thresh;
    o->firstoc = (int32_t)p->firstoc; o->shiftoc = (int32_t)p->shiftoc;
    o->eighth_octave_lines = p->eighth_octave_lines; o->total_octave_lines = p->total_octave_lines;
    o->m_val = p->m_val;
    g.octave[i] = (int32_t*)malloc(sizeof(int32_t)*n);
    g.bark[i] = (int32_t*)malloc(sizeof(int32_t)*n);
    g.tonecurves[i] = (float*)malloc(sizeof(float)*P_BANDS*P_LEVELS*(EHMER_MAX+2));
    g.noiseoffset[i] = (float*)malloc(sizeof(float)*P_NOISECURVES*n);
    for(j = 0; j < n; j++){ g.octave[i][j] = (int32_t)p->octave[j]; g.bark[i][j] = (int32_t)p->bark[j]; }
    for(j = 0; j < P_BANDS; j++) for(k = 0; k < P_LEVELS; k++)
      memcpy(g.tonecurves[i] + (j*P_LEVELS+k)*(EHMER_MAX+2), p->tonecurves[j][k], sizeof(float)*(EHMER_MAX+2));
    for(j = 0; j < P_NOISECURVES; j++) memcpy(g.noiseoffset[i] + j*n, p->noiseoffset[j], sizeof(float)*n);
    o->ath = p->ath; o->octave = g.octave[i]; o->bark = g.bark[i];
    o->tonecurves = g.tonecurves[i]; o->noiseoffset = g.noiseoffset[i];
  }
  s.ampmax_att_per_sec = gi->ampmax_att_per_sec;
  for(k = 0; k < PACKETBLOBS; k++){
    for(w = 0; w < 2; w++){
      s.coupling_pointlimit[w][k] = gi->coupling_pointlimit[w][k];
      s.sliding_lowpass[w][k] = gi->sliding_lowpass[w][k];
    }
    s.coupling_prepointamp[k] = gi->coupling_prepointamp[k];
    s.coupling_postpointamp[k] = gi->coupling_postpointamp[k];
  }
  for(w = 0; w < 2 && w < ci->modes; w++){
    vorbis_info_mapping0 *m = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
    s.coupling_steps[w] = m->coupling_steps;
    for(k = 0; k < m->coupling_steps; k++){ s.coupling_mag[w][k] = m->coupling_mag[k]; s.coupling_ang[w][k] = m->coupling_ang[k]; }
  }
  s.window[0] = _vorbis_window_get(b->window[0]);
  s.window[1] = _vorbis_window_get(b->window[1]);
  for(k = 0; k < VE_BANDS; k++){ s.preecho_thresh[k] = gi->preecho_thresh[k]; s.postecho_thresh[k] = gi->postecho_thresh[k]; }
  s.stretch_penalty = gi->stretch_penalty;
  s.preecho_minenergy = gi->preecho_minenergy;
  /* floors per submap (lib/mapping0.c:499-506); only encode-side floor 1 is bound */
  for(w = 0; w < 2 && w < ci->modes && vd->analysisp; w++){
    vorbis_info_mapping0 *m = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
    if(m->submaps > VB200_MAX_SUBMAPS) continue;
    s.submaps[w] = m->submaps;
    for(k = 0; k < vi->channels; k++) s.chmux[w][k] = (uint8_t)m->chmuxlist[k];
    for(j = 0; j < VB200_MAX_SUBMAPS; j++) s.residue[w][j].type = -1;
    for(j = 0; j < m->submaps; j++){
      int fl = m->floorsubmap[j];
      {                                               /* residue class parameters of the submap, lib/mapping0.c:663 */
        int rn = m->residuesubmap[j];
        vorbis_info_residue0 *ri = (vorbis_info_residue0*)ci->residue_param[rn];
        vb200_residue_setup *o = &s.residue[w][j];
        o->type = ci->residue_type[rn];
        o->begin = (int32_t)ri->begin; o->end = (int32_t)ri->end;
        o->grouping = ri->grouping; o->partitions = ri->partitions;
        for(i = 0; i < 64; i++){ o->classmetric1[i] = ri->classmetric1[i]; o->classmetric2[i] = ri->classmetric2[i]; }
      }
      if(ci->floor_type[fl] == 1)
        vb200vs_floor1(&s.floor1[w][j], (vorbis_info_floor1*)ci->floor_param[fl], (vorbis_look_floor1*)b->flr[fl]);
    }
  }
  rc = vb200_ctx_create(&s, device, &g.ctx);
  if(rc){
    fprintf(stderr, "vb200 shim: vb200_ctx_create failed (%d): %s\n", rc, vb200_last_error());
    bind_release(g_cur); g_cur = NULL;
    return rc;
  }
  g.vd = vd; g.setup_key = (void*)vi->codec_setup; g.analysisp = vd->analysisp; g.refs = 1;
  return bind_halfrate(vd);
}

/* drop the calling thread's current binding (the context goes with its last user) */
void vb200shim_detach(void){
  if(!g_cur) return;
  if(--g_cur->refs <= 0) bind_release(g_cur);
  g_cur = NULL;
}
/* make the binding of `vd` current for this thread (a thread that drives several attached states) */
int vb200shim_select(vorbis_dsp_state *vd){
  vb200_binding *b = vb200shim_binding(vd);
  if(!b) return VB200_EINVAL;
  g_cur = b;
  return 0;
}

unsigned long long vb200shim_launches(void){ return (g_cur && g.ctx) ? vb200_launch_count(g.ctx) : 0; }

/* the block-size flag of a transform of n points; half-rate decode builds them at blocksizes[W]>>1 */
static int W_of_n(int n){
  codec_setup_info *ci = (codec_setup_info*)g.vd->vi->codec_setup;
  return n == ci->blocksizes[1] >> ci->halfrate_flag ? 1 : 0;
}
static int look_of(vorbis_look_psy *p){
  private_state *b = (private_state*)g.vd->backend_state;
  return (int)(p - b->psy);
}

/* mdct_forward, lib/mdct.c:492 */
void vb200shim_mdct_forward(mdct_lookup *init, DATA_TYPE *in, DATA_TYPE *out){
  int rc = vb200_mdct_forward(g.ctx, W_of_n(init->n), 1, in, out);
  if(rc) shim_warn("mdct_forward", rc);
}
/* mdct_backward, lib/mdct.c:396 (in == out allowed, as at lib/mapping0.c:794) */
void vb200shim_mdct_backward(mdct_lookup *init, DATA_TYPE *in, DATA_TYPE *out){
  int n = init->n;
  float *tmp = bind_fscratch((size_t)n);
  int rc = tmp ? vb200_mdct_backward(g.ctx, W_of_n(n), 1, in, tmp) : VB200_EFAULT;
  if(rc) shim_warn("mdct_backward", rc); else memcpy(out, tmp, sizeof(float)*n);
}
/* _vorbis_apply_window, lib/window.c:2102 */
void vb200shim_apply_window(float *d, int *winno, long *blocksizes, int lW, int W, int nW){
  int32_t l = lW, r = nW;
  int rc = vb200_apply_window(g.ctx, W, 1, &l, &r, d);
  (void)winno; (void)blocksizes;
  if(rc) shim_warn("apply_window", rc);
}
/* drft_forward, lib/smallft.c:1231 */
void vb200shim_drft_forward(drft_lookup *l, float *data){
  int rc = vb200_drft_forward(g.ctx, W_of_n(l->n), 1, data);
  if(rc) shim_warn("drft_forward", rc);
}
/* _vp_noisemask, lib/psy.c:706 */
void vb200shim_noisemask(vorbis_look_psy *p, float *logmdct, float *logmask){
  int rc = vb200_noisemask(g.ctx, look_of(p), 1, logmdct, logmask);
  if(rc) shim_warn("noisemask", rc);
}
/* _vp_tonemask, lib/psy.c:754 */
void vb200shim_tonemask(vorbis_look_psy *p, float *logfft, float *logmask, float global_specmax, float local_specmax){
  int rc = vb200_tonemask(g.ctx, look_of(p), 1, logfft, &global_specmax, &local_specmax, logmask);
  if(rc) shim_warn("tonemask", rc);
}
/* _vp_offset_and_mix, lib/psy.c:779 */
void vb200shim_offset_and_mix(vorbis_look_psy *p, float *noise, float *tone, int offset_select,
                              float *logmask, float *mdct, float *logmdct){
  int rc = vb200_offset_and_mix(g.ctx, look_of(p), 1, offset_select, noise, tone, mdct, logmdct, logmask);
  if(rc) shim_warn("offset_and_mix", rc);
}
/* _vp_couple_quantize_normalize, lib/psy.c:1014 */
void vb200shim_couple_quantize_normalize(int blobno, vorbis_info_psy_global *gp, vorbis_look_psy *p,
                                         vorbis_info_mapping0 *vi, float **mdct, int **iwork, int *nonzero,
                                         int sliding_lowpass, int ch){
  int look = look_of(p), W = look >> 1, blocktype = look & 1, n = p->n, c, rc;
  float *m = bind_fscratch((size_t)ch*n);
  int32_t *iw = bind_iscratch((size_t)ch*n + ch);
  int32_t *nz = iw ? iw + (size_t)ch*n : NULL;
  (void)gp; (void)vi; (void)sliding_lowpass;
  if(!m || !iw){ shim_warn("couple_quantize_normalize (host scratch)", VB200_EFAULT); return; }
  for(c = 0; c < ch; c++){
    memcpy(m + (size_t)c*n, mdct[c], sizeof(float)*n);
    memcpy(iw + (size_t)c*n, iwork[c], sizeof(int32_t)*n);
    nz[c] = nonzero[c];
  }
  rc = vb200_couple_quantize_normalize(g.ctx, W, blocktype, blobno, 1, m, iw, nz);
  if(rc) shim_warn("couple_quantize_normalize", rc);
  else for(c = 0; c < ch; c++){ memcpy(iwork[c], iw + (size_t)c*n, sizeof(int32_t)*n); nonzero[c] = nz[c]; }
}

/* floor1_fit, lib/floor1.c:576: returns posts in vorbis_block storage, or NULL for a silent channel */
int *vb200shim_floor1_fit(vorbis_block *vb, vorbis_look_floor1 *look, const float *logmdct, const float *logmask){
  { vb200_binding *bb = vb200shim_binding(vb->vd); if(bb) g_cur = bb; }
  codec_setup_info *ci = (codec_setup_info*)g.vd->vi->codec_setup;
  private_state *b = (private_state*)g.vd->backend_state;
  vorbis_info_mapping0 *m = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[vb->W]->mapping];
  int32_t posts[VB200_FLOOR1_STRIDE], nz = 0;
  int sel = -1, j, rc, *out;
  for(j = 0; j < m->submaps; j++) if((void*)b->flr[m->floorsubmap[j]] == (void*)look) sel = j;
  if(sel < 0){ fprintf(stderr, "vb200 shim: floor1_fit: unknown floor look\n"); return NULL; }
  rc = vb200_floor1_fit(g.ctx, (int)vb->W, sel, 1, logmdct, logmask, posts, &nz);
  if(rc){ shim_warn("floor1_fit", rc); return NULL; }
  if(!nz) return NULL;
  out = (int*)_vorbis_block_alloc(vb, sizeof(*out) * look->posts);
  for(j = 0; j < look->posts; j++) out[j] = posts[j];
  return out;
}

/* _ve_envelope_search, lib/envelope.c:216-327.  The analysis loop (:232-267: _ve_amp on every new
 * 64-sample step of every channel, the stretch logic, the marks) runs on the device; the walk of
 * the cursor over the marks that picks the next block size (:269-327) is host control flow over a
 * handful of ints and is restated here.  The filter state is handed over in the reference's own
 * envelope_filter_state layout, so ve->filter / ve->stretch stay authoritative between calls.  */
/* the analysis part of _ve_envelope_search split in two so that a driver of many states can run ONE device call
 * for all of them (vb200_mapping0.c): prepare reports which steps are new, commit stores what the device found */
int vb200shim_envelope_prepare(vorbis_dsp_state *v, int *first_out){
  envelope_lookup *ve = ((private_state*)(v->backend_state))->ve;
  int first = ve->current/ve->searchstep;
  int last = v->pcm_current/ve->searchstep - VE_WIN;
  if(first < 0) first = 0;
  if(last + VE_WIN + VE_POST > ve->storage){                   /* lib/envelope.c:227-230 */
    ve->storage = last + VE_WIN + VE_POST;
    ve->mark = (int*)realloc(ve->mark, ve->storage*sizeof(*ve->mark));
  }
  *first_out = first;
  return last > first ? last - first : 0;
}
void vb200shim_envelope_state_get(vorbis_dsp_state *v, int32_t *state){
  envelope_lookup *ve = ((private_state*)(v->backend_state))->ve;
  state[0] = ve->stretch;
  memcpy(state + 1, ve->filter, sizeof(envelope_filter_state)*VE_BANDS*ve->ch);
}
void vb200shim_envelope_commit(vorbis_dsp_state *v, int first, int nsteps, const int32_t *state, const uint8_t *ret){
  envelope_lookup *ve = ((private_state*)(v->backend_state))->ve;
  ve->stretch = state[0];
  memcpy(ve->filter, state + 1, sizeof(envelope_filter_state)*VE_BANDS*ve->ch);
  vb200_envelope_apply_marks(ret, first, nsteps, (int32_t*)ve->mark);   /* int == int32_t on every libvorbis target */
  ve->current = (first + nsteps)*ve->searchstep;
}

long vb200shim_envelope_search(vorbis_dsp_state *v){
  vorbis_info *vi = v->vi;
  codec_setup_info *ci = (codec_setup_info*)vi->codec_setup;
  envelope_lookup *ve = ((private_state*)(v->backend_state))->ve;
  long j;
  int first, nsteps, last;
  { vb200_binding *bb = vb200shim_binding(v); if(bb) g_cur = bb; }   /* every block starts here: the state's binding becomes current */
  nsteps = vb200shim_envelope_prepare(v, &first);
  last = v->pcm_current/ve->searchstep - VE_WIN;
  if(nsteps > 0){
    const int ch = ve->ch;
    const long len = (long)ve->searchstep*(nsteps - 1) + ve->winlength;
    float *tmp = bind_fscratch((size_t)ch*len);
    int32_t *state = bind_iscratch((size_t)VB200_VE_STATE_WORDS(ch) + (size_t)(nsteps + 3)/4 + 1);
    uint8_t *ret = state ? (uint8_t*)(state + VB200_VE_STATE_WORDS(ch)) : NULL;
    int c, rc;
    if(!tmp || !state){ shim_warn("envelope_search (host scratch)", VB200_EFAULT); }
    else{
      for(c = 0; c < ch; c++) memcpy(tmp + (size_t)c*len, v->pcm[c] + (long)ve->searchstep*first, sizeof(float)*len);
      vb200shim_envelope_state_get(v, state);
      rc = vb200_envelope_search(g.ctx, 1, tmp, VB200_PCM_F32_PLANAR, len, 0, nsteps, state, ret);
      if(rc) shim_warn("envelope_search", rc);
      else vb200shim_envelope_commit(v, first, nsteps, state, ret);
    }
  }
  ve->current = last*ve->searchstep;
  {                                                            /* :269-327 */
    long centerW = v->centerW;
    long testW = centerW + ci->blocksizes[v->W]/4 + ci->blocksizes[1]/2 + ci->blocksizes[0]/4;
    j = ve->cursor;
    while(j < ve->current - ve->searchstep){
      if(j >= testW) return 1;
      ve->cursor = j;
      if(ve->mark[j/ve->searchstep] && j > centerW){
        ve->curmark = j;
        return j >= testW ? 1 : 0;
      }
      j += ve->searchstep;
    }
  }
  return -1;
}
