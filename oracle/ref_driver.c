/* ref_driver.c — thin driver around the UNMODIFIED reference sources.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is compiled together with the
 * reference C sources under lib/ (read in place from /root/reference, never copied)
 * into oracle/_ref/libvorbis_ref.so by oracle/Makefile.  It
 *   (1) exposes the reference's hot-path functions (mdct_forward, drft_forward,
 *       _vorbis_apply_window, _vp_noisemask, _vp_tonemask, _vp_offset_and_mix,
 *       _vp_couple_quantize_normalize, mdct_backward, vorbis_synthesis_blockin)
 *       behind flat C entry points that ctypes can call;
 *   (2) dumps the lookup tables the reference builds in _vds_shared_init
 *       (lib/block.c:170) into the vb200_setup layout of include/vorbis_b200.h;
 *   (3) runs the real encoder / decoder API loop (as in
 *       examples/encoder_example.c:210-235) and records every intermediate
 *       vector of mapping0_forward / mapping0_inverse.  The recording works by
 *       compiling lib/mapping0.c with -D<callee>=spy_<callee> (see Makefile):
 *       the reference source is unchanged, its calls just land in the spy_*
 *       functions below, which copy the arguments and forward to the real
 *       callee.
 * Nothing here is on the product path.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"
#include "codec_internal.h"
#include "registry.h"
#include "mdct.h"
#include "smallft.h"
#include "window.h"
#include "psy.h"
#include "scales.h"

#include "vorbis_b200.h"

/* ------------------------------------------------------------------------ */
typedef struct ref_handle {
  vorbis_info      vi;
  vorbis_comment   vc;
  vorbis_dsp_state vd;
  vorbis_block     vb;
  int              channels;
  long             rate;
  /* converted copies of tables for vb200_setup */
  int32_t *octave[4];
  int32_t *bark[4];
  float   *tonecurves[4];
  float   *noiseoffset[4];
  /* encoded packets kept for the decode capture */
  unsigned char **pkt;
  long  *pktbytes;
  int    npkt, pktcap;
  ogg_packet hdr[3];
  unsigned char *hdrcopy[3];
} ref_handle;

void *ref_open(int channels, long rate, float quality){
  ref_handle *h = (ref_handle*)calloc(1, sizeof(*h));
  vorbis_info_init(&h->vi);
  if(vorbis_encode_init_vbr(&h->vi, channels, rate, quality)){
    vorbis_info_clear(&h->vi);
    free(h);
    return NULL;
  }
  vorbis_comment_init(&h->vc);
  vorbis_analysis_init(&h->vd, &h->vi);
  vorbis_block_init(&h->vd, &h->vb);
  h->channels = channels;
  h->rate = rate;
  return h;
}

/* a bitrate-managed encoder (vorbis_encode_init with a nominal bitrate: lib/vorbisenc.c:1199-1222): mapping0_forward
 * then builds all PACKETBLOBS packets per block and lib/bitrate.c picks one */
void *ref_open_managed(int channels, long rate, long nominal_bitrate){
  ref_handle *h = (ref_handle*)calloc(1, sizeof(*h));
  vorbis_info_init(&h->vi);
  if(vorbis_encode_init(&h->vi, channels, rate, -1, nominal_bitrate, -1)){
    vorbis_info_clear(&h->vi);
    free(h);
    return NULL;
  }
  vorbis_comment_init(&h->vc);
  vorbis_analysis_init(&h->vd, &h->vi);
  vorbis_block_init(&h->vd, &h->vb);
  h->channels = channels;
  h->rate = rate;
  return h;
}

void ref_close(void *hv){
  ref_handle *h = (ref_handle*)hv;
  int i;
  if(!h) return;
  for(i=0;i<4;i++){
    free(h->octave[i]); free(h->bark[i]); free(h->tonecurves[i]); free(h->noiseoffset[i]);
  }
  for(i=0;i<h->npkt;i++) free(h->pkt[i]);
  free(h->pkt); free(h->pktbytes);
  for(i=0;i<3;i++) free(h->hdrcopy[i]);
  vorbis_block_clear(&h->vb);
  vorbis_dsp_clear(&h->vd);
  vorbis_comment_clear(&h->vc);
  vorbis_info_clear(&h->vi);
  free(h);
}

/* accessors used by the drop-in integration test */
void *ref_vd(void *hv){ return &((ref_handle*)hv)->vd; }

/* concatenated packet bytes kept by ref_encode_capture; returns number of packets */
int ref_get_packets(void *hv, unsigned char *buf, long cap, long *sizes, int maxn){
  ref_handle *h = (ref_handle*)hv;
  long off = 0; int i;
  for(i = 0; i < h->npkt && i < maxn; i++){
    if(off + h->pktbytes[i] > cap) return -1;
    memcpy(buf + off, h->pkt[i], h->pktbytes[i]);
    sizes[i] = h->pktbytes[i];
    off += h->pktbytes[i];
  }
  return i;
}

/* the three header packets ref_encode_capture wrote, back to back; returns 3, or -1 before the capture or when they do
 * not fit in cap bytes */
int ref_get_headers(void *hv, unsigned char *buf, long cap, long *sizes){
  ref_handle *h = (ref_handle*)hv;
  long off = 0; int i;
  if(!h->hdrcopy[0]) return -1;
  for(i = 0; i < 3; i++){
    if(off + h->hdr[i].bytes > cap) return -1;
    memcpy(buf + off, h->hdr[i].packet, h->hdr[i].bytes);
    sizes[i] = h->hdr[i].bytes;
    off += h->hdr[i].bytes;
  }
  return 3;
}

int ref_blocksize(void *hv, int W){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  return (int)ci->blocksizes[W];
}

/* fill a vb200_setup from the reference's own lookups */
int ref_get_setup(void *hv, vb200_setup *s){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_info_psy_global *g = &ci->psy_g_param;
  int i,j,k,w;
  memset(s,0,sizeof(*s));
  s->channels = h->vi.channels;
  s->rate = (int32_t)h->vi.rate;
  s->blocksizes[0] = (int32_t)ci->blocksizes[0];
  s->blocksizes[1] = (int32_t)ci->blocksizes[1];
  s->n_psy = ci->psys;
  if(ci->psys != 4) return -1;
  for(i=0;i<4;i++){
    vorbis_look_psy *p = b->psy+i;
    vorbis_info_psy *pi = p->vi;
    vb200_psy_setup *o = &s->psy[i];
    int n = p->n;
    o->n = n;
    o->blockflag = pi->blockflag;
    o->ath_adjatt = pi->ath_adjatt;
    o->ath_maxatt = pi->ath_maxatt;
    for(j=0;j<P_NOISECURVES;j++) o->tone_masteratt[j] = pi->tone_masteratt[j];
    o->tone_abs_limit = pi->tone_abs_limit;
    o->noisemaxsupp = pi->noisemaxsupp;
    o->noisewindowfixed = pi->noisewindowfixed;
    for(j=0;j<NOISE_COMPAND_LEVELS;j++) o->noisecompand[j] = pi->noisecompand[j];
    o->max_curve_dB = pi->max_curve_dB;
    o->normal_p = pi->normal_p;
    o->normal_start = pi->normal_start;
    o->normal_partition = pi->normal_partition;
    o->normal_thresh = pi->normal_thresh;
    o->firstoc = (int32_t)p->firstoc;
    o->shiftoc = (int32_t)p->shiftoc;
    o->eighth_octave_lines = p->eighth_octave_lines;
    o->total_octave_lines = p->total_octave_lines;
    o->m_val = p->m_val;
    o->ath = p->ath;
    if(!h->octave[i]){
      h->octave[i] = (int32_t*)malloc(sizeof(int32_t)*n);
      h->bark[i]   = (int32_t*)malloc(sizeof(int32_t)*n);
      h->tonecurves[i] = (float*)malloc(sizeof(float)*P_BANDS*P_LEVELS*(EHMER_MAX+2));
      h->noiseoffset[i] = (float*)malloc(sizeof(float)*P_NOISECURVES*n);
      for(j=0;j<n;j++){ h->octave[i][j]=(int32_t)p->octave[j]; h->bark[i][j]=(int32_t)p->bark[j]; }
      for(j=0;j<P_BANDS;j++)for(k=0;k<P_LEVELS;k++)
        memcpy(h->tonecurves[i]+(j*P_LEVELS+k)*(EHMER_MAX+2), p->tonecurves[j][k], sizeof(float)*(EHMER_MAX+2));
      for(j=0;j<P_NOISECURVES;j++)
        memcpy(h->noiseoffset[i]+j*n, p->noiseoffset[j], sizeof(float)*n);
    }
    o->octave = h->octave[i];
    o->bark = h->bark[i];
    o->tonecurves = h->tonecurves[i];
    o->noiseoffset = h->noiseoffset[i];
  }
  s->ampmax_att_per_sec = g->ampmax_att_per_sec;
  for(k=0;k<PACKETBLOBS;k++){
    s->coupling_pointlimit[0][k]=g->coupling_pointlimit[0][k];
    s->coupling_pointlimit[1][k]=g->coupling_pointlimit[1][k];
    s->coupling_prepointamp[k]=g->coupling_prepointamp[k];
    s->coupling_postpointamp[k]=g->coupling_postpointamp[k];
    s->sliding_lowpass[0][k]=g->sliding_lowpass[0][k];
    s->sliding_lowpass[1][k]=g->sliding_lowpass[1][k];
  }
  for(w=0;w<2;w++){
    /* mode w uses map_param[mode_param[w]->mapping]; vorbisenc sets modes==maps */
    vorbis_info_mapping0 *m = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
    s->coupling_steps[w]=m->coupling_steps;
    for(k=0;k<m->coupling_steps;k++){
      s->coupling_mag[w][k]=m->coupling_mag[k];
      s->coupling_ang[w][k]=m->coupling_ang[k];
    }
  }
  s->window[0] = _vorbis_window_get(b->window[0]);
  s->window[1] = _vorbis_window_get(b->window[1]);
  for(k=0;k<VE_BANDS;k++){
    s->preecho_thresh[k] = g->preecho_thresh[k];
    s->postecho_thresh[k] = g->postecho_thresh[k];
  }
  s->stretch_penalty = g->stretch_penalty;
  s->preecho_minenergy = g->preecho_minenergy;
  for(w=0;w<2;w++){
    vorbis_info_mapping0 *m = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
    int sm;
    if(m->submaps > VB200_MAX_SUBMAPS) return -1;
    s->submaps[w] = m->submaps;
    for(k=0;k<h->vi.channels;k++) s->chmux[w][k] = (uint8_t)m->chmuxlist[k];
    for(sm=0;sm<VB200_MAX_SUBMAPS;sm++) s->residue[w][sm].type = -1;
    for(sm=0;sm<m->submaps;sm++){
      int fl = m->floorsubmap[sm];
      {
        int rn = m->residuesubmap[sm];
        vorbis_info_residue0 *ri = (vorbis_info_residue0*)ci->residue_param[rn];
        vb200_residue_setup *o = &s->residue[w][sm];
        o->type = ci->residue_type[rn];
        o->begin = (int32_t)ri->begin; o->end = (int32_t)ri->end;
        o->grouping = ri->grouping; o->partitions = ri->partitions;
        for(k=0;k<64;k++){ o->classmetric1[k] = ri->classmetric1[k]; o->classmetric2[k] = ri->classmetric2[k]; }
      }
      if(ci->floor_type[fl]==1){
        vorbis_info_floor1 *fi = (vorbis_info_floor1*)ci->floor_param[fl];
        vorbis_look_floor1 *lk = (vorbis_look_floor1*)b->flr[fl];
        vb200_floor1_setup *o = &s->floor1[w][sm];
        o->posts = lk->posts;
        for(k=0;k<lk->posts;k++) o->postlist[k]=fi->postlist[k];
        o->mult = fi->mult; o->n = lk->n;
        o->maxover = fi->maxover; o->maxunder = fi->maxunder; o->maxerr = fi->maxerr;
        o->twofitweight = fi->twofitweight; o->twofitatten = fi->twofitatten;
      }
    }
  }
  return 0;
}

/* rewrite the coupling map of the mapping mode W uses (vorbisenc writes one mapping per mode): every later call on the
 * handle - the stage calls, the batched chains, ref_get_setup and the setup header ref_encode_capture writes - sees
 * the new map.  The map is not checked: the caller passes one mapping0_unpack accepts.  Returns 0, or -1 when the
 * two modes share a mapping or steps is out of range.                                                              */
int ref_set_coupling(void *hv, int W, int steps, const int32_t *mag, const int32_t *ang){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  vorbis_info_mapping0 *m;
  int k;
  if(W < 0 || W > 1 || ci->modes < 2 || ci->mode_param[0]->mapping == ci->mode_param[1]->mapping) return -1;
  m = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
  if(steps < 0 || steps > (int)(sizeof(m->coupling_mag)/sizeof(m->coupling_mag[0]))) return -1;
  m->coupling_steps = steps;
  for(k = 0; k < steps; k++){ m->coupling_mag[k] = mag[k]; m->coupling_ang[k] = ang[k]; }
  return 0;
}

/* copies of the reference's derived transform tables (for table parity tests):
 * which: 0 mdct trig (N+N/4), 1 bitrev (N/4), 2 window (N/2), 3 fft wa (N) */
int ref_get_table(void *hv, int W, int which, void *dst, int cap){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  int N = (int)ci->blocksizes[W];
  mdct_lookup *m = (mdct_lookup*)b->transform[W][0];
  switch(which){
  case 0: if(cap<N+N/4) return -1; memcpy(dst,m->trig,sizeof(float)*(N+N/4)); return N+N/4;
  case 1: if(cap<N/4) return -1; memcpy(dst,m->bitrev,sizeof(int)*(N/4)); return N/4;
  case 2: if(cap<N/2) return -1; memcpy(dst,_vorbis_window_get(b->window[W]),sizeof(float)*(N/2)); return N/2;
  case 3: if(cap<N) return -1; memcpy(dst,b->fft_look[W].trigcache+N,sizeof(float)*N); return N;
  }
  return -1;
}

/* ---- stage-level calls into the reference ------------------------------ */
void ref_mdct_forward(void *hv, int W, int nvec, const float *in, float *out){
  ref_handle *h = (ref_handle*)hv;
  private_state *b = (private_state*)h->vd.backend_state;
  int N = ref_blocksize(hv,W), v;
  float *tmp = (float*)malloc(sizeof(float)*N);
  for(v=0;v<nvec;v++){
    memcpy(tmp,in+(size_t)v*N,sizeof(float)*N);
    mdct_forward((mdct_lookup*)b->transform[W][0],tmp,out+(size_t)v*(N/2));
  }
  free(tmp);
}

void ref_mdct_backward(void *hv, int W, int nvec, const float *in, float *out){
  ref_handle *h = (ref_handle*)hv;
  private_state *b = (private_state*)h->vd.backend_state;
  int N = ref_blocksize(hv,W), v;
  for(v=0;v<nvec;v++){
    float *o = out+(size_t)v*N;
    memcpy(o,in+(size_t)v*(N/2),sizeof(float)*(N/2));
    mdct_backward((mdct_lookup*)b->transform[W][0],o,o); /* in place, as lib/mapping0.c:794 */
  }
}

void ref_apply_window(void *hv, int W, int nvec, const int32_t *lW, const int32_t *nW, float *data){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  int N = ref_blocksize(hv,W), v;
  for(v=0;v<nvec;v++)
    _vorbis_apply_window(data+(size_t)v*N,b->window,ci->blocksizes,lW?lW[v]:0,W,nW?nW[v]:0);
}

void ref_drft_forward(void *hv, int W, int nvec, float *data){
  ref_handle *h = (ref_handle*)hv;
  private_state *b = (private_state*)h->vd.backend_state;
  int N = ref_blocksize(hv,W), v;
  for(v=0;v<nvec;v++) drft_forward(&b->fft_look[W],data+(size_t)v*N);
}

void ref_noisemask(void *hv, int look, int nvec, const float *logmdct, float *noise){
  ref_handle *h = (ref_handle*)hv;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_look_psy *p = b->psy+look;
  int n = p->n, v;
  float *tmp = (float*)malloc(sizeof(float)*n);
  for(v=0;v<nvec;v++){
    memcpy(tmp,logmdct+(size_t)v*n,sizeof(float)*n);
    _vp_noisemask(p,tmp,noise+(size_t)v*n);
  }
  free(tmp);
}

void ref_tonemask(void *hv, int look, int nvec, const float *logfft,
                  const float *gmax, const float *lmax, float *tone){
  ref_handle *h = (ref_handle*)hv;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_look_psy *p = b->psy+look;
  int n = p->n, v;
  float *tmp = (float*)malloc(sizeof(float)*n);
  for(v=0;v<nvec;v++){
    memcpy(tmp,logfft+(size_t)v*n,sizeof(float)*n);
    _vp_tonemask(p,tmp,tone+(size_t)v*n,gmax[v],lmax[v]);
  }
  free(tmp);
}

void ref_offset_and_mix(void *hv, int look, int nvec, int offset_select,
                        const float *noise, const float *tone,
                        float *mdct, const float *logmdct, float *logmask){
  ref_handle *h = (ref_handle*)hv;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_look_psy *p = b->psy+look;
  int n = p->n, v;
  for(v=0;v<nvec;v++){
    size_t o=(size_t)v*n;
    _vp_offset_and_mix(p,(float*)noise+o,(float*)tone+o,offset_select,logmask+o,mdct+o,(float*)logmdct+o);
  }
}

/* _vp_couple_quantize_normalize over a batch; layouts [block][ch][n] */
void ref_couple_quantize_normalize(void *hv, int W, int blocktype, int blobno, int nblocks,
                                   float *mdct, int32_t *iwork, int32_t *nonzero){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_look_psy *p = b->psy+blocktype+(W?2:0);
  vorbis_info_mapping0 *info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
  int ch = h->vi.channels, n = p->n, blk, c;
  float **m = (float**)malloc(sizeof(*m)*ch);
  int   **iw = (int**)malloc(sizeof(*iw)*ch);
  int    *nz = (int*)malloc(sizeof(int)*ch);
  for(blk=0;blk<nblocks;blk++){
    for(c=0;c<ch;c++){
      m[c] = mdct+((size_t)blk*ch+c)*n;
      iw[c] = (int*)(iwork+((size_t)blk*ch+c)*n);
      nz[c] = nonzero[(size_t)blk*ch+c];
    }
    _vp_couple_quantize_normalize(blobno,&ci->psy_g_param,p,info,m,iw,nz,
                                  ci->psy_g_param.sliding_lowpass[W][blobno],ch);
    for(c=0;c<ch;c++) nonzero[(size_t)blk*ch+c]=nz[c];
  }
  free(m); free(iw); free(nz);
}

float ref_ampmax_decay(void *hv, float amp, int W){
  ref_handle *h = (ref_handle*)hv;
  long save = h->vd.W;
  float r;
  h->vd.W = W;
  r = _vp_ampmax_decay(amp,&h->vd);
  h->vd.W = save;
  return r;
}

/* ---- capture of the real API loop --------------------------------------- */
typedef struct ref_capture {
  int   maxblocks;
  int   Nmax;            /* row stride for N-long vectors; n-long use Nmax/2 */
  int   nblocks;         /* out: blocks seen */
  /* per block */
  int32_t *W, *lW, *nW, *blocktype;
  float   *ampmax_in, *ampmax_out;
  /* per block x channel; NULL = don't capture */
  float *pcm;        /* [blk][ch][Nmax]  vb->pcm before windowing */
  float *windowed;   /* [blk][ch][Nmax] */
  float *fft;        /* [blk][ch][Nmax]  drft_forward output */
  float *mdct_raw;   /* [blk][ch][Nmax/2] */
  float *logfft;     /* tonemask input */
  float *logmdct;    /* noisemask input */
  float *noise;
  float *tone;
  float *logmask;    /* after offset_and_mix(select 1) */
  float *mdct_m1;    /* gmdct after offset_and_mix(select 1) */
  float *local_ampmax;   /* [blk][ch] */
  float *global_ampmax;  /* [blk] value passed to _vp_tonemask */
  int32_t *ilogmask;     /* [blk][ch][Nmax/2] iwork entering CQN (blob 7) */
  int32_t *iwork_out;    /* [blk][ch][Nmax/2] iwork leaving CQN */
  int32_t *nonzero_in;   /* [blk][ch] */
  int32_t *nonzero_out;  /* [blk][ch] */
  int32_t *fit_posts;    /* [blk][ch][65] output of floor1_fit (blob 7); [0] = -1 when NULL */
  int32_t *enc_posts;    /* [blk][ch][65] post[] after floor1_encode's quantise/predict pass */
  /* decode side */
  float *dec_coef;   /* [blk][ch][Nmax/2] input of mdct_backward */
  float *dec_imdct;  /* [blk][ch][Nmax]   output of mdct_backward */
} ref_capture;

static ref_capture *g_cap = NULL;
static int g_blk = -1;
static int g_ch_total = 0;
static int g_cnt_window, g_cnt_mdct, g_cnt_fft, g_cnt_noise, g_cnt_tone, g_cnt_mix, g_cnt_imdct, g_cnt_fit, g_cnt_enc;

static int cap_on(void){ return g_cap && g_blk>=0 && g_blk<g_cap->maxblocks; }
static float *rowN(float *base,int c){ return base+((size_t)g_blk*g_ch_total+c)*g_cap->Nmax; }
static float *rown(float *base,int c){ return base+((size_t)g_blk*g_ch_total+c)*(g_cap->Nmax/2); }
static int32_t *irown(int32_t *base,int c){ return base+((size_t)g_blk*g_ch_total+c)*(g_cap->Nmax/2); }

/* spies: lib/mapping0.c is compiled with -D<name>=spy_<name> (oracle/Makefile) */
void spy__vorbis_apply_window(float *d,int *winno,long *blocksizes,int lW,int W,int nW){
  int N = (int)blocksizes[W];
  int c = g_cnt_window++;
  if(cap_on() && g_cap->pcm) memcpy(rowN(g_cap->pcm,c),d,sizeof(float)*N);
  _vorbis_apply_window(d,winno,blocksizes,lW,W,nW);
  if(cap_on() && g_cap->windowed) memcpy(rowN(g_cap->windowed,c),d,sizeof(float)*N);
}

void spy_mdct_forward(mdct_lookup *init, float *in, float *out){
  int c = g_cnt_mdct++;
  mdct_forward(init,in,out);
  if(cap_on() && g_cap->mdct_raw) memcpy(rown(g_cap->mdct_raw,c),out,sizeof(float)*(init->n/2));
}

void spy_drft_forward(drft_lookup *l,float *data){
  int c = g_cnt_fft++;
  drft_forward(l,data);
  if(cap_on() && g_cap->fft) memcpy(rowN(g_cap->fft,c),data,sizeof(float)*l->n);
}

void spy__vp_noisemask(vorbis_look_psy *p,float *logmdct,float *logmask){
  int c = g_cnt_noise++;
  if(cap_on() && g_cap->logmdct) memcpy(rown(g_cap->logmdct,c),logmdct,sizeof(float)*p->n);
  _vp_noisemask(p,logmdct,logmask);
  if(cap_on() && g_cap->noise) memcpy(rown(g_cap->noise,c),logmask,sizeof(float)*p->n);
}

void spy__vp_tonemask(vorbis_look_psy *p,float *logfft,float *logmask,float gmax,float lmax){
  int c = g_cnt_tone++;
  if(cap_on()){
    if(g_cap->logfft) memcpy(rown(g_cap->logfft,c),logfft,sizeof(float)*p->n);
    if(g_cap->local_ampmax) g_cap->local_ampmax[(size_t)g_blk*g_ch_total+c]=lmax;
    if(g_cap->global_ampmax) g_cap->global_ampmax[g_blk]=gmax;
  }
  _vp_tonemask(p,logfft,logmask,gmax,lmax);
  if(cap_on() && g_cap->tone) memcpy(rown(g_cap->tone,c),logmask,sizeof(float)*p->n);
}

void spy__vp_offset_and_mix(vorbis_look_psy *p,float *noise,float *tone,int offset_select,
                            float *logmask,float *mdct,float *logmdct){
  _vp_offset_and_mix(p,noise,tone,offset_select,logmask,mdct,logmdct);
  if(offset_select==1){
    int c = g_cnt_mix++;
    if(cap_on()){
      if(g_cap->logmask) memcpy(rown(g_cap->logmask,c),logmask,sizeof(float)*p->n);
      if(g_cap->mdct_m1) memcpy(rown(g_cap->mdct_m1,c),mdct,sizeof(float)*p->n);
    }
  }
}

void spy__vp_couple_quantize_normalize(int blobno,vorbis_info_psy_global *g,vorbis_look_psy *p,
                                       vorbis_info_mapping0 *vi,float **mdct,int **iwork,
                                       int *nonzero,int sliding_lowpass,int ch){
  int c, on = cap_on() && blobno==PACKETBLOBS/2;
  if(on){
    for(c=0;c<ch;c++){
      if(g_cap->ilogmask) memcpy(irown(g_cap->ilogmask,c),iwork[c],sizeof(int)*p->n);
      if(g_cap->nonzero_in) g_cap->nonzero_in[(size_t)g_blk*g_ch_total+c]=nonzero[c];
    }
  }
  _vp_couple_quantize_normalize(blobno,g,p,vi,mdct,iwork,nonzero,sliding_lowpass,ch);
  if(on){
    for(c=0;c<ch;c++){
      if(g_cap->iwork_out) memcpy(irown(g_cap->iwork_out,c),iwork[c],sizeof(int)*p->n);
      if(g_cap->nonzero_out) g_cap->nonzero_out[(size_t)g_blk*g_ch_total+c]=nonzero[c];
    }
  }
}

/* floor1_fit / floor1_encode (lib/floor1.c:576,753) as called from mapping0_forward (:500,:617).
 * Only the first fit per channel is the PACKETBLOBS/2 one in non-managed mode. */
int *spy_floor1_fit(vorbis_block *vb,vorbis_look_floor1 *look,const float *logmdct,const float *logmask){
  int c = g_cnt_fit++;
  int *r = floor1_fit(vb,look,logmdct,logmask);
  if(cap_on() && g_cap->fit_posts && c < g_ch_total){
    int32_t *dst = g_cap->fit_posts + ((size_t)g_blk*g_ch_total+c)*65;
    int k;
    for(k=0;k<65;k++) dst[k] = 0;
    if(!r) dst[0] = -1; else for(k=0;k<look->posts;k++) dst[k]=r[k];
  }
  return r;
}
int spy_floor1_encode(oggpack_buffer *opb,vorbis_block *vb,vorbis_look_floor1 *look,int *post,int *ilogmask){
  int c = g_cnt_enc++;
  int r = floor1_encode(opb,vb,look,post,ilogmask);
  if(cap_on() && g_cap->enc_posts && c < g_ch_total){
    int32_t *dst = g_cap->enc_posts + ((size_t)g_blk*g_ch_total+c)*65;
    int k;
    for(k=0;k<65;k++) dst[k] = 0;
    if(!post) dst[0] = -1; else for(k=0;k<look->posts;k++) dst[k]=post[k];
  }
  return r;
}

void spy_mdct_backward(mdct_lookup *init, float *in, float *out){
  int c = g_cnt_imdct++;
  if(cap_on() && g_cap->dec_coef) memcpy(rown(g_cap->dec_coef,c),in,sizeof(float)*(init->n/2));
  mdct_backward(init,in,out);
  if(cap_on() && g_cap->dec_imdct) memcpy(rowN(g_cap->dec_imdct,c),out,sizeof(float)*init->n);
}

static void keep_packet(ref_handle *h, ogg_packet *op){
  if(h->npkt==h->pktcap){
    h->pktcap = h->pktcap? h->pktcap*2 : 64;
    h->pkt = (unsigned char**)realloc(h->pkt,sizeof(*h->pkt)*h->pktcap);
    h->pktbytes = (long*)realloc(h->pktbytes,sizeof(*h->pktbytes)*h->pktcap);
  }
  h->pkt[h->npkt] = (unsigned char*)malloc(op->bytes? op->bytes:1);
  memcpy(h->pkt[h->npkt],op->packet,op->bytes);
  h->pktbytes[h->npkt] = op->bytes;
  h->npkt++;
}

/* Optional: record the stream's timeline as the encoder sees it - v->pcm[][] re-assembled in absolute
 * samples (sample 0 = v->pcm[][0] of the fresh state): the (pre-extrapolated) preamble of
 * blocksizes[1]/2 samples, the input, and the extrapolated tail that vorbis_analysis_wrote(v,0)
 * appends.  The buffer is [ch][cap]; *len_out = samples recorded, *eof_out = v->eofflag in the
 * same coordinates.  Call before ref_encode_capture; cleared by it.                                */
#ifdef VB200_DROPIN
int vb200_vorbis_analysis(vorbis_block *vb, ogg_packet *op);   /* vorbis_b200/host/vb200_mapping0.c */
static int g_seam1 = 0;
void ref_use_block_seam(int on){ g_seam1 = on; }   /* ref_encode_capture: vorbis_analysis through vb200_mapping0_exportbundle */
#endif
static long g_chunk = 0;
void ref_set_chunk(long n){ g_chunk = n; }   /* samples per vorbis_analysis_wrote of ref_encode_capture (default 1024) */
static float *g_tl = NULL; static long g_tl_cap = 0, g_tl_len = 0, g_tl_shift = 0, g_tl_eof = 0;
void ref_set_timeline(float *buf, long cap){ g_tl = buf; g_tl_cap = cap; g_tl_len = 0; g_tl_shift = 0; g_tl_eof = 0; }
void ref_get_timeline(long *len_out, long *eof_out){ if(len_out) *len_out = g_tl_len; if(eof_out) *eof_out = g_tl_eof; }
static void tl_record(ref_handle *h){
  int c; long k;
  if(!g_tl) return;
  for(c=0;c<h->channels;c++)
    for(k=0;k<h->vd.pcm_current;k++)
      if(g_tl_shift+k<g_tl_cap) g_tl[(size_t)c*g_tl_cap+g_tl_shift+k] = h->vd.pcm[c][k];
  if(g_tl_shift+h->vd.pcm_current>g_tl_len) g_tl_len = g_tl_shift+h->vd.pcm_current;
  if(h->vd.eofflag>0 && !g_tl_eof) g_tl_eof = g_tl_shift+h->vd.eofflag;
}

/* Encode `nsamples` samples per channel (pcm = [ch][nsamples]) through the
 * reference API, capturing into *cap.  Returns number of blocks, and the
 * total packet bytes in *bytes_out.  The handle must be fresh (one use).   */
int ref_encode_capture(void *hv, const float *pcm, long nsamples, ref_capture *cap, long *bytes_out){
  ref_handle *h = (ref_handle*)hv;
  long pos = 0, total = 0;
  int blocks = 0, i, eos = 0;
  ogg_packet op;
  const long chunk = g_chunk > 0 ? g_chunk : 1024;

  vorbis_analysis_headerout(&h->vd,&h->vc,&h->hdr[0],&h->hdr[1],&h->hdr[2]);
  for(i=0;i<3;i++){
    h->hdrcopy[i] = (unsigned char*)malloc(h->hdr[i].bytes);
    memcpy(h->hdrcopy[i],h->hdr[i].packet,h->hdr[i].bytes);
    h->hdr[i].packet = h->hdrcopy[i];
  }

  g_cap = cap; g_ch_total = h->channels;
  if(cap) cap->nblocks = 0;
  while(!eos){
    long todo = nsamples-pos < chunk ? nsamples-pos : chunk;
    if(todo>0){
      float **buf = vorbis_analysis_buffer(&h->vd,(int)todo);
      for(i=0;i<h->channels;i++) memcpy(buf[i],pcm+(size_t)i*nsamples+pos,sizeof(float)*todo);
      vorbis_analysis_wrote(&h->vd,(int)todo);
      pos += todo;
    }else{
      vorbis_analysis_wrote(&h->vd,0);
    }
    tl_record(h);
    while(1){
      long cw_before = h->vd.centerW, pc_before = h->vd.pcm_current;
      vorbis_block_internal *vbi = (vorbis_block_internal*)h->vb.internal;
      if(vorbis_analysis_blockout(&h->vd,&h->vb)!=1) break;
      /* blockout moved the buffer by movementW = what pcm_current lost (lib/block.c:659) */
      g_tl_shift += pc_before - h->vd.pcm_current; (void)cw_before;
      g_blk = blocks;
      g_cnt_window=g_cnt_mdct=g_cnt_fft=g_cnt_noise=g_cnt_tone=g_cnt_mix=g_cnt_fit=g_cnt_enc=0;
      if(cap_on()){
        cap->W[blocks]=(int32_t)h->vb.W; cap->lW[blocks]=(int32_t)h->vb.lW; cap->nW[blocks]=(int32_t)h->vb.nW;
        cap->blocktype[blocks]=vbi->blocktype;
        cap->ampmax_in[blocks]=vbi->ampmax;
      }
#ifdef VB200_DROPIN
      if(g_seam1){ if(vb200_vorbis_analysis(&h->vb,NULL)){ g_cap = NULL; g_blk = -1; g_tl = NULL; return -1; } }
      else
#endif
      vorbis_analysis(&h->vb,NULL);
      if(cap_on()) cap->ampmax_out[blocks]=vbi->ampmax;
      vorbis_bitrate_addblock(&h->vb);
      while(vorbis_bitrate_flushpacket(&h->vd,&op)){
        total += op.bytes;
        keep_packet(h,&op);
        if(op.e_o_s) eos = 1;
      }
      blocks++;
    }
    if(todo<=0 && !eos) { /* blockout returned 0 after EOF without e_o_s: done */ eos = 1; }
  }
  if(cap) cap->nblocks = blocks < cap->maxblocks ? blocks : cap->maxblocks;
  g_cap = NULL; g_blk = -1; g_tl = NULL;
  if(bytes_out) *bytes_out = total;
  return blocks;
}

/* Decode the packets kept by ref_encode_capture through the reference API
 * (vorbis_synthesis + vorbis_synthesis_blockin + pcmout), capturing the
 * mdct_backward input/output per block and the finished PCM.
 * pcm_out = [ch][pcm_cap]; returns samples produced (per channel).          */
long ref_decode_capture(void *hv, ref_capture *cap, float *pcm_out, long pcm_cap, int32_t *Wseq){
  ref_handle *h = (ref_handle*)hv;
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  long produced = 0;
  int i, k, blocks = 0;
  vorbis_info_init(&vi); vorbis_comment_init(&vc);
  for(i=0;i<3;i++){
    ogg_packet hp = h->hdr[i];
    hp.b_o_s = (i==0);
    if(vorbis_synthesis_headerin(&vi,&vc,&hp)<0){ vorbis_comment_clear(&vc); vorbis_info_clear(&vi); return -1; }
  }
  vorbis_synthesis_init(&vd,&vi);
  vorbis_block_init(&vd,&vb);
  g_cap = cap; g_ch_total = vi.channels;
  for(k=0;k<h->npkt;k++){
    ogg_packet op; float **pcm; int got;
    memset(&op,0,sizeof(op));
    op.packet = h->pkt[k]; op.bytes = h->pktbytes[k]; op.packetno = k+3; op.granulepos = -1;
    g_blk = blocks; g_cnt_imdct = 0;
    if(vorbis_synthesis(&vb,&op)==0){
      if(Wseq && cap && blocks<cap->maxblocks) Wseq[blocks]=(int32_t)vb.W;
      vorbis_synthesis_blockin(&vd,&vb);
      blocks++;
    }
    while((got=vorbis_synthesis_pcmout(&vd,&pcm))>0){
      int take = got;
      if(produced+take>pcm_cap) take = (int)(pcm_cap-produced);
      for(i=0;i<vi.channels;i++)
        if(take>0) memcpy(pcm_out+(size_t)i*pcm_cap+produced,pcm[i],sizeof(float)*take);
      produced += take;
      vorbis_synthesis_read(&vd,got);
    }
  }
  if(cap) cap->nblocks = blocks < cap->maxblocks ? blocks : cap->maxblocks;
  g_cap = NULL; g_blk = -1;
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return produced;
}

/* Pure overlap-add check: feed IMDCT outputs through vorbis_synthesis_blockin.
 * Used to pin the oracle's overlap-add independent of the bitstream.
 * imdct = [nblk][ch][Nmax]; Wseq[nblk]; pcm_out [ch][pcm_cap]               */
long ref_blockin_sequence(void *hv, int nblk, const int32_t *Wseq, const float *imdct, int Nmax,
                          float *pcm_out, long pcm_cap){
  ref_handle *h = (ref_handle*)hv;
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  long produced = 0; int i,k;
  vorbis_info_init(&vi); vorbis_comment_init(&vc);
  if(!h->hdrcopy[0]){
    vorbis_analysis_headerout(&h->vd,&h->vc,&h->hdr[0],&h->hdr[1],&h->hdr[2]);
    for(i=0;i<3;i++){
      h->hdrcopy[i] = (unsigned char*)malloc(h->hdr[i].bytes);
      memcpy(h->hdrcopy[i],h->hdr[i].packet,h->hdr[i].bytes);
      h->hdr[i].packet = h->hdrcopy[i];
    }
  }
  for(i=0;i<3;i++){
    ogg_packet hp = h->hdr[i]; hp.b_o_s=(i==0);
    if(vorbis_synthesis_headerin(&vi,&vc,&hp)<0) return -1;
  }
  vorbis_synthesis_init(&vd,&vi);
  vorbis_block_init(&vd,&vb);
  {
    codec_setup_info *ci=(codec_setup_info*)vi.codec_setup;
    float **rows=(float**)malloc(sizeof(float*)*vi.channels);
    for(k=0;k<nblk;k++){
      float **pcm; int got;
      vb.W = Wseq[k];
      vb.pcmend = (int)ci->blocksizes[vb.W];
      vb.sequence = k;
      vb.granulepos = -1;
      vb.eofflag = 0;
      for(i=0;i<vi.channels;i++) rows[i]=(float*)imdct+((size_t)k*vi.channels+i)*Nmax;
      vb.pcm = rows;
      vorbis_synthesis_blockin(&vd,&vb);
      while((got=vorbis_synthesis_pcmout(&vd,&pcm))>0){
        int take=got;
        if(produced+take>pcm_cap) take=(int)(pcm_cap-produced);
        for(i=0;i<vi.channels;i++)
          if(take>0) memcpy(pcm_out+(size_t)i*pcm_cap+produced,pcm[i],sizeof(float)*take);
        produced+=take;
        vorbis_synthesis_read(&vd,got);
      }
    }
    vb.pcm=NULL;
    free(rows);
  }
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return produced;
}

/* ---- CPU baseline helper: the reference's Phase-A calls, in order, on a
 * batch of blocks (what mapping0_forward does at lib/mapping0.c:254-470 up to
 * floor1_fit, using only the reference's functions).  Used by bench.py's
 * cpu_baseline / --impl reference leg.                                      */
void ref_phaseA_batch(void *hv, int W, int nblocks, const float *pcm, const vb200_block_desc *desc,
                      float *mdct, float *logmdct_out, float *logmask_out, float *ampmax_out){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  int ch = h->vi.channels, N = (int)ci->blocksizes[W], n = N/2, blk, i, j;
  float *work = (float*)malloc(sizeof(float)*N*ch);
  float *noise = (float*)malloc(sizeof(float)*n);
  float *tone = (float*)malloc(sizeof(float)*n);
  float *lmax = (float*)malloc(sizeof(float)*ch);
  for(blk=0;blk<nblocks;blk++){
    vorbis_look_psy *psy_look = b->psy+desc[blk].blocktype+(W?2:0);
    float gmax = desc[blk].ampmax;
    for(i=0;i<ch;i++){
      float scale=4.f/N, scale_dB, *p = work+(size_t)i*N, *gm = mdct+((size_t)blk*ch+i)*n;
      memcpy(p,pcm+((size_t)blk*ch+i)*N,sizeof(float)*N);
      scale_dB=todB(&scale)+.345;
      _vorbis_apply_window(p,b->window,ci->blocksizes,desc[blk].lW,W,desc[blk].nW);
      mdct_forward((mdct_lookup*)b->transform[W][0],p,gm);
      drft_forward(&b->fft_look[W],p);
      p[0]=scale_dB+todB(p)+.345;
      lmax[i]=p[0];
      for(j=1;j<N-1;j+=2){
        float t=p[j]*p[j]+p[j+1]*p[j+1];
        t=p[(j+1)>>1]=scale_dB+.5f*todB(&t)+.345;
        if(t>lmax[i])lmax[i]=t;
      }
      if(lmax[i]>0.f)lmax[i]=0.f;
      if(lmax[i]>gmax)gmax=lmax[i];
    }
    for(i=0;i<ch;i++){
      float *p = work+(size_t)i*N, *gm = mdct+((size_t)blk*ch+i)*n;
      float *logmdct = p+n, *logmask = p;
      for(j=0;j<n;j++) logmdct[j]=todB(gm+j)+.345;
      _vp_noisemask(psy_look,logmdct,noise);
      _vp_tonemask(psy_look,p,tone,gmax,lmax[i]);
      _vp_offset_and_mix(psy_look,noise,tone,1,logmask,gm,logmdct);
      memcpy(logmdct_out+((size_t)blk*ch+i)*n,logmdct,sizeof(float)*n);
      memcpy(logmask_out+((size_t)blk*ch+i)*n,logmask,sizeof(float)*n);
    }
    ampmax_out[blk]=gmax;
  }
  free(work); free(noise); free(tone); free(lmax);
}

/* ---- CPU baseline helper: the whole per-block DSP chain of mapping0_forward for un-managed
 * bitrate (lib/mapping0.c:230-646): the Phase-A calls above, then floor1_fit (:500),
 * floor1_encode (:617; its bits go to a scratch buffer) and _vp_couple_quantize_normalize
 * (:631-646) for blob PACKETBLOBS/2, using only the reference's functions.  This is the same work
 * vb200_encode_dsp does; used by bench.py's cpu_baseline / --impl reference leg.               */
#include "misc.h"
extern int *floor1_fit(vorbis_block *vb,vorbis_look_floor1 *look,const float *logmdct,const float *logmask);
extern int floor1_encode(oggpack_buffer *opb,vorbis_block *vb,vorbis_look_floor1 *look,int *post,int *ilogmask);

void ref_encode_dsp_batch(void *hv, int W, int nblocks, const float *pcm, const vb200_block_desc *desc,
                          int32_t *posts_out, int32_t *nonzero_out, int32_t *iwork_out, float *ampmax_out){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_info_mapping0 *info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
  int ch = h->vi.channels, N = (int)ci->blocksizes[W], n = N/2, blk, i, k;
  const int blob = PACKETBLOBS/2;
  float *mdct = (float*)malloc(sizeof(float)*n*ch);
  float *logmdct = (float*)malloc(sizeof(float)*n*ch);
  float *logmask = (float*)malloc(sizeof(float)*n*ch);
  float **m = (float**)malloc(sizeof(*m)*ch);
  int   **iw = (int**)malloc(sizeof(*iw)*ch);
  int    *nz = (int*)malloc(sizeof(int)*ch);
  oggpack_buffer opb;
  oggpack_writeinit(&opb);
  h->vb.W = W;
  h->vb.pcmend = N;               /* floor1_encode fills ilogmask up to vb->pcmend/2 (lib/floor1.c:941) */
  for(blk=0;blk<nblocks;blk++){
    vorbis_look_psy *p = b->psy+desc[blk].blocktype+(W?2:0);
    ref_phaseA_batch(hv,W,1,pcm+(size_t)blk*ch*N,desc+blk,mdct,logmdct,logmask,ampmax_out+blk);
    oggpack_reset(&opb);
    for(i=0;i<ch;i++){
      int submap = info->chmuxlist[i];
      vorbis_look_floor1 *look = (vorbis_look_floor1*)b->flr[info->floorsubmap[submap]];
      int32_t *po = posts_out+((size_t)blk*ch+i)*65;
      int *post = floor1_fit(&h->vb,look,logmdct+(size_t)i*n,logmask+(size_t)i*n);
      m[i] = mdct+(size_t)i*n;
      iw[i] = (int*)(iwork_out+((size_t)blk*ch+i)*n);
      nz[i] = floor1_encode(&opb,&h->vb,look,post,iw[i]);
      for(k=0;k<65;k++) po[k]=0;
      if(post) for(k=0;k<look->posts;k++) po[k]=post[k];
    }
    _vp_couple_quantize_normalize(blob,&ci->psy_g_param,p,info,m,iw,nz,
                                  ci->psy_g_param.sliding_lowpass[W][blob],ch);
    for(i=0;i<ch;i++) nonzero_out[(size_t)blk*ch+i]=nz[i];
    _vorbis_block_ripcord(&h->vb);
  }
  oggpack_writeclear(&opb);
  free(mdct); free(logmdct); free(logmask); free(m); free(iw); free(nz);
}


/* ---- bitrate-managed mode: what mapping0_forward does when vorbis_bitrate_managed(vb)
 * (lib/mapping0.c:500-573 and the per-blob loop :596-646), with the reference's own functions in the
 * reference's order: middle fit, then - where it exists - mask 2 + fit, mask 0 + fit, the twelve
 * floor1_interpolate_fit curves; per blob k floor1_encode (its bits go to a scratch buffer) and
 * _vp_couple_quantize_normalize(k).  Outputs blob-major: posts [15][rows][65] (0 where NULL),
 * nonzero [15][rows], iwork [15][rows][n].  Pins oracle/pyoracle.py: encode_dsp_managed.          */
extern int *floor1_interpolate_fit(vorbis_block *vb,vorbis_look_floor1 *look,int *A,int *B,int del);
void ref_encode_dsp_managed_batch(void *hv, int W, int nblocks, const float *pcm, const vb200_block_desc *desc,
                                  int32_t *posts_out, int32_t *nonzero_out, int32_t *iwork_out, float *ampmax_out){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_info_mapping0 *info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
  int ch = h->vi.channels, N = (int)ci->blocksizes[W], n = N/2, blk, i, j, k;
  size_t rows = (size_t)nblocks*ch;
  float *work = (float*)malloc(sizeof(float)*N*ch);
  float *gmdct = (float*)malloc(sizeof(float)*n*ch);
  float *noise = (float*)malloc(sizeof(float)*n);
  float *tone = (float*)malloc(sizeof(float)*n);
  float *lmax = (float*)malloc(sizeof(float)*ch);
  float **m = (float**)malloc(sizeof(*m)*ch);
  int   **iw = (int**)malloc(sizeof(*iw)*ch);
  int    *nz = (int*)malloc(sizeof(int)*ch);
  int ***floor_posts = (int***)malloc(sizeof(*floor_posts)*ch);
  oggpack_buffer opb;
  oggpack_writeinit(&opb);
  for(i=0;i<ch;i++) floor_posts[i] = (int**)malloc(sizeof(int*)*PACKETBLOBS);
  h->vb.W = W;
  h->vb.pcmend = N;
  for(blk=0;blk<nblocks;blk++){
    vorbis_look_psy *psy_look = b->psy+desc[blk].blocktype+(W?2:0);
    float gmax = desc[blk].ampmax;
    for(i=0;i<ch;i++){
      float scale=4.f/N, scale_dB, *p = work+(size_t)i*N, *gm = gmdct+(size_t)i*n;
      memcpy(p,pcm+((size_t)blk*ch+i)*N,sizeof(float)*N);
      scale_dB=todB(&scale)+.345;
      _vorbis_apply_window(p,b->window,ci->blocksizes,desc[blk].lW,W,desc[blk].nW);
      mdct_forward((mdct_lookup*)b->transform[W][0],p,gm);
      drft_forward(&b->fft_look[W],p);
      p[0]=scale_dB+todB(p)+.345;
      lmax[i]=p[0];
      for(j=1;j<N-1;j+=2){
        float t=p[j]*p[j]+p[j+1]*p[j+1];
        t=p[(j+1)>>1]=scale_dB+.5f*todB(&t)+.345;
        if(t>lmax[i])lmax[i]=t;
      }
      if(lmax[i]>0.f)lmax[i]=0.f;
      if(lmax[i]>gmax)gmax=lmax[i];
    }
    for(i=0;i<ch;i++){
      int submap = info->chmuxlist[i];
      vorbis_look_floor1 *look = (vorbis_look_floor1*)b->flr[info->floorsubmap[submap]];
      float *p = work+(size_t)i*N, *gm = gmdct+(size_t)i*n;
      float *logmdct = p+n, *logmask = p;
      for(k=0;k<PACKETBLOBS;k++) floor_posts[i][k]=NULL;
      for(j=0;j<n;j++) logmdct[j]=todB(gm+j)+.345;
      _vp_noisemask(psy_look,logmdct,noise);
      _vp_tonemask(psy_look,p,tone,gmax,lmax[i]);
      _vp_offset_and_mix(psy_look,noise,tone,1,logmask,gm,logmdct);
      floor_posts[i][PACKETBLOBS/2]=floor1_fit(&h->vb,look,logmdct,logmask);
      if(floor_posts[i][PACKETBLOBS/2]){
        _vp_offset_and_mix(psy_look,noise,tone,2,logmask,gm,logmdct);
        floor_posts[i][PACKETBLOBS-1]=floor1_fit(&h->vb,look,logmdct,logmask);
        _vp_offset_and_mix(psy_look,noise,tone,0,logmask,gm,logmdct);
        floor_posts[i][0]=floor1_fit(&h->vb,look,logmdct,logmask);
        for(k=1;k<PACKETBLOBS/2;k++)
          floor_posts[i][k]=floor1_interpolate_fit(&h->vb,look,floor_posts[i][0],floor_posts[i][PACKETBLOBS/2],
                                                   k*65536/(PACKETBLOBS/2));
        for(k=PACKETBLOBS/2+1;k<PACKETBLOBS-1;k++)
          floor_posts[i][k]=floor1_interpolate_fit(&h->vb,look,floor_posts[i][PACKETBLOBS/2],floor_posts[i][PACKETBLOBS-1],
                                                   (k-PACKETBLOBS/2)*65536/(PACKETBLOBS/2));
      }
    }
    ampmax_out[blk]=gmax;
    for(k=0;k<PACKETBLOBS;k++){
      oggpack_reset(&opb);
      for(i=0;i<ch;i++){
        int submap = info->chmuxlist[i];
        vorbis_look_floor1 *look = (vorbis_look_floor1*)b->flr[info->floorsubmap[submap]];
        size_t row = (size_t)blk*ch+i;
        int32_t *po = posts_out+((size_t)k*rows+row)*65;
        m[i] = gmdct+(size_t)i*n;
        iw[i] = (int*)(iwork_out+((size_t)k*rows+row)*n);
        nz[i] = floor1_encode(&opb,&h->vb,look,floor_posts[i][k],iw[i]);
        for(j=0;j<65;j++) po[j]=0;
        if(floor_posts[i][k]) for(j=0;j<look->posts;j++) po[j]=floor_posts[i][k][j];
      }
      _vp_couple_quantize_normalize(k,&ci->psy_g_param,psy_look,info,m,iw,nz,
                                    ci->psy_g_param.sliding_lowpass[W][k],ch);
      for(i=0;i<ch;i++) nonzero_out[(size_t)k*rows+(size_t)blk*ch+i]=nz[i];
    }
    _vorbis_block_ripcord(&h->vb);
  }
  oggpack_writeclear(&opb);
  for(i=0;i<ch;i++) free(floor_posts[i]);
  free(floor_posts); free(work); free(gmdct); free(noise); free(tone); free(lmax); free(m); free(iw); free(nz);
}


/* ---- envelope detector: the reference's own _ve_envelope_search (lib/envelope.c:216) on a fresh
 * vorbis_dsp_state holding `nsamples` samples per channel (planar pcm [ch][nsamples]); no blockout
 * happens, so the one call analyses every step the buffer allows.  Copies out ve->mark[0..steps+VE_POST),
 * the filter states and stretch afterwards, and the stream buffer itself ([ch][bs1/2+nsamples]);
 * returns the number of steps analysed (`last`).                                                 */
#include "envelope.h"
long ref_envelope_marks(void *hv, const float *pcm, long nsamples, int32_t *marks, long markcap,
                        int32_t *state_out, float *stream_out){
  ref_handle *h = (ref_handle*)hv;
  vorbis_dsp_state vd;
  private_state *b;
  envelope_lookup *ve;
  float **buf;
  long steps, k;
  int c, ch = h->vi.channels;
  if(vorbis_analysis_init(&vd,&h->vi)) return -1;
  buf = vorbis_analysis_buffer(&vd,(int)nsamples);
  for(c=0;c<ch;c++) memcpy(buf[c],pcm+(size_t)c*nsamples,sizeof(float)*nsamples);
  vorbis_analysis_wrote(&vd,(int)nsamples);
  _ve_envelope_search(&vd);
  b = (private_state*)vd.backend_state;
  ve = b->ve;
  /* the stream buffer the detector saw: blocksizes[1]/2 samples of preamble (zeros, or the reverse
   * LPC extrapolation of _preextrapolate_helper, lib/block.c:415-456) followed by the input */
  if(stream_out)
    for(c=0;c<ch;c++) memcpy(stream_out+(size_t)c*vd.pcm_current,vd.pcm[c],sizeof(float)*vd.pcm_current);
  steps = vd.pcm_current/ve->searchstep-VE_WIN;
  if(steps<0) steps=0;
  for(k=0;k<markcap;k++) marks[k] = (k<steps+VE_POST && k<ve->storage) ? ve->mark[k] : 0;
  if(state_out){
    state_out[0] = ve->stretch;
    memcpy(state_out+1, ve->filter, sizeof(envelope_filter_state)*VE_BANDS*ch);
  }
  vorbis_dsp_clear(&vd);
  return steps;
}


/* ---- decode floor: the reference's own floor1_inverse2 (static, lib/floor1.c:1041) through its
 * export bundle, on a batch of rows laid out [block][channel]: row r uses the floor of channel
 * r % channels of mode W.  fit [rows][65] = fit_value[] as floor1_inverse1 would return it,
 * present[r] == 0 <=> memo NULL.                                                              */
#include "backends.h"
extern const vorbis_func_floor floor1_exportbundle;
void ref_floor1_inverse2(void *hv, int W, int nrows, const int32_t *fit, const int32_t *present, float *data){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_info_mapping0 *info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
  int ch = h->vi.channels, n = (int)ci->blocksizes[W]/2, r, k;
  int memo[65];
  h->vb.W = W;
  for(r=0;r<nrows;r++){
    int c = r % ch;
    vorbis_look_floor *look = b->flr[info->floorsubmap[info->chmuxlist[c]]];
    for(k=0;k<65;k++) memo[k] = fit[(size_t)r*65+k];
    floor1_exportbundle.inverse2(&h->vb, look, present[r] ? (void*)memo : NULL, data+(size_t)r*n);
  }
}


/* ---- residue classification: the reference's own res{0,1,2}_class through _residue_P[] exactly as
 * mapping0_forward calls it per submap (lib/mapping0.c:660-672), on a batch laid out [block][ch][n].
 * classes [block][ch][stride], written in the layout documented for vb200_residue_classify.      */
void ref_residue_classify(void *hv, int W, int nblocks, const int32_t *iwork, const int32_t *nonzero,
                          int32_t *classes, int stride){
  ref_handle *h = (ref_handle*)hv;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_info_mapping0 *info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
  int ch = h->vi.channels, n = (int)ci->blocksizes[W]/2, blk, i, j, k;
  int **bundle = (int**)malloc(sizeof(*bundle)*ch);
  int *zb = (int*)malloc(sizeof(int)*ch), *chan = (int*)malloc(sizeof(int)*ch);
  int *copy = (int*)malloc(sizeof(int)*(size_t)ch*n);
  h->vb.W = W; h->vb.pcmend = 2*n;
  memset(classes,0,sizeof(int32_t)*(size_t)nblocks*ch*stride);
  for(blk=0;blk<nblocks;blk++){
    memcpy(copy,iwork+(size_t)blk*ch*n,sizeof(int)*(size_t)ch*n);
    for(i=0;i<info->submaps;i++){
      int cib=0, resnum=info->residuesubmap[i], type=ci->residue_type[resnum];
      vorbis_info_residue0 *ri=(vorbis_info_residue0*)ci->residue_param[resnum];
      int partvals=(int)((ri->end-ri->begin)/ri->grouping);
      long **pw;
      for(j=0;j<ch;j++) if(info->chmuxlist[j]==i){
        zb[cib]=nonzero[(size_t)blk*ch+j]?1:0; chan[cib]=j; bundle[cib++]=copy+(size_t)j*n;
      }
      pw=_residue_P[type]->class(&h->vb,b->residue[resnum],bundle,zb,cib);
      if(pw){
        if(type==2){
          int32_t *dst=classes+((size_t)blk*ch+chan[0])*stride;
          for(k=0;k<partvals;k++) dst[k]=(int32_t)pw[0][k];
        }else{
          int u=0;
          for(j=0;j<cib;j++) if(zb[j]){
            int32_t *dst=classes+((size_t)blk*ch+chan[j])*stride;
            for(k=0;k<partvals;k++) dst[k]=(int32_t)pw[u][k];
            u++;
          }
        }
      }
    }
    _vorbis_block_ripcord(&h->vb);
  }
  free(bundle); free(zb); free(chan); free(copy);
}



/* packet summary: (count, bytes, FNV-1a over all packet bytes in order) of one encoder run */
typedef struct { uint64_t *hash; long *bytes, *count; int *eos; } ms_sum;
static void ms_sink(void *user, int stream, ogg_packet *op){
  ms_sum *s = (ms_sum*)user;
  long k;
  uint64_t h = s->hash[stream];
  for(k = 0; k < op->bytes; k++){ h ^= op->packet[k]; h *= 1099511628211ULL; }
  h ^= (uint64_t)op->bytes; h *= 1099511628211ULL;
  s->hash[stream] = h; s->bytes[stream] += op->bytes; s->count[stream]++;
  if(op->e_o_s) s->eos[stream] = 1;
}
/* the same summary for ONE stock reference encoder (this library's vorbis_analysis: the unmodified CPU path in libvorbis_ref.so) */
long ref_stock_encode_summary(int ch, long rate, float quality, const float *pcm, long nsamples,
                              uint64_t *hash, long *bytes, long *count){
  ref_handle *h = (ref_handle*)ref_open(ch, rate, quality);
  ms_sum sum; int eos = 0, i; long pos = 0, blocks = 0;
  ogg_packet op;
  const long chunk = g_chunk > 0 ? g_chunk : 1024;
  if(!h) return -1;
  *hash = 1469598103934665603ULL; *bytes = 0; *count = 0;
  sum.hash = hash; sum.bytes = bytes; sum.count = count; sum.eos = &eos;
  while(!eos){
    long todo = nsamples - pos < chunk ? nsamples - pos : chunk;
    if(todo > 0){
      float **buf = vorbis_analysis_buffer(&h->vd, (int)todo);
      for(i = 0; i < ch; i++) memcpy(buf[i], pcm + (size_t)i*nsamples + pos, sizeof(float)*todo);
      vorbis_analysis_wrote(&h->vd, (int)todo);
      pos += todo;
    }else vorbis_analysis_wrote(&h->vd, 0);
    while(vorbis_analysis_blockout(&h->vd, &h->vb) == 1){
      vorbis_analysis(&h->vb, NULL);
      vorbis_bitrate_addblock(&h->vb);
      while(vorbis_bitrate_flushpacket(&h->vd, &op)) ms_sink(&sum, 0, &op);
      blocks++;
    }
    if(todo <= 0) eos = 1;
  }
  ref_close(h);
  return blocks;
}

#ifdef VB200_DROPIN
/* ---- multi-stream driver test hook (vorbis_b200/host/vb200_mapping0.c): N encoders of one configuration fed in
 * lockstep with 1024-sample writes; every stream's packets are summarised as (count, bytes, FNV-1a hash of all
 * packet bytes in order) so that they can be compared with N runs of the stock reference encoder.             */
typedef struct vb200ms vb200ms;
typedef void (*vb200ms_sink)(void *user, int stream, ogg_packet *op);
vb200ms *vb200ms_open(int nstreams, int channels, long rate, float quality, int device);
void vb200ms_close(vb200ms *m);
vorbis_dsp_state *vb200ms_state(vb200ms *m, int stream);
int vb200ms_round(vb200ms *m, vb200ms_sink sink, void *user);

/* pcm [nstreams][ch][nsamples]; returns total blocks, or <0 */
long ref_ms_encode(int nstreams, int ch, long rate, float quality, int device, const float *pcm, long nsamples,
                   uint64_t *hash, long *bytes, long *count){
  vb200ms *m = vb200ms_open(nstreams, ch, rate, quality, device);
  ms_sum sum;
  long pos = 0, blocks = 0;
  int i, c, r, alldone = 0;
  const long chunk = g_chunk > 0 ? g_chunk : 1024;
  int *eos = (int*)calloc(nstreams, sizeof(int));
  if(!m){ free(eos); return -1; }
  for(i = 0; i < nstreams; i++){ hash[i] = 1469598103934665603ULL; bytes[i] = 0; count[i] = 0; }
  sum.hash = hash; sum.bytes = bytes; sum.count = count; sum.eos = eos;
  while(!alldone){
    long todo = nsamples - pos < chunk ? nsamples - pos : chunk;
    /* the application's side: N independent streams are fed by all host threads (the first and the last write of
     * a stream run the reference's LPC pre-/post-extrapolation, ~1 ms each) */
#pragma omp parallel for private(c) schedule(dynamic, 8) if(nstreams > 8)
    for(i = 0; i < nstreams; i++){
      vorbis_dsp_state *vd = vb200ms_state(m, i);
      if(todo > 0){
        float **buf = vorbis_analysis_buffer(vd, (int)todo);
        for(c = 0; c < ch; c++) memcpy(buf[c], pcm + ((size_t)i*ch + c)*nsamples + pos, sizeof(float)*todo);
        vorbis_analysis_wrote(vd, (int)todo);
      }else vorbis_analysis_wrote(vd, 0);
    }
    pos += todo > 0 ? todo : 0;
    while((r = vb200ms_round(m, ms_sink, &sum)) > 0) blocks += r;
    if(r < 0){ blocks = r; break; }
    if(todo <= 0) alldone = 1;
  }
  vb200ms_close(m);
  free(eos);
  return blocks;
}

#endif
