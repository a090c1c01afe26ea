/* vb200_mapping0.c — the block-level binding (SURVEY §8b seam 1): a `vorbis_func_mapping` whose
 * forward() hands a whole block to the device in ONE call, and a multi-stream driver that hands the
 * ready blocks of MANY vorbis_dsp_states to the device in one call per block size.
 *
 *   reference                                            this file
 *   mapping0_exportbundle (lib/mapping0.c:802-808)   ->  vb200_mapping0_exportbundle: pack / unpack / free_info /
 *                                                        inverse are the reference's own, forward is below
 *   mapping0_forward (lib/mapping0.c:230-696)        ->  vb200_mapping0_forward: ONE vb200_encode_dsp call for
 *                                                        everything between vb->pcm and the entropy coder
 *                                                        (window, MDCT, FFT, masks, floor fit + render, couple /
 *                                                        quantise / normalise), then on the host exactly what the
 *                                                        reference does with bits: mode header (:603-610), the
 *                                                        reference's own floor1_encode (lib/floor1.c:753) for the
 *                                                        floor bits and _residue_P[]->class / ->forward
 *                                                        (lib/mapping0.c:660-683) for the residue
 *   a loop of vorbis_analysis over N encoders        ->  vb200ms_*: blockout for every stream, the blocks that are
 *                                                        ready go to the device together, packets come back per stream;
 *                                                        the packets are entropy coded on the device too (one
 *                                                        vb200_encode_packets[_managed] call per block size and round)
 *
 * floor1_encode is fed the device's posts re-expanded to the fit scale: its quantise step maps them back to
 * the same integers and its predict/flag pass is idempotent on them, so it writes exactly the bits it would
 * have written for the fit (its own render into a scratch curve is redundant host work of ~n integer ops per
 * channel; the curve the residue was built from is the device's).  No reference source is restated here.
 *
 * Bitrate-managed encoders (vorbis_encode_init) take the same path: one vb200_encode_dsp_managed call per batch
 * returns all PACKETBLOBS curves of every block and the host writes all PACKETBLOBS packets of each (the seam is
 * the batch of one block; vb200ms_open_managed opens a managed multi-stream driver, which codes all PACKETBLOBS
 * packets on the device where the context takes the setup).  A CUDA failure surfaces as OV_EFAULT from vorbis_analysis and latches in
 * the binding (vb200shim_error).  Compiled like any libvorbis-internal backend against lib/codec_internal.h
 * (oracle/Makefile target `dropin`); INTEGRATION.md shows the registry line a maintainer changes.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"
#include "codec_internal.h"
#include "registry.h"
#include "bitrate.h"

#include "vorbis_b200.h"
#include "vb200_vorbis_setup.h"

#ifdef _OPENMP
#include <omp.h>
#endif
#include <time.h>

/* optional wall-clock breakdown of the multi-stream driver (VB200MS_PROFILE=1): seconds per phase, printed at close */
static double g_prof[8];
static int g_prof_on = -1;
static double now_s(void){ struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9*t.tv_nsec; }
#define PROF_T0() double prof_t0_ = (g_prof_on > 0) ? now_s() : 0.0
#define PROF_ADD(k) do { if(g_prof_on > 0){ const double t_ = now_s(); g_prof[k] += t_ - prof_t0_; prof_t0_ = t_; } } while(0)

/* from vb200_ref_shim.c */
typedef struct vb200_binding vb200_binding;
int vb200shim_envelope_prepare(vorbis_dsp_state *v, int *first_out);
void vb200shim_envelope_state_get(vorbis_dsp_state *v, int32_t *state);
void vb200shim_envelope_commit(vorbis_dsp_state *v, int first, int nsteps, const int32_t *state, const uint8_t *ret);
int vb200shim_attach(vorbis_dsp_state *vd, int device);
void vb200shim_detach(void);
int vb200shim_select(vorbis_dsp_state *vd);
vb200_binding *vb200shim_binding(vorbis_dsp_state *vd);
vb200_ctx *vb200shim_ctx(vb200_binding *b);
void vb200shim_set_error(vb200_binding *b, int rc);

extern const vorbis_func_mapping mapping0_exportbundle;      /* the reference's own bundle (lib/mapping0.c:802) */
extern int floor1_encode(oggpack_buffer *opb, vorbis_block *vb, vorbis_look_floor1 *look, int *post, int *ilogmask);

/* ---- host half of one block: header bits, floor bits, residue bits -----------------------------------------
 * posts [ch][VB200_FLOOR1_STRIDE], nonzero [ch] (after coupling), iwork [ch][n]: what vb200_encode_dsp returned */
static int pack_block_blob(vorbis_block *vb, int k, const int32_t *posts, const int32_t *nonzero_dev, const int32_t *iwork_dev){
  vorbis_dsp_state *vd = vb->vd;
  vorbis_info *vi = vd->vi;
  codec_setup_info *ci = (codec_setup_info*)vi->codec_setup;
  private_state *b = (private_state*)vd->backend_state;
  vorbis_block_internal *vbi = (vorbis_block_internal*)vb->internal;
  const int ch = vi->channels, n = vb->pcmend/2;
  const int modenumber = (int)vb->W;
  vorbis_info_mapping0 *info = (vorbis_info_mapping0*)ci->map_param[modenumber];
  oggpack_buffer *opb = vbi->packetblob[k];
  int **iwork = (int**)_vorbis_block_alloc(vb, ch*sizeof(*iwork));
  int **couple_bundle = (int**)_vorbis_block_alloc(vb, ch*sizeof(*couple_bundle));
  int *zerobundle = (int*)_vorbis_block_alloc(vb, ch*sizeof(*zerobundle));
  int *scratch = (int*)_vorbis_block_alloc(vb, n*sizeof(*scratch));
  int i, j;
  vb->mode = modenumber;
  for(i = 0; i < ch; i++){                                     /* the residue backend wants int** rows */
    iwork[i] = (int*)_vorbis_block_alloc(vb, n*sizeof(**iwork));
    memcpy(iwork[i], iwork_dev + (size_t)i*n, n*sizeof(int));
  }
  oggpack_write(opb, 0, 1);                                    /* packet type: audio */
  oggpack_write(opb, modenumber, b->modebits);
  if(vb->W){
    oggpack_write(opb, vb->lW, 1);
    oggpack_write(opb, vb->nW, 1);
  }
  for(i = 0; i < ch; i++){
    const int submap = info->chmuxlist[i];
    vorbis_look_floor1 *look = (vorbis_look_floor1*)b->flr[info->floorsubmap[submap]];
    const int32_t *p = posts + (size_t)i*VB200_FLOOR1_STRIDE;
    const int P = look->posts, mult = look->vi->mult;
    int any = 0, fit[VIF_POSIT+2];
    if(ci->floor_type[info->floorsubmap[submap]] != 1) return -1;
    for(j = 0; j < P; j++) any |= p[j];
    if(!any){                                                  /* floor1_fit returned NULL: an all-zero row (vorbis_b200.h) */
      floor1_encode(opb, vb, look, NULL, scratch);
      continue;
    }
    for(j = 0; j < P; j++){                                    /* back to the fit scale: the quantiser undoes it exactly */
      const int v = p[j] & 0x7fff;
      const int e = mult == 1 ? v << 2 : mult == 2 ? v << 3 : mult == 3 ? v*12 : v << 4;
      fit[j] = e | (p[j] & 0x8000);
    }
    floor1_encode(opb, vb, look, fit, scratch);
  }
  for(i = 0; i < info->submaps; i++){                          /* classify and encode by submap */
    int ch_in_bundle = 0;
    long **classifications;
    const int resnum = info->residuesubmap[i];
    for(j = 0; j < ch; j++)
      if(info->chmuxlist[j] == i){
        zerobundle[ch_in_bundle] = nonzero_dev[j] ? 1 : 0;
        couple_bundle[ch_in_bundle++] = iwork[j];
      }
    classifications = _residue_P[ci->residue_type[resnum]]->class(vb, b->residue[resnum], couple_bundle, zerobundle, ch_in_bundle);
    ch_in_bundle = 0;
    for(j = 0; j < ch; j++)
      if(info->chmuxlist[j] == i) couple_bundle[ch_in_bundle++] = iwork[j];
    _residue_P[ci->residue_type[resnum]]->forward(opb, vb, b->residue[resnum], couple_bundle, zerobundle, ch_in_bundle, classifications, i);
  }
  return 0;
}

static int pack_block(vorbis_block *vb, const int32_t *posts, const int32_t *nonzero_dev, int32_t *iwork_dev){
  return pack_block_blob(vb, PACKETBLOBS/2, posts, nonzero_dev, iwork_dev);    /* un-managed: the middle curve only */
}

/* ---- device half for a set of blocks of ONE size ------------------------------------------------------------ */
typedef struct {
  float *pcm; vb200_block_desc *desc; int32_t *posts, *nonzero, *iwork; float *ampmax;
  size_t cap_blocks; int ch, N, curves;
  uint8_t *pkt; int64_t *pkt_off; int32_t *pkt_bits; size_t pkt_cap;   /* the device coder's packed packets */
} ms_batch;

/* curves: 1 (un-managed) or PACKETBLOBS (bitrate-managed: posts / nonzero / iwork hold every curve, blob-major) */
static int batch_reserve(ms_batch *B, size_t nb, int ch, int N, int curves){
  if(B->cap_blocks >= nb && B->ch == ch && B->N == N && B->curves == curves) return 0;
  free(B->pcm); free(B->desc); free(B->posts); free(B->nonzero); free(B->iwork); free(B->ampmax);
  free(B->pkt); free(B->pkt_off); free(B->pkt_bits);
  memset(B, 0, sizeof(*B));
  B->pcm = (float*)malloc(sizeof(float)*nb*ch*N);
  B->desc = (vb200_block_desc*)malloc(sizeof(vb200_block_desc)*nb);
  B->posts = (int32_t*)malloc(sizeof(int32_t)*curves*nb*ch*VB200_FLOOR1_STRIDE);
  B->nonzero = (int32_t*)malloc(sizeof(int32_t)*curves*nb*ch);
  B->iwork = (int32_t*)malloc(sizeof(int32_t)*curves*nb*ch*(N/2));
  B->ampmax = (float*)malloc(sizeof(float)*nb);
  if(!B->pcm || !B->desc || !B->posts || !B->nonzero || !B->iwork || !B->ampmax) return OV_EFAULT;
  B->cap_blocks = nb; B->ch = ch; B->N = N; B->curves = curves;
  return 0;
}

/* blocks[0..nb) all have vb->W == W and belong to states of ONE binding, all bitrate-managed or all not.  The
 * staging copies and the host half (bits) of different blocks are independent - different vorbis_dsp_states share
 * nothing that is written - so both loops run on all host threads; `after` (optional) is called by the thread that
 * packed block i.  Bitrate-managed (lib/mapping0.c:507-573, 596-687): ONE vb200_encode_dsp_managed call gives the
 * posts, nonzero flags and quantised residue of all PACKETBLOBS curves of every block; the host then writes
 * packetblob[k] for every k exactly as it writes the single packet of un-managed mode, and lib/bitrate.c picks among
 * them afterwards. */
typedef void (*batch_after)(void *user, int i);
static int forward_batch(vb200_binding *bind, ms_batch *B, vorbis_block **blocks, int nb, int W, batch_after after, void *user){
  vorbis_info *vi = blocks[0]->vd->vi;
  const int ch = vi->channels, N = (int)blocks[0]->pcmend, n = N/2;
  const int managed = vorbis_bitrate_managed(blocks[0]);
  vb200_encode_io io;
  int i, c, rc;
  int err = 0;
  PROF_T0();
  if((rc = batch_reserve(B, (size_t)nb, ch, N, managed ? PACKETBLOBS : 1))) return rc;
#pragma omp parallel for private(c) schedule(static) if(nb > 8)
  for(i = 0; i < nb; i++){
    vorbis_block_internal *vbi = (vorbis_block_internal*)blocks[i]->internal;
    for(c = 0; c < ch; c++) memcpy(B->pcm + ((size_t)i*ch + c)*N, blocks[i]->pcm[c], sizeof(float)*N);
    B->desc[i].lW = (int32_t)blocks[i]->lW; B->desc[i].nW = (int32_t)blocks[i]->nW;
    B->desc[i].blocktype = vbi->blocktype; B->desc[i].ampmax = vbi->ampmax;
  }
  memset(&io, 0, sizeof(io));
  io.pcm = B->pcm; io.pcm_fmt = VB200_PCM_F32_BLOCKS; io.desc = B->desc; io.independent = 1;
  io.posts = B->posts; io.nonzero = B->nonzero; io.iwork = B->iwork; io.ampmax_out = B->ampmax;
  PROF_ADD(2);
  rc = managed ? vb200_encode_dsp_managed(vb200shim_ctx(bind), W, nb, 1, &io)
               : vb200_encode_dsp(vb200shim_ctx(bind), W, nb, 1, PACKETBLOBS/2, &io);   /* one H2D, the kernels, one D2H */
  PROF_ADD(3);
  if(rc){
    vb200shim_set_error(bind, rc);
    fprintf(stderr, "vb200 mapping0: vb200_encode_dsp%s failed (%d): %s\n", managed ? "_managed" : "", rc, vb200_last_error());
    return OV_EFAULT;
  }
#pragma omp parallel for schedule(dynamic, 4) if(nb > 8)
  for(i = 0; i < nb; i++){
    vorbis_block_internal *vbi = (vorbis_block_internal*)blocks[i]->internal;
    int r = 0, k;
    vbi->ampmax = B->ampmax[i];                                /* lib/mapping0.c:576 */
    if(!managed)
      r = pack_block(blocks[i], B->posts + (size_t)i*ch*VB200_FLOOR1_STRIDE, B->nonzero + (size_t)i*ch,
                     B->iwork + (size_t)i*ch*n);
    for(k = 0; managed && k < PACKETBLOBS && !r; k++){          /* curve k of block i: row (k*nb + i)*ch */
      const size_t r0 = ((size_t)k*nb + i)*ch;
      r = pack_block_blob(blocks[i], k, B->posts + r0*VB200_FLOOR1_STRIDE, B->nonzero + r0, B->iwork + r0*n);
    }
    if(r){
#pragma omp atomic write
      err = r;
    }else if(after) after(user, i);
  }
  PROF_ADD(4);
  return err;
}

/* ---- the device entropy coder ------------------------------------------------------------------------------------ */
/* The struct vb200_encode_entropy_setup of an encoder after vorbis_analysis_init: every book of ci->fullbooks (its
 * lengthlist, codelist and integer lattice), the floor-1 and residue fields of both modes' submaps with the stage
 * books laid out as res0_look lays out partbooks (lib/res0.c:274-292), modebits.  The codeword arrays point into the
 * encoder's own books, so the setup is valid as long as that vorbis_info; es->books is malloc'd (free() it).
 * Returns 0, OV_EIMPL for a mode layout the device coder does not take, or OV_EFAULT. */
int vb200ms_entropy_setup_build(vorbis_dsp_state *vd, struct vb200_encode_entropy_setup *es){
  codec_setup_info *ci = (codec_setup_info*)vd->vi->codec_setup;
  private_state *b = (private_state*)vd->backend_state;
  vb200_enc_codebook *books;
  int i;
  memset(es, 0, sizeof(*es));
  if(!ci->fullbooks) return OV_EIMPL;
  books = (vb200_enc_codebook*)calloc(ci->books > 0 ? ci->books : 1, sizeof(*books));
  if(!books) return OV_EFAULT;
  for(i = 0; i < ci->books; i++){
    const codebook *cb = ci->fullbooks + i;
    books[i].dim = (int32_t)cb->dim; books[i].entries = (int32_t)cb->entries;
    books[i].length = (const uint8_t*)cb->c->lengthlist; books[i].codeword = cb->codelist;
    books[i].minval = cb->minval; books[i].delta = cb->delta; books[i].quantvals = cb->quantvals;
  }
  es->nbooks = ci->books; es->books = books; es->modebits = b->modebits;
  if(vb200vs_entropy(ci, &books[0].dim, sizeof(*books), es->floor, es->residue)){
    free(books);
    es->books = NULL;
    return OV_EIMPL;
  }
  return 0;
}

/* bits bits of a device packet (bit k of the packet is bit k%8 of byte k/8) onto opb, in pieces of up to 32 bits
 * (oggpack_write is all that libogg and the stand-in both provide) */
static void write_packet_bits(oggpack_buffer *opb, const uint8_t *p, long bits){
  long k;
  int c;
  for(k = 0; k < bits; k += 32){
    const int take = bits - k < 32 ? (int)(bits - k) : 32, nbytes = (take + 7) >> 3;
    unsigned long v = 0;
    for(c = 0; c < nbytes; c++) v |= (unsigned long)p[(k >> 3) + c] << (8*c);
    oggpack_write(opb, v, take);
  }
}

/* blocks[0..nb) of one size, entropy coded on the device: ONE vb200_encode_packets call (PCM in, packets out; when
 * bitrate-managed ONE vb200_encode_packets_managed call, all PACKETBLOBS packets of every block), then per block on
 * all host threads the state mapping0_forward leaves (vbi->ampmax, vb->mode) and the packet bits into
 * packetblob[PACKETBLOBS/2] (managed: packet k into packetblob[k], for lib/bitrate.c to choose from) */
static int forward_batch_packets(vb200_binding *bind, ms_batch *B, vorbis_block **blocks, int nb, int W, batch_after after,
                                 void *user){
  vb200_ctx *ctx = vb200shim_ctx(bind);
  vorbis_info *vi = blocks[0]->vd->vi;
  const int ch = vi->channels, N = (int)blocks[0]->pcmend;
  const int managed = vorbis_bitrate_managed(blocks[0]), curves = managed ? PACKETBLOBS : 1;
  const int bound = vb200_encode_packet_bound(ctx, W);
  vb200_encode_io io;
  int i, c, rc;
  PROF_T0();
  if(bound < 0) return OV_EFAULT;
  if((rc = batch_reserve(B, (size_t)nb, ch, N, 1))) return rc;
  if(B->pkt_cap < (size_t)curves*nb*bound || !B->pkt_off){
    free(B->pkt); free(B->pkt_off); free(B->pkt_bits);
    B->pkt = (uint8_t*)malloc((size_t)curves*nb*bound);
    B->pkt_off = (int64_t*)malloc(sizeof(int64_t)*curves*B->cap_blocks);
    B->pkt_bits = (int32_t*)malloc(sizeof(int32_t)*curves*B->cap_blocks);
    B->pkt_cap = B->pkt ? (size_t)curves*nb*bound : 0;
    if(!B->pkt || !B->pkt_off || !B->pkt_bits) return OV_EFAULT;
  }
#pragma omp parallel for private(c) schedule(static) if(nb > 8)
  for(i = 0; i < nb; i++){
    vorbis_block_internal *vbi = (vorbis_block_internal*)blocks[i]->internal;
    for(c = 0; c < ch; c++) memcpy(B->pcm + ((size_t)i*ch + c)*N, blocks[i]->pcm[c], sizeof(float)*N);
    B->desc[i].lW = (int32_t)blocks[i]->lW; B->desc[i].nW = (int32_t)blocks[i]->nW;
    B->desc[i].blocktype = vbi->blocktype; B->desc[i].ampmax = vbi->ampmax;
  }
  memset(&io, 0, sizeof(io));
  io.pcm = B->pcm; io.pcm_fmt = VB200_PCM_F32_BLOCKS; io.desc = B->desc; io.independent = 1; io.ampmax_out = B->ampmax;
  PROF_ADD(2);
  rc = managed ? vb200_encode_packets_managed(ctx, W, nb, 1, &io, B->pkt_off, B->pkt_bits, B->pkt, (int64_t)B->pkt_cap)
               : vb200_encode_packets(ctx, W, nb, 1, PACKETBLOBS/2, &io, B->pkt_off, B->pkt_bits, B->pkt, (int64_t)B->pkt_cap);
  PROF_ADD(3);
  if(rc){
    vb200shim_set_error(bind, rc);
    fprintf(stderr, "vb200 mapping0: vb200_encode_packets%s failed (%d): %s\n", managed ? "_managed" : "", rc, vb200_last_error());
    return OV_EFAULT;
  }
#pragma omp parallel for schedule(dynamic, 4) if(nb > 8)
  for(i = 0; i < nb; i++){
    vorbis_block_internal *vbi = (vorbis_block_internal*)blocks[i]->internal;
    int k;
    vbi->ampmax = B->ampmax[i];                                /* lib/mapping0.c:576 */
    blocks[i]->mode = W;
    for(k = 0; k < curves; k++){                               /* curve k of block i: packet k*nb + i */
      const size_t j = (size_t)k*nb + i;
      write_packet_bits(vbi->packetblob[managed ? k : PACKETBLOBS/2], B->pkt + B->pkt_off[j], B->pkt_bits[j]);
    }
    if(after) after(user, i);
  }
  PROF_ADD(4);
  return 0;
}

/* ---- seam 1: vorbis_func_mapping ---------------------------------------------------------------------------- */
static ms_batch g_single[2];                                   /* the single-block path's staging (one per block size) */

static int vb200_mapping0_forward(vorbis_block *vb){
  vb200_binding *bind = vb200shim_binding(vb->vd);
  if(!bind){ fprintf(stderr, "vb200 mapping0: vorbis_dsp_state is not attached (vb200shim_attach)\n"); return OV_EFAULT; }
  return forward_batch(bind, &g_single[vb->W ? 1 : 0], &vb, 1, (int)vb->W, NULL, NULL);
}
static void vb_pack(vorbis_info *vi, vorbis_info_mapping *vm, oggpack_buffer *opb){ mapping0_exportbundle.pack(vi, vm, opb); }
static vorbis_info_mapping *vb_unpack(vorbis_info *vi, oggpack_buffer *opb){ return mapping0_exportbundle.unpack(vi, opb); }
static void vb_free_info(vorbis_info_mapping *m){ mapping0_exportbundle.free_info(m); }
static int vb_inverse(vorbis_block *vb, vorbis_info_mapping *m){ return mapping0_exportbundle.inverse(vb, m); }

const vorbis_func_mapping vb200_mapping0_exportbundle = { &vb_pack, &vb_unpack, &vb_free_info, &vb200_mapping0_forward, &vb_inverse };

/* vorbis_analysis (lib/analysis.c:29-63) with the mapping call bound to the bundle above: what a libvorbis built
 * with `_mapping_P[0] = &vb200_mapping0_exportbundle` does.  Kept as a function so that the unmodified reference
 * objects and this seam can live in one test library. */
int vb200_vorbis_analysis(vorbis_block *vb, ogg_packet *op){
  vorbis_block_internal *vbi = (vorbis_block_internal*)vb->internal;
  int ret, i;
  vb->glue_bits = 0; vb->time_bits = 0; vb->floor_bits = 0; vb->res_bits = 0;
  for(i = 0; i < PACKETBLOBS; i++) oggpack_reset(vbi->packetblob[i]);
  if((ret = vb200_mapping0_exportbundle.forward(vb))) return ret;
  if(op){
    if(vorbis_bitrate_managed(vb)) return OV_EINVAL;
    op->packet = oggpack_get_buffer(&vb->opb);
    op->bytes = oggpack_bytes(&vb->opb);
    op->b_o_s = 0; op->e_o_s = vb->eofflag; op->granulepos = vb->granulepos; op->packetno = vb->sequence;
  }
  return 0;
}

/* ---- multi-stream driver: N independent encoders, the device sees their blocks together ---------------------- */
typedef void (*vb200ms_sink_t)(void *user, int stream, ogg_packet *op);
typedef struct vb200ms {
  int nstreams, channels, device;
  vorbis_info *vi;               /* one vorbis_info per stream (each owns its codec setup -> one binding each... */
  vorbis_comment vc;
  vorbis_dsp_state *vd;
  vorbis_block *vb;
  vb200_binding *bind;           /* ...so all states are initialised from stream 0's vorbis_info: one shared binding */
  ms_batch batch[2];
  vorbis_block **ready[2];
  int *ready_stream[2];
  /* the batched envelope search: staging of every stream's new 64-sample steps */
  int *env_first, *env_steps, *env_list;
  int32_t *env_nsteps;
  float *env_pcm; size_t env_pcm_cap;
  int32_t *env_state; uint8_t *env_ret; size_t env_ret_cap;
  int threads;
  vb200ms_sink_t sink; void *sink_user; int cur_w;
  int entropy_dev;               /* the context took the encoder's vb200_encode_entropy_setup */
  int host_entropy;              /* diagnostic: code on the host anyway (vb200ms_set_host_entropy) */
} vb200ms;

void vb200ms_close(vb200ms *m){
  int i, w;
  if(!m) return;
  if(g_prof_on > 0){
    fprintf(stderr, "vb200ms profile (s): envelope %.3f  blockout %.3f  stage %.3f  device call %.3f  host half %.3f  threads %d\n",
            g_prof[0], g_prof[1], g_prof[2], g_prof[3], g_prof[4], m->threads);
    memset(g_prof, 0, sizeof(g_prof));
  }
  if(m->bind){ vb200shim_select(&m->vd[0]); vb200shim_detach(); }
  for(i = 0; i < m->nstreams; i++){
    if(m->vb) vorbis_block_clear(&m->vb[i]);
    if(m->vd) vorbis_dsp_clear(&m->vd[i]);
  }
  if(m->vi){ vorbis_info_clear(&m->vi[0]); }
  vorbis_comment_clear(&m->vc);
  for(w = 0; w < 2; w++){
    free(m->batch[w].pcm); free(m->batch[w].desc); free(m->batch[w].posts); free(m->batch[w].nonzero);
    free(m->batch[w].iwork); free(m->batch[w].ampmax); free(m->ready[w]); free(m->ready_stream[w]);
    free(m->batch[w].pkt); free(m->batch[w].pkt_off); free(m->batch[w].pkt_bits);
  }
  free(m->env_first); free(m->env_steps); free(m->env_list); free(m->env_nsteps); free(m->env_pcm); free(m->env_state); free(m->env_ret);
  free(m->vi); free(m->vd); free(m->vb); free(m);
}

static int host_threads(void){
  const char *e = getenv("VB200MS_THREADS");
  int n = e ? atoi(e) : 0;
#ifdef _OPENMP
  if(n < 1){
    n = omp_get_num_procs();
    { /* a container may own fewer CPUs than it sees (cgroup quota) */
      FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
      long q = 0, per = 0;
      if(f){ if(fscanf(f, "%ld %ld", &q, &per) == 2 && q > 0 && per > 0 && q/per < n) n = (int)(q/per); fclose(f); }
    }
    if(n > 32) n = 32;
  }
  if(n < 1) n = 1;
  return n;
#else
  (void)n; return 1;
#endif
}

/* N encoders of one configuration, all bound to one device context: vorbis_encode_init_vbr(quality) or, when
 * managed, vorbis_encode_init(max, nominal, min bitrate; -1 = unset) */
static vb200ms *ms_open(int nstreams, int channels, long rate, float quality, int managed, long max_br, long nominal_br,
                        long min_br, int device){
  vb200ms *m = (vb200ms*)calloc(1, sizeof(*m));
  int i, w;
  if(!m || nstreams < 1) { free(m); return NULL; }
  m->nstreams = nstreams; m->channels = channels; m->device = device;
  m->vi = (vorbis_info*)calloc(1, sizeof(*m->vi));
  m->vd = (vorbis_dsp_state*)calloc(nstreams, sizeof(*m->vd));
  m->vb = (vorbis_block*)calloc(nstreams, sizeof(*m->vb));
  for(w = 0; w < 2; w++){
    m->ready[w] = (vorbis_block**)calloc(nstreams, sizeof(vorbis_block*));
    m->ready_stream[w] = (int*)calloc(nstreams, sizeof(int));
  }
  m->env_first = (int*)calloc(nstreams, sizeof(int)); m->env_steps = (int*)calloc(nstreams, sizeof(int));
  m->env_list = (int*)calloc(nstreams, sizeof(int)); m->env_nsteps = (int32_t*)calloc(nstreams, sizeof(int32_t));
  m->env_state = (int32_t*)calloc((size_t)nstreams*VB200_VE_STATE_WORDS(channels), sizeof(int32_t));
  m->threads = host_threads();
#ifdef _OPENMP
  omp_set_num_threads(m->threads);
#endif
  vorbis_comment_init(&m->vc);
  vorbis_info_init(&m->vi[0]);
  if(managed ? vorbis_encode_init(&m->vi[0], channels, rate, max_br, nominal_br, min_br)
             : vorbis_encode_init_vbr(&m->vi[0], channels, rate, quality)){ vb200ms_close(m); return NULL; }
  /* every state reads the same (read-only) setup; the first vorbis_analysis_init also builds the setup's shared
   * encode codebooks (ci->fullbooks, lib/block.c:211-224), so it runs alone, the others on all host threads
   * (each builds its own psy / floor / residue lookups, ~1.5 ms) */
  vorbis_analysis_init(&m->vd[0], &m->vi[0]);
  vorbis_block_init(&m->vd[0], &m->vb[0]);
#pragma omp parallel for schedule(dynamic, 4) if(nstreams > 8)
  for(i = 1; i < nstreams; i++){
    vorbis_analysis_init(&m->vd[i], &m->vi[0]);
    vorbis_block_init(&m->vd[i], &m->vb[i]);
  }
  if(vb200shim_attach(&m->vd[0], device)){ vb200ms_close(m); return NULL; }
  m->bind = vb200shim_binding(&m->vd[0]);
  {                              /* the device coder where the context takes this setup, else the host path */
    struct vb200_encode_entropy_setup es;
    int rc = vb200ms_entropy_setup_build(&m->vd[0], &es);
    if(!rc){
      rc = vb200_encode_entropy_setup(vb200shim_ctx(m->bind), &es);
      free((void*)es.books);
    }
    if(rc && rc != VB200_EIMPL){                      /* == OV_EIMPL */
      fprintf(stderr, "vb200 multistream: encode entropy setup failed (%d): %s\n", rc, vb200_last_error());
      vb200ms_close(m);
      return NULL;
    }
    m->entropy_dev = rc == 0;
  }
  return m;
}

int vb200ms_entropy_on_device(vb200ms *m){ return m->entropy_dev && !m->host_entropy; }
void vb200ms_set_host_entropy(vb200ms *m, int on){ m->host_entropy = on ? 1 : 0; }
vb200_ctx *vb200ms_context(vb200ms *m){ return vb200shim_ctx(m->bind); }

vb200ms *vb200ms_open(int nstreams, int channels, long rate, float quality, int device){
  return ms_open(nstreams, channels, rate, quality, 0, -1, -1, -1, device);
}

/* bitrate-managed encoders (CBR / ABR): each round's blocks of a size go to the device in one
 * vb200_encode_packets_managed call (vb200_encode_dsp_managed on the host path), and every stream's bitrate manager
 * picks its packets in round_after */
vb200ms *vb200ms_open_managed(int nstreams, int channels, long rate, long max_br, long nominal_br, long min_br, int device){
  return ms_open(nstreams, channels, rate, 0.f, 1, max_br, nominal_br, min_br, device);
}

vorbis_dsp_state *vb200ms_state(vb200ms *m, int stream){ return &m->vd[stream]; }

/* the analysis loop of _ve_envelope_search for ALL streams in one device call: the steps every stream has not
 * analysed yet are staged side by side (their counts differ - vb200_envelope_search_var), the results go back into
 * each state's envelope_lookup, and the blockout calls that follow find nothing left to analyse */
static int env_round(vb200ms *m){
  const int ch = m->channels;
  int i, na = 0, maxsteps = 0, rc;
#pragma omp parallel for schedule(static) if(m->nstreams > 8)
  for(i = 0; i < m->nstreams; i++) m->env_steps[i] = vb200shim_envelope_prepare(&m->vd[i], &m->env_first[i]);
  for(i = 0; i < m->nstreams; i++)
    if(m->env_steps[i] > 0){ m->env_list[na++] = i; if(m->env_steps[i] > maxsteps) maxsteps = m->env_steps[i]; }
  if(!na) return 0;
  {
    const long stride = ((64L*(maxsteps - 1) + 128) + 3) & ~3L;
    const size_t need = (size_t)na*ch*stride, rneed = (size_t)na*maxsteps;
    const size_t sw = VB200_VE_STATE_WORDS(ch);
    if(m->env_pcm_cap < need){ free(m->env_pcm); m->env_pcm = (float*)malloc(sizeof(float)*need); m->env_pcm_cap = m->env_pcm ? need : 0; }
    if(m->env_ret_cap < rneed){ free(m->env_ret); m->env_ret = (uint8_t*)malloc(rneed); m->env_ret_cap = m->env_ret ? rneed : 0; }
    if(!m->env_pcm || !m->env_ret) return OV_EFAULT;
#pragma omp parallel for schedule(static) if(na > 8)
    for(i = 0; i < na; i++){
      vorbis_dsp_state *v = &m->vd[m->env_list[i]];
      const long len = 64L*(m->env_steps[m->env_list[i]] - 1) + 128;
      int c;
      for(c = 0; c < ch; c++){
        float *dst = m->env_pcm + ((size_t)i*ch + c)*stride;
        memcpy(dst, v->pcm[c] + 64L*m->env_first[m->env_list[i]], sizeof(float)*len);
        if(len < stride) memset(dst + len, 0, sizeof(float)*(stride - len));
      }
      vb200shim_envelope_state_get(v, m->env_state + (size_t)i*sw);
      m->env_nsteps[i] = m->env_steps[m->env_list[i]];
    }
    rc = vb200_envelope_search_var(vb200shim_ctx(m->bind), na, m->env_pcm, VB200_PCM_F32_PLANAR, stride, maxsteps,
                                   m->env_nsteps, m->env_state, m->env_ret);
    if(rc){ vb200shim_set_error(m->bind, rc); fprintf(stderr, "vb200 multistream: envelope search failed (%d): %s\n", rc, vb200_last_error()); return OV_EFAULT; }
#pragma omp parallel for schedule(static) if(na > 8)
    for(i = 0; i < na; i++){
      const int s = m->env_list[i];
      vb200shim_envelope_commit(&m->vd[s], m->env_first[s], m->env_steps[s], m->env_state + (size_t)i*sw, m->env_ret + (size_t)i*maxsteps);
    }
  }
  return 0;
}

static void round_after(void *user, int i){                   /* run by the thread that packed block i of the current size */
  vb200ms *m = (vb200ms*)user;
  const int s = m->ready_stream[m->cur_w][i];
  ogg_packet op;
  vorbis_bitrate_addblock(&m->vb[s]);
  while(vorbis_bitrate_flushpacket(&m->vd[s], &op)) if(m->sink) m->sink(m->sink_user, s, &op);
}

/* One round: the envelope search of every stream in one device call, then every stream that has a block ready
 * (vorbis_analysis_blockout) contributes it; the blocks go to the device in one call per block size; the host half
 * (the reference's floor1_encode and residue backend, the per-stream bitrate queue) runs on all host threads, one
 * stream per thread at a time; packets are handed to `sink` (called from those threads, never concurrently for
 * one stream) in block order.  Returns the number of blocks processed (0: every stream needs more data), or a
 * negative OV_* code. */
typedef void (*vb200ms_sink)(void *user, int stream, ogg_packet *op);
int vb200ms_round(vb200ms *m, vb200ms_sink sink, void *user){
  int cnt[2] = {0, 0}, i, w, rc, total = 0;
  char *got;
  if(g_prof_on < 0){ const char *e = getenv("VB200MS_PROFILE"); g_prof_on = (e && atoi(e)) ? 1 : 0; }
  PROF_T0();
  if((rc = env_round(m))) return rc;
  PROF_ADD(0);
  got = (char*)calloc(m->nstreams, 1);
  if(!got) return OV_EFAULT;
#pragma omp parallel for schedule(dynamic, 8) if(m->nstreams > 8)
  for(i = 0; i < m->nstreams; i++){
    if(vorbis_analysis_blockout(&m->vd[i], &m->vb[i]) == 1){
      vorbis_block_internal *vbi = (vorbis_block_internal*)m->vb[i].internal;
      int k;
      m->vb[i].glue_bits = 0; m->vb[i].time_bits = 0; m->vb[i].floor_bits = 0; m->vb[i].res_bits = 0;
      for(k = 0; k < PACKETBLOBS; k++) oggpack_reset(vbi->packetblob[k]);      /* lib/analysis.c:37-41 */
      got[i] = 1;
    }
  }
  for(i = 0; i < m->nstreams; i++)
    if(got[i]){
      w = m->vb[i].W ? 1 : 0;
      m->ready[w][cnt[w]] = &m->vb[i];
      m->ready_stream[w][cnt[w]++] = i;
    }
  free(got);
  PROF_ADD(1);
  m->sink = sink; m->sink_user = user;
  for(w = 0; w < 2; w++){
    if(!cnt[w]) continue;
    m->cur_w = w;
    rc = vb200ms_entropy_on_device(m) ? forward_batch_packets(m->bind, &m->batch[w], m->ready[w], cnt[w], w, round_after, m)
                                      : forward_batch(m->bind, &m->batch[w], m->ready[w], cnt[w], w, round_after, m);
    if(rc) return rc;
    total += cnt[w];
  }
  return total;
}
