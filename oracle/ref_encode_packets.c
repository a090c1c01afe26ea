/* ref_encode_packets.c — checkers of the device entropy coder.  TEST INFRASTRUCTURE ONLY.
 *
 *   rep_ref_packets   the reference's own packet writing of mapping0_forward (lib/mapping0.c:603-683) on caller-given
 *                     posts / nonzero / iwork / lW / nW: header bits, floor1_encode per channel, then per submap
 *                     _residue_P[]->class and ->forward; returns the packets, the posts floor1_encode leaves, and
 *                     how many stage-0 residue vectors land on an unused lattice entry (each runs the fallback search
 *                     of local_book_besterror, lib/res0.c:349-376)
 *   (-DVB200_DROPIN, linked with the multi-stream driver)
 *   rep_open / rep_ctx / rep_on_device / rep_close   a vb200ms_open'd driver and its device context
 *   rep_setup_new / rep_setup_free                   the driver's struct vb200_encode_entropy_setup, for editing
 *   rep_ms_encode                                    ref_ms_encode with the host entropy path forced or not
 *
 * oracle/encode_packets.py links this file with the stock reference objects, and once more with the driver and the
 * drop-in objects.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"
#include "codec_internal.h"
#include "backends.h"
#include "registry.h"

#include "vorbis_b200.h"

#ifndef VB200_DROPIN
extern int floor1_encode(oggpack_buffer *opb, vorbis_block *vb, vorbis_look_floor1 *look, int *post, int *ilogmask);

static int rep_ilog(unsigned v){ int r = 0; while(v){ r++; v >>= 1; } return r; }

/* stage-0 book of partition class cls of residue ri (the partbooks layout of res0_look), or -1 */
static int stage0_book(const vorbis_info_residue0 *ri, int cls){
  int acc = 0, c, k;
  for(c = 0; c < cls; c++)
    for(k = 0; k < rep_ilog((unsigned)ri->secondstages[c]); k++) acc += (ri->secondstages[c] >> k) & 1;
  return (ri->secondstages[cls] & 1) ? ri->booklist[acc] : -1;
}

/* 1 where the integer lattice index of a[0..dim) names an entry without a codeword */
static int lattice_unused(const codebook *b, const int *a){
  const int ze = b->quantvals >> 1;
  int idx = 0, o;
  for(o = (int)b->dim - 1; o >= 0; o--){
    const int v = b->delta != 1 ? (a[o] - b->minval + (b->delta >> 1)) / b->delta : a[o] - b->minval;
    const int m = v < ze ? ((ze - v) << 1) - 1 : ((v - ze) << 1);
    idx = idx * b->quantvals + (m < 0 ? 0 : (m >= b->quantvals ? b->quantvals - 1 : m));
  }
  return b->c->lengthlist[idx] <= 0;
}

static long count_unused(codec_setup_info *ci, const vorbis_info_residue0 *ri, int type, int **in, int nvec, int cib,
                         long **partword){
  const int pv = (int)((ri->end - ri->begin) / ri->grouping);
  long hits = 0;
  int i, j, k, q;
  int tmp[256];
  if(!partword) return 0;
  for(i = 0; i < pv; i++)
    for(j = 0; j < nvec; j++){
      const int book = stage0_book(ri, (int)partword[j][i]);
      const codebook *b;
      if(book < 0) continue;
      b = ci->fullbooks + book;
      for(q = 0; q + b->dim <= ri->grouping; q += b->dim){
        for(k = 0; k < b->dim; k++){
          const long x = ri->begin + (long)i * ri->grouping + q + k;
          tmp[k] = type == 2 ? in[x % cib][x / cib] : in[j][x];
        }
        hits += lattice_unused(b, tmp);
      }
    }
  return hits;
}

/* nblocks blocks of size W of an encoder vorbis_encode_init_vbr(ch, rate, q): desc [nblocks][2] = lW, nW;
 * posts [nblocks][ch][VB200_FLOOR1_STRIDE] at the quantised scale (all zero: a silent channel), replaced by what
 * floor1_encode leaves; nonzero [nblocks][ch]; iwork [nblocks][ch][n] (modified: the residue forward subtracts in
 * place).  Packets back to back into out (cap bytes), off / bytes per block; *hits as above.  Returns 0 or -1. */
long rep_ref_packets(int ch, long rate, float q, int W, long nblocks, const int *desc, int *posts, const int *nonzero,
                     int *iwork, unsigned char *out, long cap, long *off, long *bytes, long *hits){
  vorbis_info vi; vorbis_dsp_state vd; vorbis_block vb;
  codec_setup_info *ci;
  private_state *b;
  vorbis_info_mapping0 *info;
  long blk, at = 0;
  int rc = 0;
  vorbis_info_init(&vi);
  if(vorbis_encode_init_vbr(&vi, ch, rate, q)){ vorbis_info_clear(&vi); return -1; }
  vorbis_analysis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  ci = (codec_setup_info*)vi.codec_setup;
  b = (private_state*)vd.backend_state;
  info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
  *hits = 0;
  for(blk = 0; blk < nblocks && !rc; blk++){
    const int n = (int)(ci->blocksizes[W] / 2);
    oggpack_buffer opb;
    int **rows = (int**)malloc(sizeof(int*) * ch), **bundle = (int**)malloc(sizeof(int*) * ch);
    int *zero = (int*)malloc(sizeof(int) * ch), *scratch = (int*)malloc(sizeof(int) * n);
    int i, j;
    _vorbis_block_ripcord(&vb);
    vb.W = W; vb.lW = desc[blk * 2]; vb.nW = desc[blk * 2 + 1]; vb.pcmend = ci->blocksizes[W]; vb.mode = W;
    oggpack_writeinit(&opb);
    oggpack_write(&opb, 0, 1);
    oggpack_write(&opb, W, b->modebits);
    if(W){ oggpack_write(&opb, vb.lW, 1); oggpack_write(&opb, vb.nW, 1); }
    for(i = 0; i < ch; i++){
      vorbis_look_floor1 *look = (vorbis_look_floor1*)b->flr[info->floorsubmap[info->chmuxlist[i]]];
      int *p = posts + ((size_t)blk * ch + i) * VB200_FLOOR1_STRIDE, any = 0, fit[VIF_POSIT + 2];
      const int mult = look->vi->mult;
      for(j = 0; j < look->posts; j++) any |= p[j];
      if(!any){ floor1_encode(&opb, &vb, look, NULL, scratch); continue; }
      for(j = 0; j < look->posts; j++){                /* back to the fit scale, as the host path of the driver does */
        const int v = p[j] & 0x7fff;
        fit[j] = (mult == 1 ? v << 2 : mult == 2 ? v << 3 : mult == 3 ? v * 12 : v << 4) | (p[j] & 0x8000);
      }
      floor1_encode(&opb, &vb, look, fit, scratch);
      for(j = 0; j < look->posts; j++) p[j] = fit[j];
    }
    for(i = 0; i < ch; i++) rows[i] = iwork + ((size_t)blk * ch + i) * n;
    for(i = 0; i < info->submaps; i++){
      const int resnum = info->residuesubmap[i], type = ci->residue_type[resnum];
      int cib = 0, used = 0;
      long **cls;
      for(j = 0; j < ch; j++)
        if(info->chmuxlist[j] == i){
          zero[cib] = nonzero[(size_t)blk * ch + j] ? 1 : 0;
          bundle[cib++] = rows[j];
        }
      cls = _residue_P[type]->class(&vb, b->residue[resnum], bundle, zero, cib);
      for(j = 0; j < cib; j++) used += zero[j];
      cib = 0;                                         /* res1_class compacted bundle[]: refill it */
      for(j = 0; j < ch; j++) if(info->chmuxlist[j] == i) bundle[cib++] = rows[j];
      if(type == 2) *hits += count_unused(ci, (vorbis_info_residue0*)ci->residue_param[resnum], 2, bundle, used ? 1 : 0, cib, cls);
      else{
        int *ub[256], u = 0;
        for(j = 0; j < cib; j++) if(zero[j]) ub[u++] = bundle[j];
        *hits += count_unused(ci, (vorbis_info_residue0*)ci->residue_param[resnum], type, ub, u, cib, cls);
      }
      _residue_P[type]->forward(&opb, &vb, b->residue[resnum], bundle, zero, cib, cls, i);
    }
    bytes[blk] = oggpack_bytes(&opb);
    off[blk] = at;
    if(at + bytes[blk] > cap) rc = -1;
    else memcpy(out + at, oggpack_get_buffer(&opb), bytes[blk]);
    at += bytes[blk];
    oggpack_writeclear(&opb);
    free(rows); free(bundle); free(zero); free(scratch);
  }
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_info_clear(&vi);
  return rc;
}
#endif

#ifdef VB200_DROPIN
typedef struct vb200ms vb200ms;
typedef void (*vb200ms_sink)(void *user, int stream, ogg_packet *op);
vb200ms *vb200ms_open(int nstreams, int channels, long rate, float quality, int device);
void vb200ms_close(vb200ms *m);
vorbis_dsp_state *vb200ms_state(vb200ms *m, int stream);
int vb200ms_round(vb200ms *m, vb200ms_sink sink, void *user);
int vb200ms_entropy_on_device(vb200ms *m);
void vb200ms_set_host_entropy(vb200ms *m, int on);
vb200_ctx *vb200ms_context(vb200ms *m);
int vb200ms_entropy_setup_build(vorbis_dsp_state *vd, struct vb200_encode_entropy_setup *es);

void *rep_open(int ns, int ch, long rate, float q, int device){ return vb200ms_open(ns, ch, rate, q, device); }
void *rep_ctx(void *m){ return vb200ms_context((vb200ms*)m); }
int rep_on_device(void *m){ return vb200ms_entropy_on_device((vb200ms*)m); }
void rep_close(void *m){ vb200ms_close((vb200ms*)m); }
int rep_blocksize(void *m, int w){ return vorbis_info_blocksize(vb200ms_state((vb200ms*)m, 0)->vi, w); }

/* a copy of the setup the driver registered (its codeword arrays still point into the driver's encoder) */
struct vb200_encode_entropy_setup *rep_setup_new(void *m){
  struct vb200_encode_entropy_setup *es = (struct vb200_encode_entropy_setup*)malloc(sizeof(*es));
  if(es && vb200ms_entropy_setup_build(vb200ms_state((vb200ms*)m, 0), es)){ free(es); es = NULL; }
  return es;
}
void rep_setup_free(struct vb200_encode_entropy_setup *es){ if(es){ free((void*)es->books); free(es); } }

typedef struct { uint64_t *hash; long *bytes, *count; int *eos; } rep_sum;
static void rep_sink(void *user, int stream, ogg_packet *op){       /* the summary of ref_driver.c's ms_sink */
  rep_sum *s = (rep_sum*)user;
  long k;
  uint64_t h = s->hash[stream];
  for(k = 0; k < op->bytes; k++){ h ^= op->packet[k]; h *= 1099511628211ULL; }
  h ^= (uint64_t)op->bytes; h *= 1099511628211ULL;
  s->hash[stream] = h; s->bytes[stream] += op->bytes; s->count[stream]++;
  if(op->e_o_s) s->eos[stream] = 1;
}

/* pcm [nstreams][ch][nsamples] through one driver in 1024-sample writes; host_entropy forces the host path.
 * *on_device: the path the driver took.  Returns total blocks, or < 0 */
long rep_ms_encode(int nstreams, int ch, long rate, float q, int device, int host_entropy, const float *pcm,
                   long nsamples, uint64_t *hash, long *bytes, long *count, int *on_device){
  vb200ms *m = vb200ms_open(nstreams, ch, rate, q, device);
  rep_sum sum;
  long pos = 0, blocks = 0;
  int i, c, r, alldone = 0;
  int *eos = (int*)calloc(nstreams, sizeof(int));
  if(!m){ free(eos); return -1; }
  vb200ms_set_host_entropy(m, host_entropy);
  *on_device = vb200ms_entropy_on_device(m);
  for(i = 0; i < nstreams; i++){ hash[i] = 1469598103934665603ULL; bytes[i] = 0; count[i] = 0; }
  sum.hash = hash; sum.bytes = bytes; sum.count = count; sum.eos = eos;
  while(!alldone){
    const long todo = nsamples - pos < 1024 ? nsamples - pos : 1024;
    for(i = 0; i < nstreams; i++){
      vorbis_dsp_state *vd = vb200ms_state(m, i);
      if(todo > 0){
        float **buf = vorbis_analysis_buffer(vd, (int)todo);
        for(c = 0; c < ch; c++) memcpy(buf[c], pcm + ((size_t)i * ch + c) * nsamples + pos, sizeof(float) * todo);
        vorbis_analysis_wrote(vd, (int)todo);
      }else vorbis_analysis_wrote(vd, 0);
    }
    pos += todo > 0 ? todo : 0;
    while((r = vb200ms_round(m, rep_sink, &sum)) > 0) blocks += r;
    if(r < 0){ blocks = r; break; }
    if(todo <= 0) alldone = 1;
  }
  vb200ms_close(m);
  free(eos);
  return blocks;
}
#endif
