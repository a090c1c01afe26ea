/* vb200_decode.c — many libvorbis decoders of one codec setup, one device call per round: vb200md_*.
 *
 * The decode counterpart of vb200ms_* (vb200_mapping0.c).  A round decodes every packet queued since the last
 * round, for all streams at once.  On the device path (taken when vb200_decode_entropy_setup accepts the setup
 * that vb200md_entropy_new derives from the decoder's codebooks, floors and residues):
 *   1. host: the packet header as vorbis_synthesis reads it (lib/synthesis.c:37-82); the packets of all streams
 *      are laid out back to back in one byte buffer with per-block offsets and sizes.  A packet whose header
 *      does not parse is dropped, as examples/decoder_example.c drops it when vorbis_synthesis fails.
 *   2. device: the packet buffer and the small per-block arrays go up, then ONE vb200_decode_packets_resume_dev
 *      call for every stream and both block sizes (entropy decode, de-coupling, floor multiply, IMDCT,
 *      overlap-add; two kernel launches), and the PCM comes back.  The overlap of every (stream, channel) stays
 *      in device memory between rounds.
 * On the host path (any other setup, or vb200md_set_host_entropy) step 1 also runs the entropy half of
 * mapping0_inverse (lib/mapping0.c:714-751) on all host threads (OpenMP, one stream per thread at a time)
 * through the reference's own _floor_P[]->inverse1 and _residue_P[]->inverse, straight into the staging area of
 * vb200_decode_dsp_resume (residue vectors, floor-1 fit_value memo, block flags), and step 2 uploads that
 * staging and makes one vb200_decode_dsp_resume_dev call instead.
 *   3. host: the sample bookkeeping of vorbis_synthesis_blockin / pcmout (lib/block.c:741-751, 835-941) on each
 *      stream's counters (the first block returns nothing, a sequence gap loses the granule count, granulepos trims
 *      the first and the last packet), then each stream's finished samples go to the sink in order.
 * The device context is built here from the decoder's own lookups (floor-1 setups included) rather than through
 * vb200shim_attach, whose decoder bindings carry only what the function-level mdct_backward shim needs.
 * Limits: floor type 1 only (OV_EIMPL otherwise), two modes with blockflag 0 and 1, full-rate decode; the device
 * path also needs residue types 1 and 2 (type 0 keeps the host path).
 * Compiled like any libvorbis-internal backend against lib/codec_internal.h (oracle/decode.py builds it).
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "vorbis/codec.h"
#include "codec_internal.h"
#include "backends.h"
#include "registry.h"
#include "misc.h"
#include "window.h"

#include "vorbis_b200.h"

#ifdef _OPENMP
#include <omp.h>
#endif

typedef void (*vb200md_sink)(void *user, int stream, const void *pcm, long samples);

typedef struct {
  unsigned char *data;
  long bytes;
  ogg_int64_t granulepos, packetno;
  int eos;
  int W;                              /* block flag; -1 = header does not parse: dropped */
} md_packet;

typedef struct {
  md_packet *q; int nq, capq;        /* packets queued since the last round */
  /* the counters of vorbis_dsp_state / private_state that blockin and pcmout use (lib/block.c:741-941) */
  int W, lW, fresh;                   /* fresh: pcm_returned == -1 */
  ogg_int64_t sequence, granulepos, sample_count;
  int lastW;                          /* the carried block flag on the device, -1 = none */
} md_stream;

typedef struct vb200md {
  int nstreams, ch, pcm_s16, threads;
  long bs[2];
  vorbis_info vi;
  vorbis_comment vc;
  vorbis_dsp_state vd;               /* the decoder lookups every stream shares (read only after init) */
  vorbis_block *vb;                  /* one per thread */
  vb200_ctx *ctx;
  md_stream *st;
  vb200_decode_carry carry;          /* device */
  /* staging, grown never shrunk: host arrays and their device mirrors */
  size_t cap_blk, cap_res, cap_pcm;
  int32_t *Wseq, *count, *posts, *present;
  int64_t *coef_off, *pcm_off;
  int32_t *fin;                       /* samples block k of stream s finishes on the device */
  float *res;
  void *pcm;
  void *d_Wseq, *d_count, *d_posts, *d_present, *d_coef_off, *d_pcm_off, *d_res, *d_pcm;
  float *gather;                      /* float output of one stream, [ch][samples] for the sink */
  size_t cap_gather;
  /* device entropy decode: ent_dev = the context took the entropy setup; host_entropy = forced host path */
  int ent_dev, host_entropy;
  size_t cap_pkt;
  unsigned char *pkt;                 /* the packets of one round, back to back */
  int64_t *pkt_off;
  int32_t *pkt_bytes;
  void *d_pkt, *d_pkt_off, *d_pkt_bytes;
  /* counters */
  long rounds, blocks, packets;
  double device_s, host_s;
} vb200md;

static double md_now(void){ struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9*t.tv_nsec; }

void vb200md_close(vb200md *m){
  int i, k;
  if(!m) return;
  if(m->ctx){
    void *d[] = {m->carry.tail, m->carry.W, m->d_Wseq, m->d_count, m->d_posts, m->d_present, m->d_coef_off,
                 m->d_pcm_off, m->d_res, m->d_pcm, m->d_pkt, m->d_pkt_off, m->d_pkt_bytes};
    for(i = 0; i < (int)(sizeof(d)/sizeof(d[0])); i++) if(d[i]) vb200_free_device(m->ctx, d[i]);
    vb200_ctx_destroy(m->ctx);
  }
  if(m->vb){ for(i = 0; i < m->threads; i++) vorbis_block_clear(&m->vb[i]); free(m->vb); }
  if(m->vd.backend_state) vorbis_dsp_clear(&m->vd);
  vorbis_comment_clear(&m->vc);
  vorbis_info_clear(&m->vi);
  if(m->st){
    for(i = 0; i < m->nstreams; i++){ for(k = 0; k < m->st[i].nq; k++) free(m->st[i].q[k].data); free(m->st[i].q); }
    free(m->st);
  }
  free(m->Wseq); free(m->count); free(m->posts); free(m->present); free(m->coef_off); free(m->pcm_off);
  free(m->fin); free(m->res); free(m->pcm); free(m->gather);
  free(m->pkt); free(m->pkt_off); free(m->pkt_bytes);
  free(m);
}

/* the device setup of this decoder: transforms, windows, coupling and the floor-1 curve of every submap per
 * block size (lib/mapping0.c:714-795 reads nothing else) */
static int md_setup(vb200md *m, vb200_setup *s){
  codec_setup_info *ci = (codec_setup_info*)m->vi.codec_setup;
  private_state *b = (private_state*)m->vd.backend_state;
  int w, j, k;
  memset(s, 0, sizeof(*s));
  s->channels = m->vi.channels;
  s->rate = (int32_t)m->vi.rate;
  s->blocksizes[0] = (int32_t)ci->blocksizes[0];
  s->blocksizes[1] = (int32_t)ci->blocksizes[1];
  s->window[0] = _vorbis_window_get(b->window[0]);
  s->window[1] = _vorbis_window_get(b->window[1]);
  if(ci->modes != 2 || m->vi.channels > VB200_MAX_CHANNELS) return OV_EIMPL;
  for(w = 0; w < 2; w++){
    vorbis_info_mapping0 *mp;
    if(ci->mode_param[w]->blockflag != w || ci->map_type[ci->mode_param[w]->mapping] != 0) return OV_EIMPL;
    mp = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
    if(mp->submaps > VB200_MAX_SUBMAPS || mp->coupling_steps > VB200_MAX_COUPLING) return OV_EIMPL;
    s->coupling_steps[w] = mp->coupling_steps;
    for(k = 0; k < mp->coupling_steps; k++){ s->coupling_mag[w][k] = mp->coupling_mag[k]; s->coupling_ang[w][k] = mp->coupling_ang[k]; }
    s->submaps[w] = mp->submaps;
    for(k = 0; k < m->vi.channels; k++) s->chmux[w][k] = (uint8_t)mp->chmuxlist[k];
    for(j = 0; j < VB200_MAX_SUBMAPS; j++) s->residue[w][j].type = -1;
    for(j = 0; j < mp->submaps; j++){
      int fl = mp->floorsubmap[j];
      vorbis_info_floor1 *fi;
      vorbis_look_floor1 *lk;
      vb200_floor1_setup *o = &s->floor1[w][j];
      if(ci->floor_type[fl] != 1) return OV_EIMPL;
      fi = (vorbis_info_floor1*)ci->floor_param[fl];
      lk = (vorbis_look_floor1*)b->flr[fl];
      if(lk->posts > VB200_FLOOR1_STRIDE) return OV_EIMPL;
      o->posts = lk->posts;
      for(k = 0; k < lk->posts; k++) o->postlist[k] = fi->postlist[k];
      o->mult = fi->mult; o->n = lk->n;
      o->maxover = fi->maxover; o->maxunder = fi->maxunder; o->maxerr = fi->maxerr;
      o->twofitweight = fi->twofitweight; o->twofitatten = fi->twofitatten;
    }
  }
  return 0;
}


/* ---- the entropy setup of the device decoder, derived from the decoder's own tables ---------------------------- */
typedef struct {
  vb200_entropy_setup es;             /* first: the struct handed out */
  vb200_codebook *books;
  uint8_t *length;
  uint32_t *bits;
  int32_t *entry;
} md_entropy_tables;

static uint32_t md_bitrev(uint32_t x){
  x = ((x >> 16) & 0x0000ffffU) | ((x << 16) & 0xffff0000U);
  x = ((x >>  8) & 0x00ff00ffU) | ((x <<  8) & 0xff00ff00U);
  x = ((x >>  4) & 0x0f0f0f0fU) | ((x <<  4) & 0xf0f0f0f0U);
  x = ((x >>  2) & 0x33333333U) | ((x <<  2) & 0xccccccccU);
  return ((x >> 1) & 0x55555555U) | ((x << 1) & 0xaaaaaaaaU);
}

static int md_ilog(unsigned v){ int r = 0; while(v){ r++; v >>= 1; } return r; }

/* the codewords of one decode book (NULL arrays: count only), for both layouts of lib/codebook.h:73-110
 * (lib/sharedbook.c:393-519).  Unordered: codelist holds each codeword left-aligned, codelengths its length and
 * index its entry, n = hi_max (1 for the single-entry book, which has no hi_max).  Ordered: index[l] counts the
 * entries of lengths minlength..minlength+l, codelist[l] is the last codeword of that length left-aligned with
 * trailing ones, and the entries of one length take consecutive codes. */
static long md_book_codewords(const dec_codebook *db, uint8_t *len, uint32_t *bits, int32_t *entry){
  long i, n = 0;
  if(!db->codelist) return 0;
  if(db->codelengths){
    n = db->hi_max > 0 ? db->hi_max : 1;
    if(len)
      for(i = 0; i < n; i++){
        len[i] = (uint8_t)db->codelengths[i];
        bits[i] = md_bitrev(db->codelist[i]);
        entry[i] = db->index[i];
      }
  }else{
    int l, nl = db->maxlength - db->minlength + 1;
    long prev = 0;
    n = db->entries;
    if(len)
      for(l = 0; l < nl; l++){
        const int length = db->minlength + l;
        long e;
        for(e = prev; e < db->index[l]; e++){
          const uint32_t code = db->codelist[l] + 1U - ((uint32_t)(db->index[l] - e) << (32 - length));
          len[e] = (uint8_t)length;
          bits[e] = md_bitrev(code);
          entry[e] = (int32_t)e;
        }
        prev = db->index[l];
      }
  }
  return n;
}

void vb200md_entropy_free(vb200_entropy_setup *es){
  md_entropy_tables *t = (md_entropy_tables*)es;
  if(!t) return;
  free(t->books); free(t->length); free(t->bits); free(t->entry);
  free(t);
}

/* The vb200_entropy_setup of a decoder after vorbis_synthesis_init: every book of ci->decbooks, the floor and
 * residue decode fields of both modes' submaps, modebits.  Checks once that every codeword decodes to its entry
 * through the reference's vorbis_book_decode.  NULL on failure with *err = OV_EIMPL (a mode layout the driver
 * does not take), OV_EFAULT (no memory) or OV_EBADHEADER (a codeword that does not decode to its entry).
 * Free with vb200md_entropy_free. */
vb200_entropy_setup *vb200md_entropy_new(vorbis_info *vi, vorbis_dsp_state *vd, int *err){
  codec_setup_info *ci = (codec_setup_info*)vi->codec_setup;
  private_state *b = (private_state*)vd->backend_state;
  md_entropy_tables *t = (md_entropy_tables*)calloc(1, sizeof(*t));
  long total = 0, at = 0;
  int i, w, j, k, rc = OV_EFAULT;
  oggpack_buffer opb;
  if(!t) goto fail;
  for(i = 0; i < ci->books; i++) total += md_book_codewords(ci->decbooks + i, NULL, NULL, NULL);
  t->books = (vb200_codebook*)calloc(ci->books > 0 ? ci->books : 1, sizeof(*t->books));
  t->length = (uint8_t*)malloc(total > 0 ? total : 1);
  t->bits = (uint32_t*)malloc(sizeof(uint32_t) * (total > 0 ? total : 1));
  t->entry = (int32_t*)malloc(sizeof(int32_t) * (total > 0 ? total : 1));
  if(!t->books || !t->length || !t->bits || !t->entry) goto fail;
  t->es.nbooks = ci->books;
  t->es.books = t->books;
  t->es.modebits = b->modebits;
  rc = OV_EBADHEADER;
  oggpack_writeinit(&opb);
  for(i = 0; i < ci->books; i++){
    dec_codebook *db = ci->decbooks + i;
    vb200_codebook *o = &t->books[i];
    const long n = md_book_codewords(db, t->length + at, t->bits + at, t->entry + at);
    o->dim = db->dim; o->used = (int32_t)n;
    o->length = t->length + at; o->bits = t->bits + at; o->entry = t->entry + at;
    o->value = db->valuelist;
    for(k = 0; k < n; k++){                      /* self-check: the codeword decodes to its entry */
      oggpack_buffer rd;
      oggpack_reset(&opb);
      oggpack_write(&opb, o->bits[k], o->length[k]);
      oggpack_readinit(&rd, oggpack_get_buffer(&opb), (int)oggpack_bytes(&opb));
      if(vorbis_book_decode(db, &rd) != o->entry[k]){ oggpack_writeclear(&opb); goto fail; }
    }
    at += n;
  }
  oggpack_writeclear(&opb);
  rc = OV_EIMPL;
  if(ci->modes != 2) goto fail;
  for(w = 0; w < 2; w++){
    vorbis_info_mapping0 *mp;
    if(ci->mode_param[w]->blockflag != w || ci->map_type[ci->mode_param[w]->mapping] != 0) goto fail;
    mp = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
    if(mp->submaps > VB200_MAX_SUBMAPS) goto fail;
    for(j = 0; j < mp->submaps; j++){
      const int fl = mp->floorsubmap[j], rs = mp->residuesubmap[j];
      vb200_floor_decode *f = &t->es.floor[w][j];
      vb200_residue_decode *r = &t->es.residue[w][j];
      f->type = ci->floor_type[fl];
      if(f->type == 1){
        const vorbis_info_floor1 *fi = (const vorbis_info_floor1*)ci->floor_param[fl];
        f->partitions = fi->partitions;
        for(k = 0; k < fi->partitions && k < 31; k++) f->partitionclass[k] = fi->partitionclass[k];
        for(k = 0; k < 16; k++){
          int s;
          f->class_dim[k] = fi->class_dim[k]; f->class_subs[k] = fi->class_subs[k]; f->class_book[k] = fi->class_book[k];
          for(s = 0; s < 8; s++) f->class_subbook[k][s] = fi->class_subbook[k][s];
        }
      }
      r->type = ci->residue_type[rs];
      {
        const vorbis_info_residue0 *ri = (const vorbis_info_residue0*)ci->residue_param[rs];
        int acc = 0, c;
        r->begin = (int32_t)ri->begin; r->end = (int32_t)ri->end; r->grouping = ri->grouping;
        r->partitions = ri->partitions; r->partvals = ri->partvals; r->groupbook = ri->groupbook;
        for(c = 0; c < 64; c++){                  /* as res0_look lays them out, lib/res0.c:274-292 */
          const int stages = c < ri->partitions ? md_ilog((unsigned)ri->secondstages[c]) : 0;
          for(k = 0; k < 8; k++)
            r->stagebook[c][k] = k < stages && (ri->secondstages[c] & (1 << k)) ? ri->booklist[acc++] : -1;
        }
      }
    }
  }
  if(err) *err = 0;
  return &t->es;
fail:
  if(err) *err = rc;
  vb200md_entropy_free(t ? &t->es : NULL);
  return NULL;
}

static void md_reset(md_stream *t){
  t->fresh = 1; t->sequence = -1; t->granulepos = -1; t->sample_count = -1; t->lastW = -1;
}

/* hdr: the identification, comment and setup headers.  NULL on failure; *err (if given) = OV_* */
vb200md *vb200md_open_err(int nstreams, ogg_packet hdr[3], int pcm_s16, int device, int *err){
  vb200md *m = (vb200md*)calloc(1, sizeof(*m));
  vb200_setup s;
  size_t tail;
  int i, rc = OV_EFAULT;
  if(!m || nstreams <= 0 || !hdr){ rc = OV_EINVAL; goto fail; }
  m->nstreams = nstreams; m->pcm_s16 = pcm_s16 ? 1 : 0;
  vorbis_info_init(&m->vi);
  vorbis_comment_init(&m->vc);
  for(i = 0; i < 3; i++) if((rc = vorbis_synthesis_headerin(&m->vi, &m->vc, &hdr[i])) != 0) goto fail;
  if((rc = vorbis_synthesis_init(&m->vd, &m->vi)) != 0) goto fail;
  m->ch = m->vi.channels;
  m->bs[0] = vorbis_info_blocksize(&m->vi, 0);
  m->bs[1] = vorbis_info_blocksize(&m->vi, 1);
  if((rc = md_setup(m, &s)) != 0) goto fail;
#ifdef _OPENMP
  m->threads = omp_get_max_threads();
#else
  m->threads = 1;
#endif
  m->vb = (vorbis_block*)calloc(m->threads, sizeof(vorbis_block));
  m->st = (md_stream*)calloc(nstreams, sizeof(md_stream));
  if(!m->vb || !m->st){ rc = OV_EFAULT; goto fail; }
  for(i = 0; i < m->threads; i++) vorbis_block_init(&m->vd, &m->vb[i]);
  for(i = 0; i < nstreams; i++) md_reset(&m->st[i]);
  rc = OV_EFAULT;
  if(vb200_ctx_create(&s, device, &m->ctx)){ m->ctx = NULL; goto fail; }
  tail = (size_t)nstreams * m->ch;
  if(vb200_malloc_device(m->ctx, sizeof(float) * tail * (m->bs[1] / 2), (void**)&m->carry.tail)) goto fail;
  if(vb200_malloc_device(m->ctx, sizeof(int32_t) * tail, (void**)&m->carry.W)) goto fail;
  {
    int32_t *neg = (int32_t*)malloc(sizeof(int32_t) * tail);
    if(!neg) goto fail;
    for(i = 0; i < (int)tail; i++) neg[i] = -1;
    i = vb200_memcpy_h2d(m->ctx, m->carry.W, neg, sizeof(int32_t) * tail);
    free(neg);
    if(i) goto fail;
  }
  {                                   /* the device path where the context takes the entropy setup */
    int e;
    vb200_entropy_setup *es = vb200md_entropy_new(&m->vi, &m->vd, &e);
    if(!es){ rc = e; goto fail; }
    e = vb200_decode_entropy_setup(m->ctx, es);
    vb200md_entropy_free(es);
    if(e == VB200_EFAULT){ rc = OV_EFAULT; goto fail; }
    m->ent_dev = e == 0;
  }
  if(err) *err = 0;
  return m;
fail:
  if(err) *err = rc;
  vb200md_close(m);
  return NULL;
}

vb200md *vb200md_open(int nstreams, ogg_packet hdr[3], int pcm_s16, int device){
  return vb200md_open_err(nstreams, hdr, pcm_s16, device, NULL);
}

int vb200md_channels(vb200md *m){ return m->ch; }
/* the device context the driver built (its entropy setup registered where the device path is taken) */
vb200_ctx *vb200md_context(vb200md *m){ return m->ctx; }
/* 1 where rounds decode the packets on the device (vb200_decode_packets_resume_dev), 0 where the entropy half
 * runs on the host */
int vb200md_entropy_on_device(vb200md *m){ return m->ent_dev && !m->host_entropy; }
/* Diagnostic: on != 0 forces the host entropy path (to compare the two paths and to keep the fallback covered);
 * 0 returns to the path the setup allows.  Takes effect at the next round. */
void vb200md_set_host_entropy(vb200md *m, int on){ m->host_entropy = on ? 1 : 0; }
unsigned long long vb200md_launches(vb200md *m){ return vb200_launch_count(m->ctx); }
/* rounds that decoded blocks, blocks, audio packets; seconds in step 2 (copies in, the call, copies out) and in
 * steps 1 + 3 */
void vb200md_stats(vb200md *m, long *rounds, long *blocks, long *packets, double *device_s, double *host_s){
  *rounds = m->rounds; *blocks = m->blocks; *packets = m->packets; *device_s = m->device_s; *host_s = m->host_s;
}

int vb200md_packet(vb200md *m, int stream, const ogg_packet *op){
  md_stream *t;
  md_packet *p;
  if(!m || stream < 0 || stream >= m->nstreams || !op || op->bytes < 0 || (op->bytes && !op->packet)) return OV_EINVAL;
  t = &m->st[stream];
  if(t->nq == t->capq){
    int cap = t->capq ? 2 * t->capq : 8;
    md_packet *q = (md_packet*)realloc(t->q, sizeof(*q) * cap);
    if(!q) return OV_EFAULT;
    t->q = q; t->capq = cap;
  }
  p = &t->q[t->nq];
  p->data = (unsigned char*)malloc(op->bytes ? op->bytes : 1);
  if(!p->data) return OV_EFAULT;
  memcpy(p->data, op->packet, op->bytes);
  p->bytes = op->bytes; p->granulepos = op->granulepos; p->packetno = op->packetno; p->eos = op->e_o_s ? 1 : 0;
  t->nq++;
  return 0;
}

/* as vorbis_synthesis_restart (lib/block.c:695-716): the stream's next block primes a fresh overlap; packets
 * queued for it and not yet decoded are dropped */
void vb200md_restart(vb200md *m, int stream){
  md_stream *t;
  int k;
  if(!m || stream < 0 || stream >= m->nstreams) return;
  t = &m->st[stream];
  for(k = 0; k < t->nq; k++) free(t->q[k].data);
  t->nq = 0;
  if(t->lastW >= 0){
    int32_t *neg = (int32_t*)malloc(sizeof(int32_t) * m->ch);
    if(neg){
      for(k = 0; k < m->ch; k++) neg[k] = -1;
      vb200_memcpy_h2d(m->ctx, m->carry.W + (size_t)stream * m->ch, neg, sizeof(int32_t) * m->ch);
      free(neg);
    }
  }
  md_reset(t);
}

/* the packet header as vorbis_synthesis reads it, lib/synthesis.c:37-82; the block flag or -1 */
static int md_header(vb200md *m, vorbis_block *vb, const md_packet *p){
  codec_setup_info *ci = (codec_setup_info*)m->vi.codec_setup;
  private_state *b = (private_state*)m->vd.backend_state;
  oggpack_buffer *opb = &vb->opb;
  int mode;
  _vorbis_block_ripcord(vb);
  oggpack_readinit(opb, p->data, p->bytes);
  if(oggpack_read(opb, 1) != 0) return -1;                  /* not an audio packet */
  mode = oggpack_read(opb, b->modebits);
  if(mode == -1 || mode >= ci->modes || !ci->mode_param[mode]) return -1;
  vb->mode = mode;
  vb->W = ci->mode_param[mode]->blockflag;
  if(vb->W){
    vb->lW = oggpack_read(opb, 1);
    vb->nW = oggpack_read(opb, 1);
    if(vb->nW == -1) return -1;
  }else{
    vb->lW = 0; vb->nW = 0;
  }
  vb->pcmend = ci->blocksizes[vb->W];
  return vb->W;
}

/* the entropy half of mapping0_inverse, lib/mapping0.c:714-751, into the staging rows of one block */
static void md_entropy(vb200md *m, vorbis_block *vb, float *res, int32_t *posts, int32_t *present){
  codec_setup_info *ci = (codec_setup_info*)m->vi.codec_setup;
  private_state *b = (private_state*)m->vd.backend_state;
  vorbis_info_mapping0 *info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[vb->mode]->mapping];
  const int ch = m->ch;
  const long n = ci->blocksizes[vb->W];
  float *pcmbundle[VB200_MAX_CHANNELS];
  int zerobundle[VB200_MAX_CHANNELS], nonzero[VB200_MAX_CHANNELS];
  int i, j;
  for(i = 0; i < ch; i++){
    int submap = info->chmuxlist[i];
    int fl = info->floorsubmap[submap];
    int *memo = (int*)_floor_P[ci->floor_type[fl]]->inverse1(vb, b->flr[fl]);
    int32_t *row = posts + (size_t)i * VB200_FLOOR1_STRIDE;
    memset(row, 0, sizeof(int32_t) * VB200_FLOOR1_STRIDE);
    nonzero[i] = memo ? 1 : 0;
    present[i] = nonzero[i];
    if(memo){
      const int np = ((vorbis_look_floor1*)b->flr[fl])->posts;
      for(j = 0; j < np; j++) row[j] = memo[j];
    }
    memset(res + (size_t)i * (n / 2), 0, sizeof(float) * (n / 2));
  }
  for(i = 0; i < info->coupling_steps; i++)
    if(nonzero[info->coupling_mag[i]] || nonzero[info->coupling_ang[i]]){
      nonzero[info->coupling_mag[i]] = 1;
      nonzero[info->coupling_ang[i]] = 1;
    }
  for(i = 0; i < info->submaps; i++){
    int in_bundle = 0;
    for(j = 0; j < ch; j++)
      if(info->chmuxlist[j] == i){
        zerobundle[in_bundle] = nonzero[j] ? 1 : 0;
        pcmbundle[in_bundle++] = res + (size_t)j * (n / 2);
      }
    _residue_P[ci->residue_type[info->residuesubmap[i]]]->inverse(vb, b->residue[info->residuesubmap[i]],
                                                                 pcmbundle, zerobundle, in_bundle);
  }
}

#define GROW(ptr, cap_needed, cap, T) do { T *q_ = (T*)realloc((ptr), sizeof(T) * (cap_needed)); if(!q_) return OV_EFAULT; (ptr) = q_; } while(0)

static int md_reserve(vb200md *m, size_t nblk_total, size_t nres, size_t npcm, size_t npkt){
  const int ch = m->ch;
  const size_t pcm_el = m->pcm_s16 ? sizeof(int16_t) : sizeof(float);
  if(nblk_total > m->cap_blk){
    size_t c = nblk_total + nblk_total / 2;
    GROW(m->Wseq, c, 0, int32_t); GROW(m->coef_off, c, 0, int64_t); GROW(m->pcm_off, c, 0, int64_t);
    GROW(m->fin, c, 0, int32_t); GROW(m->present, c * ch, 0, int32_t);
    GROW(m->posts, c * ch * VB200_FLOOR1_STRIDE, 0, int32_t);
    GROW(m->pkt_off, c, 0, int64_t); GROW(m->pkt_bytes, c, 0, int32_t);
    if(m->d_pkt_off){ vb200_free_device(m->ctx, m->d_pkt_off); vb200_free_device(m->ctx, m->d_pkt_bytes); }
    m->d_pkt_off = m->d_pkt_bytes = NULL;
    if(vb200_malloc_device(m->ctx, sizeof(int64_t) * c, &m->d_pkt_off) ||
       vb200_malloc_device(m->ctx, sizeof(int32_t) * c, &m->d_pkt_bytes)) return OV_EFAULT;
    if(m->d_Wseq){ vb200_free_device(m->ctx, m->d_Wseq); vb200_free_device(m->ctx, m->d_coef_off);
                   vb200_free_device(m->ctx, m->d_pcm_off); vb200_free_device(m->ctx, m->d_present);
                   vb200_free_device(m->ctx, m->d_posts); }
    m->d_Wseq = m->d_coef_off = m->d_pcm_off = m->d_present = m->d_posts = NULL;
    if(vb200_malloc_device(m->ctx, sizeof(int32_t) * c, &m->d_Wseq) ||
       vb200_malloc_device(m->ctx, sizeof(int64_t) * c, &m->d_coef_off) ||
       vb200_malloc_device(m->ctx, sizeof(int64_t) * c, &m->d_pcm_off) ||
       vb200_malloc_device(m->ctx, sizeof(int32_t) * c * ch, &m->d_present) ||
       vb200_malloc_device(m->ctx, sizeof(int32_t) * c * ch * VB200_FLOOR1_STRIDE, &m->d_posts)) return OV_EFAULT;
    m->cap_blk = c;
  }
  if(!m->count){
    m->count = (int32_t*)malloc(sizeof(int32_t) * m->nstreams);
    if(!m->count || vb200_malloc_device(m->ctx, sizeof(int32_t) * m->nstreams, &m->d_count)) return OV_EFAULT;
  }
  if(npkt > m->cap_pkt){
    size_t c = npkt + npkt / 2;
    GROW(m->pkt, c, 0, unsigned char);
    if(m->d_pkt) vb200_free_device(m->ctx, m->d_pkt);
    m->d_pkt = NULL;
    if(vb200_malloc_device(m->ctx, c, &m->d_pkt)) return OV_EFAULT;
    m->cap_pkt = c;
  }
  if(nres > m->cap_res){
    size_t c = nres + nres / 2;
    GROW(m->res, c, 0, float);
    if(m->d_res) vb200_free_device(m->ctx, m->d_res);
    m->d_res = NULL;
    if(vb200_malloc_device(m->ctx, sizeof(float) * c, &m->d_res)) return OV_EFAULT;
    m->cap_res = c;
  }
  if(npcm > m->cap_pcm){
    size_t c = npcm + npcm / 2;
    void *q = realloc(m->pcm, pcm_el * c);
    if(!q) return OV_EFAULT;
    m->pcm = q;
    if(m->d_pcm) vb200_free_device(m->ctx, m->d_pcm);
    m->d_pcm = NULL;
    if(vb200_malloc_device(m->ctx, pcm_el * c, &m->d_pcm)) return OV_EFAULT;
    m->cap_pcm = c;
  }
  return 0;
}

/* one block's sample bookkeeping of vorbis_synthesis_blockin (lib/block.c:741-751, 835-941), full rate: of the
 * fin samples the device finished for it, [*lo, *hi) are returned */
static void md_blockin(vb200md *m, md_stream *t, const md_packet *p, long fin, long *lo, long *hi){
  t->lW = t->W;
  t->W = p->W;
  if(t->sequence == -1 || t->sequence + 1 != p->packetno){ t->granulepos = -1; t->sample_count = -1; }
  t->sequence = p->packetno;
  *lo = 0; *hi = t->fresh ? 0 : fin;
  t->fresh = 0;
  if(t->sample_count == -1) t->sample_count = 0;
  else t->sample_count += m->bs[t->lW] / 4 + m->bs[t->W] / 4;
  if(t->granulepos == -1){
    if(p->granulepos != -1){
      t->granulepos = p->granulepos;
      if(t->sample_count > t->granulepos){
        long extra = (long)(t->sample_count - p->granulepos);
        if(extra < 0) extra = 0;
        if(p->eos){                                            /* trim the end */
          if(extra > *hi - *lo) extra = *hi - *lo;
          *hi -= extra;
        }else{                                                 /* trim the beginning */
          *lo += extra;
          if(*lo > *hi) *lo = *hi;
        }
      }
    }
  }else{
    t->granulepos += m->bs[t->lW] / 4 + m->bs[t->W] / 4;
    if(p->granulepos != -1 && t->granulepos != p->granulepos){
      if(t->granulepos > p->granulepos){
        long extra = (long)(t->granulepos - p->granulepos);
        if(extra && p->eos){                                   /* partial last frame */
          if(extra > *hi - *lo) extra = *hi - *lo;
          if(extra < 0) extra = 0;
          *hi -= extra;
        }
      }
      t->granulepos = p->granulepos;
    }
  }
}

/* decode every queued packet of every stream: the number of blocks decoded, 0 if none was queued, or < 0 (OV_*) */
int vb200md_round(vb200md *m, vb200md_sink sink, void *user){
  const int ns = m->nstreams, ch = m->ch;
  double t0 = md_now(), t1, t2;
  int s, nblk = 0, rc;
  long total = 0, maxpcm = 0;
  size_t nres = 0, npkt = 0;
  const int on_dev = vb200md_entropy_on_device(m);
  /* step 1a: headers (cheap), block counts and the packed layout */
  for(s = 0; s < ns; s++){
    md_stream *t = &m->st[s];
    int k, n = 0;
    for(k = 0; k < t->nq; k++){ t->q[k].W = md_header(m, &m->vb[0], &t->q[k]); if(t->q[k].W >= 0) n++; }
    if(n > nblk) nblk = n;
    total += n;
  }
  if(total == 0){
    for(s = 0; s < ns; s++){ int k; for(k = 0; k < m->st[s].nq; k++) free(m->st[s].q[k].data); m->st[s].nq = 0; }
    m->host_s += md_now() - t0;
    return 0;
  }
  if((rc = md_reserve(m, (size_t)ns * nblk, 0, 0, 0))) return rc;
  for(s = 0; s < ns; s++){
    md_stream *t = &m->st[s];
    int k, j = 0, prev = t->lastW;
    long pos = 0;
    for(k = 0; k < t->nq; k++){
      const int W = t->q[k].W;
      const size_t it = (size_t)s * nblk + j;
      if(W < 0) continue;
      m->Wseq[it] = W;
      m->pkt_off[it] = (int64_t)npkt;
      m->pkt_bytes[it] = (int32_t)t->q[k].bytes;
      npkt += (size_t)t->q[k].bytes;
      m->coef_off[it] = (int64_t)nres;
      m->pcm_off[it] = pos;
      m->fin[it] = prev >= 0 ? (int32_t)(m->bs[prev] / 4 + m->bs[W] / 4) : 0;
      pos += m->fin[it];
      nres += (size_t)ch * (m->bs[W] / 2);
      prev = W; j++;
    }
    m->count[s] = j;
    for(; j < nblk; j++){
      const size_t it = (size_t)s * nblk + j;
      m->Wseq[it] = 0; m->coef_off[it] = 0; m->pcm_off[it] = 0; m->fin[it] = 0; m->pkt_off[it] = 0; m->pkt_bytes[it] = 0;
    }
    if(pos > maxpcm) maxpcm = pos;
  }
  if(maxpcm < 1) maxpcm = 1;
  if((rc = md_reserve(m, (size_t)ns * nblk, nres ? nres : 1, (size_t)ns * ch * maxpcm, npkt + 1))) return rc;
  /* step 1b, device path: the packets back to back */
  if(on_dev)
    for(s = 0; s < ns; s++){
      md_stream *t = &m->st[s];
      int k, j = 0;
      for(k = 0; k < t->nq; k++)
        if(t->q[k].W >= 0){
          const size_t it = (size_t)s * nblk + j++;
          memcpy(m->pkt + m->pkt_off[it], t->q[k].data, (size_t)t->q[k].bytes);
        }
    }
  /* step 1b, host path: the entropy half, one stream per thread at a time */
#pragma omp parallel for schedule(dynamic, 1)
  for(s = 0; s < (on_dev ? 0 : ns); s++){
    md_stream *t = &m->st[s];
#ifdef _OPENMP
    vorbis_block *vb = &m->vb[omp_get_thread_num()];
#else
    vorbis_block *vb = &m->vb[0];
#endif
    int k, j = 0;
    for(k = 0; k < t->nq; k++){
      const size_t it = (size_t)s * nblk + j;
      if(t->q[k].W < 0) continue;
      md_header(m, vb, &t->q[k]);
      md_entropy(m, vb, m->res + m->coef_off[it], m->posts + it * ch * VB200_FLOOR1_STRIDE, m->present + it * ch);
      j++;
    }
  }
  /* step 2: the device */
  t1 = md_now();
  {
    const size_t nb = (size_t)ns * nblk;
    const size_t pbytes = (m->pcm_s16 ? sizeof(int16_t) : sizeof(float)) * (size_t)ns * ch * maxpcm;
    if(vb200_memcpy_h2d(m->ctx, m->d_Wseq, m->Wseq, sizeof(int32_t) * nb) ||
       vb200_memcpy_h2d(m->ctx, m->d_count, m->count, sizeof(int32_t) * ns) ||
       vb200_memcpy_h2d(m->ctx, m->d_coef_off, m->coef_off, sizeof(int64_t) * nb) ||
       vb200_memcpy_h2d(m->ctx, m->d_pcm_off, m->pcm_off, sizeof(int64_t) * nb)) return OV_EFAULT;
    if(on_dev){
      if((npkt && vb200_memcpy_h2d(m->ctx, m->d_pkt, m->pkt, npkt)) ||
         vb200_memcpy_h2d(m->ctx, m->d_pkt_off, m->pkt_off, sizeof(int64_t) * nb) ||
         vb200_memcpy_h2d(m->ctx, m->d_pkt_bytes, m->pkt_bytes, sizeof(int32_t) * nb)) return OV_EFAULT;
      if(vb200_decode_packets_resume_dev(m->ctx, ns, nblk, (const int32_t*)m->d_count, (const int32_t*)m->d_Wseq,
                                         (const int64_t*)m->d_coef_off, (float*)m->d_res,
                                         (const int64_t*)m->d_pkt_off, (const int32_t*)m->d_pkt_bytes,
                                         (const uint8_t*)m->d_pkt, (const int64_t*)m->d_pcm_off, m->d_pcm,
                                         m->pcm_s16, maxpcm, &m->carry, NULL)) return OV_EFAULT;
    }else{
      if(vb200_memcpy_h2d(m->ctx, m->d_res, m->res, sizeof(float) * nres) ||
         vb200_memcpy_h2d(m->ctx, m->d_posts, m->posts, sizeof(int32_t) * nb * ch * VB200_FLOOR1_STRIDE) ||
         vb200_memcpy_h2d(m->ctx, m->d_present, m->present, sizeof(int32_t) * nb * ch)) return OV_EFAULT;
      if(vb200_decode_dsp_resume_dev(m->ctx, ns, nblk, (const int32_t*)m->d_count, (const int32_t*)m->d_Wseq,
                                     (const int64_t*)m->d_coef_off, (float*)m->d_res, (const int32_t*)m->d_posts,
                                     (const int32_t*)m->d_present, (const int64_t*)m->d_pcm_off, m->d_pcm,
                                     m->pcm_s16, maxpcm, &m->carry, NULL)) return OV_EFAULT;
    }
    if(vb200_memcpy_d2h(m->ctx, m->pcm, m->d_pcm, pbytes) || vb200_synchronize(m->ctx)) return OV_EFAULT;
  }
  t2 = md_now();
  /* step 3: the sample bookkeeping and the sink */
  for(s = 0; s < ns; s++){
    md_stream *t = &m->st[s];
    int k, j = 0;
    for(k = 0; k < t->nq; k++){
      md_packet *p = &t->q[k];
      if(p->W >= 0){
        const size_t it = (size_t)s * nblk + j;
        long lo, hi;
        md_blockin(m, t, p, m->fin[it], &lo, &hi);
        t->lastW = p->W;
        if(hi > lo){
          const long at = (long)m->pcm_off[it] + lo, n = hi - lo;
          if(m->pcm_s16){
            if(sink) sink(user, s, (const int16_t*)m->pcm + ((size_t)s * maxpcm + at) * ch, n);
          }else{
            int c;
            if((size_t)n * ch > m->cap_gather){
              float *q = (float*)realloc(m->gather, sizeof(float) * (size_t)n * ch);
              if(!q) return OV_EFAULT;
              m->gather = q; m->cap_gather = (size_t)n * ch;
            }
            /* [ch][samples] of this block: the sink is called per block, in order */
            for(c = 0; c < ch; c++)
              memcpy(m->gather + (size_t)c * n, (const float*)m->pcm + ((size_t)s * ch + c) * maxpcm + at, sizeof(float) * n);
            if(sink) sink(user, s, m->gather, n);
          }
        }
        j++;
      }
      free(p->data);
    }
    t->nq = 0;
  }
  m->packets += total;
  m->blocks += total;
  m->rounds++;
  m->device_s += t2 - t1;
  m->host_s += (t1 - t0) + (md_now() - t2);
  return (int)total;
}
