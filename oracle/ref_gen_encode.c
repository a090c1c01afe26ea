/* ref_gen_encode.c — the reference's encoder functions on a setup read from three header packets.  TEST
 * INFRASTRUCTURE ONLY.
 *
 *   rge_open       vorbis_synthesis_headerin on the identification, comment and setup packets; the encoder-only
 *                  fields the headers do not carry written in (per floor maxover, maxunder, maxerr, twofitweight,
 *                  twofitatten; per residue classmetric1 / classmetric2); then vorbis_analysis_init, whose
 *                  _vds_shared_init builds the books with vorbis_book_init_encode from book_param (the static
 *                  books rge_books reads from the setup packet: this reference's headerin fills only its decoder's
 *                  books).  *refused = the preconditions below that the setup breaks (RGE_* bits), and
 *                  where that is 0 the handle carries the product's vb200ms_entropy_setup_build of the encoder, the
 *                  decoder-side vb200_setup with the encoder fields and the classification setup written in, and
 *                  modebits.
 *   rge_fit        floor1_fit on rows of (logmdct, logmask)
 *   rge_encode     floor1_encode on rows of posts at the fit scale: the packed bits, the posts it leaves, ilogmask
 *   rge_classify   _residue_P[type]->class per submap, the channels bundled as mapping0_forward bundles them
 *   rge_packets    the packets mapping0_forward writes (lib/mapping0.c:603-683) from posts / nonzero / iwork
 *   rge_counts     fallback walks, dropped floor values, NULL fits
 *
 * Reference preconditions.  Outside the set below libvorbis's encoder reads or writes past its own arrays, so it
 * cannot serve as a reference there; rge_open refuses such a setup:
 *   RGE_STAGE_MAP    a residue stage book not of map type 1, or of a dimension outside 1..8 (p[8] and e[8] of
 *                    local_book_besterror, lib/res0.c:322-376)
 *   RGE_DELTA        a stage book whose rint(q_delta) < 1
 *   RGE_LATTICE      a stage book whose lattice is not full and centred: entries != quantvals^dim, an even
 *                    quantvals, or minval != -(quantvals >> 1) * delta (the fallback walk enumerates the vq/ value
 *                    pattern and carries past the last dimension otherwise)
 *   RGE_WALK8        a dimension-8 stage book with unused entries: the walk's last carry reads e[8]
 *   RGE_FLOOR        a floor with more than 65 posts, or postlist[1] above the half block of a mode using it
 *   RGE_RESIDUE      more than 64 residue partitions (classmetric1/2 have 64 entries), a residue that ends past its
 *                    rows (n for type 1, n times the bundle for type 2), or a type-2 residue whose _2class walk runs
 *                    past a row: begin/ch + partitions * ceil(grouping/ch) > n
 *   RGE_MODES        not two modes of block flags 0 and 1 on mapping type 0, or a book without codewords where
 *                    _make_words refused it
 * oracle/Makefile links this file with the stock reference objects, vorbis_b200/host/vb200_mapping0.c (for the
 * entropy setup builder) and the product library.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "codec_internal.h"
#include "backends.h"
#include "registry.h"
#include "window.h"

#include "vorbis_b200.h"

#define RGE_STAGE_MAP 1
#define RGE_DELTA     2
#define RGE_LATTICE   4
#define RGE_WALK8     8
#define RGE_FLOOR     16
#define RGE_RESIDUE   32
#define RGE_MODES     64

extern int *floor1_fit(vorbis_block *vb, vorbis_look_floor1 *look, const float *logmdct, const float *logmask);
extern int floor1_encode(oggpack_buffer *opb, vorbis_block *vb, vorbis_look_floor1 *look, int *post, int *ilogmask);
int vb200ms_entropy_setup_build(vorbis_dsp_state *vd, struct vb200_encode_entropy_setup *es);

typedef struct {
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  int init;
  vb200_setup s;
  struct vb200_encode_entropy_setup es;
  long fallback, dropped, nullfit;
} rge;

void rge_close(rge *h){
  if(!h) return;
  if(h->es.books) free((void*)h->es.books);
  if(h->init){ vorbis_block_clear(&h->vb); vorbis_dsp_clear(&h->vd); }
  vorbis_comment_clear(&h->vc);
  vorbis_info_clear(&h->vi);
  free(h);
}

static vorbis_info_mapping0 *rge_map(codec_setup_info *ci, int W){
  return (vorbis_info_mapping0*)ci->map_param[ci->mode_param[W]->mapping];
}

static int rge_ilog(unsigned long v){ int r = 0; while(v){ r++; v >>= 1; } return r; }

/* the setup packet's codebooks (Vorbis I spec 3.2.1) as static_codebooks in ci->book_param: this reference's
 * headerin unpacks books straight into its decoder's form and leaves book_param empty, while its encoder builds
 * its books (vorbis_book_init_encode) and floor1_encode reads entry counts from the static form.  0 or -1 */
static int rge_books(codec_setup_info *ci, const unsigned char *st, long st_bytes){
  oggpack_buffer opb;
  int i;
  long k;
  oggpack_readinit(&opb, (unsigned char*)st, (int)st_bytes);
  oggpack_adv(&opb, 56);
  if(oggpack_read(&opb, 8) + 1 != ci->books) return -1;
  for(i = 0; i < ci->books; i++){
    static_codebook *s = (static_codebook*)calloc(1, sizeof(*s));
    long nq;
    if(!s) return -1;
    ci->book_param[i] = s;
    s->allocedp = 1;
    if(oggpack_read(&opb, 24) != 0x564342) return -1;
    s->dim = oggpack_read(&opb, 16);
    s->entries = oggpack_read(&opb, 24);
    if(s->dim < 1 || s->entries < 1 || !(s->lengthlist = (char*)malloc(s->entries))) return -1;
    if(oggpack_read(&opb, 1)){                         /* ordered */
      long len = oggpack_read(&opb, 5) + 1, at = 0;
      while(at < s->entries){
        const long num = oggpack_read(&opb, rge_ilog(s->entries - at));
        if(num < 0 || at + num > s->entries || len > 32) return -1;
        memset(s->lengthlist + at, (int)len, num);
        at += num; len++;
      }
    }else{
      const int sparse = (int)oggpack_read(&opb, 1);
      for(k = 0; k < s->entries; k++)
        s->lengthlist[k] = sparse && !oggpack_read(&opb, 1) ? 0 : (char)(oggpack_read(&opb, 5) + 1);
    }
    s->maptype = (int)oggpack_read(&opb, 4);
    if(s->maptype < 0 || s->maptype > 2) return -1;
    if(!s->maptype) continue;
    s->q_min = oggpack_read(&opb, 32);
    s->q_delta = oggpack_read(&opb, 32);
    s->q_quant = (int)oggpack_read(&opb, 4) + 1;
    s->q_sequencep = (int)oggpack_read(&opb, 1);
    nq = s->maptype == 1 ? _book_maptype1_quantvals(s->dim, s->entries) : s->entries * s->dim;
    if(!(s->quantlist = (long*)malloc(sizeof(long) * nq))) return -1;
    for(k = 0; k < nq; k++) s->quantlist[k] = oggpack_read(&opb, s->q_quant);
    if(s->quantlist[nq - 1] < 0) return -1;            /* the packet ended */
  }
  return 0;
}

/* stage book k of partition class c of a residue (the partbooks layout of res0_look), or -1 */
static int rge_stage_book(const vorbis_info_residue0 *ri, int c, int k){
  int acc = 0, i, j;
  if(!((ri->secondstages[c] >> k) & 1)) return -1;
  for(i = 0; i < c; i++)
    for(j = 0; j < 8; j++) acc += (ri->secondstages[i] >> j) & 1;
  for(j = 0; j < k; j++) acc += (ri->secondstages[c] >> j) & 1;
  return ri->booklist[acc];
}

/* the preconditions above, on the header-level setup (before vorbis_analysis_init touches it) */
static int rge_refusal(rge *h){
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  int why = 0, w, j, r, c, k;
  if(ci->modes != 2 || ci->mode_param[0]->blockflag != 0 || ci->mode_param[1]->blockflag != 1 ||
     ci->map_type[ci->mode_param[0]->mapping] != 0 || ci->map_type[ci->mode_param[1]->mapping] != 0)
    return RGE_MODES;
  for(r = 0; r < ci->residues; r++){
    const vorbis_info_residue0 *ri = (const vorbis_info_residue0*)ci->residue_param[r];
    if(ri->partitions > 64){ why |= RGE_RESIDUE; continue; }
    for(c = 0; c < ri->partitions; c++)
      for(k = 0; k < 8; k++){
        const int b = rge_stage_book(ri, c, k);
        const static_codebook *s;
        long qv, lat = 1, e;
        int delta, minval, unused = 0;
        if(b < 0) continue;
        s = ci->book_param[b];
        if(s->maptype != 1 || s->dim < 1 || s->dim > 8){ why |= RGE_STAGE_MAP; continue; }
        qv = _book_maptype1_quantvals(s->dim, s->entries);
        delta = (int)rint(_float32_unpack((long)s->q_delta));
        minval = (int)rint(_float32_unpack((long)s->q_min));
        if(delta < 1) why |= RGE_DELTA;
        for(e = 0; e < s->dim; e++) lat *= qv;
        if(lat != s->entries || !(qv & 1) || minval != -(int)(qv >> 1) * delta) why |= RGE_LATTICE;
        for(e = 0; e < s->entries; e++) unused |= s->lengthlist[e] <= 0;
        if(s->dim == 8 && unused) why |= RGE_WALK8;
      }
  }
  for(w = 0; w < 2; w++){
    vorbis_info_mapping0 *mp = rge_map(ci, w);
    const int n = (int)(ci->blocksizes[w] / 2);
    for(j = 0; j < mp->submaps; j++){
      const int fl = mp->floorsubmap[j], rs = mp->residuesubmap[j];
      const vorbis_info_residue0 *ri = (const vorbis_info_residue0*)ci->residue_param[rs];
      int posts = 2, cib = 0, i;
      if(ci->floor_type[fl] != 1){ why |= RGE_MODES; continue; }
      {
        const vorbis_info_floor1 *fi = (const vorbis_info_floor1*)ci->floor_param[fl];
        for(i = 0; i < fi->partitions; i++) posts += fi->class_dim[fi->partitionclass[i]];
        if(posts > VIF_POSIT + 2 || fi->postlist[1] > n) why |= RGE_FLOOR;
      }
      for(i = 0; i < h->vi.channels; i++) cib += mp->chmuxlist[i] == j;
      if(ci->residue_type[rs] == 1 && ri->end > n) why |= RGE_RESIDUE;
      if(ci->residue_type[rs] == 2 && cib > 0){
        const long pv = (ri->end - ri->begin) / ri->grouping, per = (ri->grouping + cib - 1) / cib;
        if(ri->end > (long)n * cib || ri->begin / cib + pv * per > n) why |= RGE_RESIDUE;
      }
      if(ci->residue_type[rs] != 1 && ci->residue_type[rs] != 2) why |= RGE_RESIDUE;
    }
  }
  return why;
}

/* vb200md_setup's fields (as ref_headers.c takes them) plus the encoder fields and the classification setup */
static void rge_setup(rge *h){
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vb200_setup *s = &h->s;
  int w, j, k;
  memset(s, 0, sizeof(*s));
  s->channels = h->vi.channels;
  s->rate = (int32_t)h->vi.rate;
  s->blocksizes[0] = (int32_t)ci->blocksizes[0];
  s->blocksizes[1] = (int32_t)ci->blocksizes[1];
  s->window[0] = _vorbis_window_get(b->window[0]);
  s->window[1] = _vorbis_window_get(b->window[1]);
  for(w = 0; w < 2; w++){
    vorbis_info_mapping0 *mp = rge_map(ci, w);
    s->coupling_steps[w] = mp->coupling_steps;
    for(k = 0; k < mp->coupling_steps; k++){ s->coupling_mag[w][k] = mp->coupling_mag[k]; s->coupling_ang[w][k] = mp->coupling_ang[k]; }
    s->submaps[w] = mp->submaps;
    for(k = 0; k < h->vi.channels; k++) s->chmux[w][k] = (uint8_t)mp->chmuxlist[k];
    for(j = 0; j < VB200_MAX_SUBMAPS; j++) s->residue[w][j].type = -1;
    for(j = 0; j < mp->submaps; j++){
      const int fl = mp->floorsubmap[j], rs = mp->residuesubmap[j];
      vorbis_info_floor1 *fi = (vorbis_info_floor1*)ci->floor_param[fl];
      vorbis_look_floor1 *lk = (vorbis_look_floor1*)b->flr[fl];
      const vorbis_info_residue0 *ri = (const vorbis_info_residue0*)ci->residue_param[rs];
      vb200_floor1_setup *o = &s->floor1[w][j];
      vb200_residue_setup *r = &s->residue[w][j];
      o->posts = lk->posts;
      for(k = 0; k < lk->posts; k++) o->postlist[k] = fi->postlist[k];
      o->mult = fi->mult; o->n = lk->n;
      o->maxover = fi->maxover; o->maxunder = fi->maxunder; o->maxerr = fi->maxerr;
      o->twofitweight = fi->twofitweight; o->twofitatten = fi->twofitatten;
      r->type = ci->residue_type[rs];
      r->begin = (int32_t)ri->begin; r->end = (int32_t)ri->end; r->grouping = ri->grouping;
      r->partitions = ri->partitions;
      for(k = 0; k < 64; k++){ r->classmetric1[k] = ri->classmetric1[k]; r->classmetric2[k] = ri->classmetric2[k]; }
    }
  }
}

/* ffields [floors][5]: maxover, maxunder, maxerr, twofitweight, twofitatten; cmetric [residues][2][64] */
rge *rge_open(const unsigned char *id, long id_bytes, const unsigned char *cm, long cm_bytes,
              const unsigned char *st, long st_bytes, const float *ffields, int nfloors, const int *cmetric,
              int nresidues, int *rc, int *refused){
  rge *h = (rge*)calloc(1, sizeof(*h));
  const unsigned char *pk[3] = {id, cm, st};
  const long n[3] = {id_bytes, cm_bytes, st_bytes};
  codec_setup_info *ci;
  int k, i;
  *refused = 0;
  vorbis_info_init(&h->vi);
  vorbis_comment_init(&h->vc);
  for(k = 0; k < 3; k++){
    ogg_packet op;
    memset(&op, 0, sizeof(op));
    op.packet = (unsigned char*)pk[k]; op.bytes = n[k]; op.b_o_s = k == 0; op.packetno = k;
    if((*rc = vorbis_synthesis_headerin(&h->vi, &h->vc, &op)) != 0){ rge_close(h); return NULL; }
  }
  ci = (codec_setup_info*)h->vi.codec_setup;
  *rc = -1;
  if(nfloors != ci->floors || nresidues != ci->residues ){ rge_close(h); return NULL; }
  if(rge_books(ci, st, st_bytes)){ rge_close(h); return NULL; }
  if((*refused = rge_refusal(h)) != 0){ *rc = 0; return h; }
  for(k = 0; k < ci->floors; k++){
    vorbis_info_floor1 *fi = (vorbis_info_floor1*)ci->floor_param[k];
    const float *f = ffields + 5 * k;
    fi->maxover = f[0]; fi->maxunder = f[1]; fi->maxerr = f[2]; fi->twofitweight = f[3]; fi->twofitatten = f[4];
  }
  for(k = 0; k < ci->residues; k++){
    vorbis_info_residue0 *ri = (vorbis_info_residue0*)ci->residue_param[k];
    for(i = 0; i < 64; i++){                         /* const in the struct: written once, before any look */
      ((int*)ri->classmetric1)[i] = cmetric[128 * k + i];
      ((int*)ri->classmetric2)[i] = cmetric[128 * k + 64 + i];
    }
  }
  if(vorbis_analysis_init(&h->vd, &h->vi)){ rge_close(h); return NULL; }
  vorbis_block_init(&h->vd, &h->vb);
  h->init = 1;
  for(k = 0; k < ci->books; k++)
    if(!ci->fullbooks[k].codelist){ *refused = RGE_MODES; *rc = 0; return h; }
  rge_setup(h);
  if((*rc = vb200ms_entropy_setup_build(&h->vd, &h->es)) != 0){ rge_close(h); return NULL; }
  return h;
}

vb200_setup *rge_vb200_setup(rge *h){ return &h->s; }
struct vb200_encode_entropy_setup *rge_entropy(rge *h){ return &h->es; }
int rge_modebits(rge *h){ return ((private_state*)h->vd.backend_state)->modebits; }
/* fallback walks (stage-0 vectors on an unused lattice entry), dropped floor values, NULL fits */
void rge_counts(rge *h, long *out){ out[0] = h->fallback; out[1] = h->dropped; out[2] = h->nullfit; }
/* per book: dim, entries, minval, delta, quantvals of the encoder's codebook */
void rge_book(rge *h, int i, long *out){
  const codebook *b = ((codec_setup_info*)h->vi.codec_setup)->fullbooks + i;
  out[0] = b->dim; out[1] = b->entries; out[2] = b->minval; out[3] = b->delta; out[4] = b->quantvals;
}

static vorbis_look_floor1 *rge_floor(rge *h, int W, int submap){
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  return (vorbis_look_floor1*)((private_state*)h->vd.backend_state)->flr[rge_map(ci, W)->floorsubmap[submap]];
}

static void rge_block(rge *h, int W, int lW, int nW){
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  _vorbis_block_ripcord(&h->vb);
  h->vb.W = W; h->vb.lW = lW; h->vb.nW = nW; h->vb.pcmend = ci->blocksizes[W]; h->vb.mode = W;
}

/* floor1_fit of the floor of mode W, submap `submap`, on rows [nrows][n]: posts [nrows][VB200_FLOOR1_STRIDE] (zero
 * where the fit returned NULL), nonzero [nrows] */
void rge_fit(rge *h, int W, int submap, long nrows, const float *logmdct, const float *logmask, int *posts,
             int *nonzero){
  vorbis_look_floor1 *look = rge_floor(h, W, submap);
  const int n = (int)(((codec_setup_info*)h->vi.codec_setup)->blocksizes[W] / 2);
  long r;
  int j;
  for(r = 0; r < nrows; r++){
    int *p, *o = posts + r * VB200_FLOOR1_STRIDE;
    rge_block(h, W, 0, 0);
    p = floor1_fit(&h->vb, look, logmdct + r * n, logmask + r * n);
    memset(o, 0, sizeof(int) * VB200_FLOOR1_STRIDE);
    nonzero[r] = p != NULL;
    if(!p){ h->nullfit++; continue; }
    for(j = 0; j < look->posts; j++) o[j] = p[j];
  }
}

/* the floor values floor1_encode writes (lib/floor1.c:786-831) from the posts it leaves at the quantised scale: 0
 * where the post is unused or on its prediction, else the wrapped deviation */
static int rge_render_point(int x0, int x1, int y0, int y1, int x){
  int dy, adx, ady, err, off;
  y0 &= 0x7fff; y1 &= 0x7fff;
  dy = y1 - y0; adx = x1 - x0; ady = abs(dy);
  err = ady * (x - x0);
  off = err / adx;
  return dy < 0 ? y0 - off : y0 + off;
}

static long rge_dropped(rge *h, vorbis_look_floor1 *look, const int *post){
  const vorbis_info_floor1 *fi = look->vi;
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  int out[VIF_POSIT + 2], i, j, k, l;
  long drop = 0;
  for(i = 2; i < look->posts; i++){
    const int ln = look->loneighbor[i - 2], hn = look->hineighbor[i - 2];
    const int pr = rge_render_point(fi->postlist[ln], fi->postlist[hn], post[ln], post[hn], fi->postlist[i]);
    const int v = post[i] - pr, head = look->quant_q - pr < pr ? look->quant_q - pr : pr;
    if((post[i] & 0x8000) || (post[i] & 0x7fff) == pr) out[i] = 0;
    else if(v < 0) out[i] = v < -head ? head - v - 1 : -1 - v * 2;
    else out[i] = v >= head ? v + head : v << 1;
  }
  for(i = 0, j = 2; i < fi->partitions; i++){
    const int cl = fi->partitionclass[i], cdim = fi->class_dim[cl], csub = 1 << fi->class_subs[cl];
    for(k = 0; k < cdim; k++){
      int pick = 0, book;
      if(fi->class_subs[cl])
        for(l = 0; l < csub; l++){
          const int sb = fi->class_subbook[cl][l];
          if(out[j + k] < (sb < 0 ? 1 : ci->book_param[sb]->entries)){ pick = l; break; }
        }
      book = fi->class_subbook[cl][pick];
      if(book < 0) drop += out[j + k] != 0;
      else drop += out[j + k] >= ci->book_param[book]->entries || ci->book_param[book]->lengthlist[out[j + k]] <= 0;
    }
    j += cdim;
  }
  return drop;
}

/* floor1_encode of the floor of mode W, submap `submap`, on rows of posts [nrows][VB200_FLOOR1_STRIDE] at the fit
 * scale (an all-zero row is a NULL fit), replaced by the posts it leaves; the packed bits of row r at
 * bits + r*cap (cap bytes), nbits [nrows]; ilogmask [nrows][n]; ret [nrows] its return value */
void rge_encode(rge *h, int W, int submap, long nrows, int *posts, unsigned char *bits, long cap, long *nbits,
                int *ilogmask, int *ret){
  vorbis_look_floor1 *look = rge_floor(h, W, submap);
  const int n = (int)(((codec_setup_info*)h->vi.codec_setup)->blocksizes[W] / 2);
  long r;
  int j, any;
  for(r = 0; r < nrows; r++){
    int *p = posts + r * VB200_FLOOR1_STRIDE;
    oggpack_buffer opb;
    rge_block(h, W, 0, 0);
    oggpack_writeinit(&opb);
    for(j = any = 0; j < look->posts; j++) any |= p[j];
    ret[r] = floor1_encode(&opb, &h->vb, look, any ? p : NULL, ilogmask + r * n);
    if(any) h->dropped += rge_dropped(h, look, p);
    nbits[r] = opb.endbyte * 8 + opb.endbit;          /* the stand-in keeps libogg's fields */
    memset(bits + r * cap, 0, cap);
    memcpy(bits + r * cap, oggpack_get_buffer(&opb), oggpack_bytes(&opb) < cap ? oggpack_bytes(&opb) : cap);
    oggpack_writeclear(&opb);
  }
}

/* the classification of every submap of one block, as mapping0_forward calls it (lib/mapping0.c:660-672): classes
 * [ch][stride], left as given (-1) where nothing is classified; type 1 fills the rows of the bundle's used channels,
 * type 2 the row of the bundle's first channel */
static void rge_classify_block(rge *h, int W, int **rows, const int *nonzero, int *classes, int stride){
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_info_mapping0 *info = rge_map(ci, W);
  const int ch = h->vi.channels;
  int **bundle = (int**)malloc(sizeof(int*) * ch), *zero = (int*)malloc(sizeof(int) * ch), *who = (int*)malloc(sizeof(int) * ch);
  int i, j, k;
  for(i = 0; i < info->submaps; i++){
    const int rs = info->residuesubmap[i], type = ci->residue_type[rs];
    const vorbis_info_residue0 *ri = (const vorbis_info_residue0*)ci->residue_param[rs];
    const int pv = (int)((ri->end - ri->begin) / ri->grouping);
    int cib = 0, u = 0;
    long **cls;
    for(j = 0; j < ch; j++)
      if(info->chmuxlist[j] == i){ zero[cib] = nonzero[j] ? 1 : 0; who[cib] = j; bundle[cib++] = rows[j]; }
    cls = _residue_P[type]->class(&h->vb, b->residue[rs], bundle, zero, cib);
    if(!cls) continue;
    for(j = 0; j < (type == 2 ? 1 : cib); j++){
      int row;
      if(type == 2) row = who[0];
      else if(zero[j]) row = who[j];
      else continue;
      for(k = 0; k < pv && k < stride; k++) classes[(size_t)row * stride + k] = (int)cls[u][k];
      u++;
    }
  }
  free(bundle); free(zero); free(who);
}

void rge_classify(rge *h, int W, long nblocks, const int *iwork, const int *nonzero, int *classes, int stride){
  const int ch = h->vi.channels, n = (int)(((codec_setup_info*)h->vi.codec_setup)->blocksizes[W] / 2);
  int **rows = (int**)malloc(sizeof(int*) * ch);
  long blk;
  int i;
  for(blk = 0; blk < nblocks; blk++){
    rge_block(h, W, 0, 0);
    for(i = 0; i < ch; i++) rows[i] = (int*)iwork + ((size_t)blk * ch + i) * n;
    rge_classify_block(h, W, rows, nonzero + blk * ch, classes + (size_t)blk * ch * stride, stride);
  }
  free(rows);
}

/* 1 where the integer lattice index of a[0..dim) names an entry without a codeword (local_book_besterror's first
 * pass, lib/res0.c:333-349) */
static int rge_unused(const codebook *b, const int *a){
  const int ze = b->quantvals >> 1;
  int idx = 0, o;
  for(o = (int)b->dim - 1; o >= 0; o--){
    const int v = b->delta != 1 ? (a[o] - b->minval + (b->delta >> 1)) / b->delta : a[o] - b->minval;
    const int m = v < ze ? ((ze - v) << 1) - 1 : ((v - ze) << 1);
    idx = idx * b->quantvals + (m < 0 ? 0 : (m >= b->quantvals ? b->quantvals - 1 : m));
  }
  return b->c->lengthlist[idx] <= 0;
}

/* stage-0 vectors of one submap that take the fallback walk: vecs are the vectors the forward encodes (type 1: the
 * used channels; type 2: the bundle interleaved, cib channels) */
static long rge_walks(codec_setup_info *ci, const vorbis_info_residue0 *ri, int type, int **vecs, int nvec, int cib,
                      long **partword){
  const int pv = (int)((ri->end - ri->begin) / ri->grouping);
  long hits = 0;
  int i, j, k, q, tmp[8];
  for(i = 0; i < pv; i++)
    for(j = 0; j < nvec; j++){
      const int book = rge_stage_book(ri, (int)partword[j][i], 0);
      const codebook *b;
      if(book < 0) continue;
      b = ci->fullbooks + book;
      for(q = 0; q + b->dim <= ri->grouping; q += b->dim){
        for(k = 0; k < b->dim; k++){
          const long x = ri->begin + (long)i * ri->grouping + q + k;
          tmp[k] = type == 2 ? vecs[x % cib][x / cib] : vecs[j][x];
        }
        hits += rge_unused(b, tmp);
      }
    }
  return hits;
}

/* nblocks blocks of size W: desc [nblocks][2] = lW, nW; posts [nblocks][ch][VB200_FLOOR1_STRIDE] at the quantised
 * scale (all zero: a silent channel), replaced by what floor1_encode leaves; nonzero [nblocks][ch]; iwork
 * [nblocks][ch][n] (modified: the residue forward subtracts in place).  Packets back to back into out (cap bytes),
 * off / bytes per block.  Returns 0 or -1 (out too small). */
long rge_packets(rge *h, int W, long nblocks, const int *desc, int *posts, const int *nonzero, int *iwork,
                 unsigned char *out, long cap, long *off, long *bytes){
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  private_state *b = (private_state*)h->vd.backend_state;
  vorbis_info_mapping0 *info = rge_map(ci, W);
  const int ch = h->vi.channels, n = (int)(ci->blocksizes[W] / 2);
  int **rows = (int**)malloc(sizeof(int*) * ch), **bundle = (int**)malloc(sizeof(int*) * ch);
  int **ub = (int**)malloc(sizeof(int*) * ch);
  int *zero = (int*)malloc(sizeof(int) * ch), *scratch = (int*)malloc(sizeof(int) * n);
  long blk, at = 0;
  int rc = 0, i, j;
  for(blk = 0; blk < nblocks && !rc; blk++){
    oggpack_buffer opb;
    rge_block(h, W, desc[blk * 2], desc[blk * 2 + 1]);
    oggpack_writeinit(&opb);
    oggpack_write(&opb, 0, 1);
    oggpack_write(&opb, W, b->modebits);
    if(W){ oggpack_write(&opb, h->vb.lW, 1); oggpack_write(&opb, h->vb.nW, 1); }
    for(i = 0; i < ch; i++){
      vorbis_look_floor1 *look = rge_floor(h, W, info->chmuxlist[i]);
      int *p = posts + ((size_t)blk * ch + i) * VB200_FLOOR1_STRIDE, any = 0, fit[VIF_POSIT + 2];
      const int mult = look->vi->mult;
      for(j = 0; j < look->posts; j++) any |= p[j];
      if(!any){ floor1_encode(&opb, &h->vb, look, NULL, scratch); continue; }
      for(j = 0; j < look->posts; j++){                /* back to the fit scale */
        const int v = p[j] & 0x7fff;
        fit[j] = (mult == 1 ? v << 2 : mult == 2 ? v << 3 : mult == 3 ? v * 12 : v << 4) | (p[j] & 0x8000);
      }
      floor1_encode(&opb, &h->vb, look, fit, scratch);
      h->dropped += rge_dropped(h, look, fit);
      for(j = 0; j < look->posts; j++) p[j] = fit[j];
    }
    for(i = 0; i < ch; i++) rows[i] = iwork + ((size_t)blk * ch + i) * n;
    for(i = 0; i < info->submaps; i++){
      const int rs = info->residuesubmap[i], type = ci->residue_type[rs];
      const vorbis_info_residue0 *ri = (const vorbis_info_residue0*)ci->residue_param[rs];
      int cib = 0, used = 0, u = 0;
      long **cls;
      for(j = 0; j < ch; j++)
        if(info->chmuxlist[j] == i){ zero[cib] = nonzero[(size_t)blk * ch + j] ? 1 : 0; bundle[cib++] = rows[j]; }
      cls = _residue_P[type]->class(&h->vb, b->residue[rs], bundle, zero, cib);
      for(j = 0; j < cib; j++) used += zero[j];
      cib = 0;                                         /* res1_class compacted bundle[]: refill it */
      for(j = 0; j < ch; j++) if(info->chmuxlist[j] == i) bundle[cib++] = rows[j];
      for(j = 0; j < cib; j++) if(zero[j]) ub[u++] = bundle[j];
      if(cls) h->fallback += type == 2 ? rge_walks(ci, ri, 2, bundle, 1, cib, cls) : rge_walks(ci, ri, 1, ub, u, cib, cls);
      _residue_P[type]->forward(&opb, &h->vb, b->residue[rs], bundle, zero, cib, cls, i);
    }
    bytes[blk] = oggpack_bytes(&opb);
    off[blk] = at;
    if(at + bytes[blk] > cap) rc = -1;
    else memcpy(out + at, oggpack_get_buffer(&opb), bytes[blk]);
    at += bytes[blk];
    oggpack_writeclear(&opb);
  }
  free(rows); free(bundle); free(ub); free(zero); free(scratch);
  return rc;
}
