/* vb_oracle_decode_streams.c — plain-C restatement of the per-stream plan of vb200_decode_streams_packets
 * (vorbis_b200/csrc/vb200_decode_streams.cuh).  TEST INFRASTRUCTURE ONLY; no reference source is used.
 *
 * The packet header of vorbis_synthesis (lib/synthesis.c:41-71) with modes 0 and 1 of block flags 0 and 1, then the
 * sample bookkeeping of vorbis_synthesis_blockin / vorbis_synthesis_pcmout (lib/block.c:741-751, 835-941): which of
 * the samples a block finishes the loop returns ([lo, hi)), granulepos and sample_count, at full and half rate.  It
 * also keeps centerW so that pcm_returned and pcm_current can be compared with the reference's own.
 *
 *   vbo_ds_init   the state vorbis_synthesis_restart leaves
 *   vbo_ds_run    npkt packets in order; per packet REC values as oracle/ref_decode_plan.c records them
 *                 (status, W, samples, granulepos, pcm_returned, pcm_current, sequence, sample_count) plus the
 *                 returned window lo, hi and the finished-sample count fin of that block.
 */
#include <stdint.h>
#include <string.h>

#define META 5
#define REC 11

typedef struct {
  int64_t granulepos, sample_count, sequence, pcm_returned, pcm_current;
  int32_t W, centerW;          /* W = -1: no block since the restart (pcm_returned == -1) */
} vbo_ds_state;

void vbo_ds_init(vbo_ds_state *s, const int *bs, int hs){
  memset(s, 0, sizeof(*s));
  s->granulepos = -1; s->sample_count = -1; s->sequence = -1; s->pcm_returned = -1; s->W = -1;
  s->centerW = bs[1] >> (hs + 1);
  s->pcm_current = s->centerW >> hs;
}

/* oggpack_read of lib/bitwise.c: k bits LSb first if k bits remain, else -1 and every later read fails */
typedef struct { const unsigned char *p; long nbits, pos; } rd;
static long rd_bits(rd *r, int k){
  long v = 0;
  int i;
  if(r->pos + k > r->nbits){ r->pos = r->nbits + 1; return -1; }
  for(i = 0; i < k; i++, r->pos++) v |= (long)((r->p[r->pos >> 3] >> (r->pos & 7)) & 1) << i;
  return v;
}

static int header(const unsigned char *p, long bytes, int modebits){
  rd r = {p, 8 * bytes, 0};
  long mode;
  if(rd_bits(&r, 1) != 0) return -135;                    /* OV_ENOTAUDIO */
  mode = rd_bits(&r, modebits);
  if(mode == -1 || mode >= 2) return -136;                /* OV_EBADPACKET: no mode_param */
  if(mode == 0) return 0;
  rd_bits(&r, 1);
  return rd_bits(&r, 1) == -1 ? -136 : 1;
}

void vbo_ds_run(vbo_ds_state *s, const unsigned char *buf, const long *meta, long npkt, int modebits, const int *bs,
                int hs, int64_t *rec){
  long k;
  for(k = 0; k < npkt; k++){
    const long *m = meta + k * META;
    int64_t *r = rec + k * REC;
    const int v = header(buf + m[0], m[1], modebits);
    const int64_t pgp = m[2], eos = m[3], pno = m[4];
    int64_t lo = 0, hi = 0, fin = 0;
    r[0] = v < 0 ? v : 0; r[1] = v < 0 ? -1 : v;
    if(v >= 0){
      const int lW = s->W, W = v, n1 = bs[1] >> (hs + 1);
      const int thisCenter = s->centerW ? n1 : 0, prevCenter = s->centerW ? 0 : n1;
      fin = lW >= 0 ? (bs[lW] / 4 + bs[W] / 4) >> hs : 0;
      if(s->sequence == -1 || s->sequence + 1 != pno){ s->granulepos = -1; s->sample_count = -1; }
      s->sequence = pno;
      hi = fin;
      s->centerW = s->centerW ? 0 : n1;
      if(s->sample_count == -1) s->sample_count = 0;
      else s->sample_count += bs[lW] / 4 + bs[W] / 4;
      if(s->granulepos == -1){
        if(pgp != -1){
          s->granulepos = pgp;
          if(s->sample_count > s->granulepos){
            int64_t extra = s->sample_count - pgp;
            if(extra < 0) extra = 0;
            if(eos){
              if(extra > (hi - lo) << hs) extra = (hi - lo) << hs;
              hi -= extra >> hs;
            }else{
              lo += extra >> hs;
              if(lo > hi) lo = hi;
            }
          }
        }
      }else{
        s->granulepos += bs[lW] / 4 + bs[W] / 4;
        if(pgp != -1 && s->granulepos != pgp){
          if(s->granulepos > pgp){
            int64_t extra = s->granulepos - pgp;
            if(extra && eos){
              if(extra > (hi - lo) << hs) extra = (hi - lo) << hs;
              if(extra < 0) extra = 0;
              hi -= extra >> hs;
            }
          }
          s->granulepos = pgp;
        }
      }
      if(lW < 0){ s->pcm_returned = s->pcm_current = thisCenter; }   /* the first block returns nothing */
      else{ s->pcm_returned = prevCenter + lo; s->pcm_current = prevCenter + hi; }
      s->W = W;
    }
    r[2] = hi - lo;
    r[3] = s->granulepos; r[4] = s->pcm_returned; r[5] = s->pcm_current; r[6] = s->sequence;
    r[7] = s->sample_count; r[8] = lo; r[9] = hi; r[10] = fin;
    if(v >= 0) s->pcm_returned = s->pcm_current;            /* vorbis_synthesis_read of everything returned */
  }
}
