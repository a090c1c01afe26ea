/* ref_decode_streams.c — decode runs for the tests and tools/decode_throughput.py.  TEST INFRASTRUCTURE ONLY.
 *
 *   rds_encode          the stock encoder (vorbis_encode_init_vbr): every packet's bytes with its granulepos,
 *                       e_o_s and packetno (3 headers, then audio)
 *   rds_stock_decode    the stock decoder on such packets with their real granulepos: vorbis_synthesis ->
 *                       vorbis_synthesis_blockin -> vorbis_synthesis_pcmout, float planar or the int16 of
 *                       examples/decoder_example.c:250-262; rds_stock_decode_many: many streams on all host threads
 *   rds_md_run          (-DVB200_DROPIN) the same packets of many streams through the multi-stream decode driver
 *                       (vorbis_b200/host/vb200_decode.c), fed in a given per-round schedule
 *
 * Packets live back to back in one byte buffer; meta[i] = {offset, bytes, granulepos, e_o_s, packetno}.
 * oracle/decode.py links this file with the objects oracle/Makefile compiles from the unmodified reference sources.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"

#define META 5

static int keep(const ogg_packet *op, unsigned char *buf, long cap, long *off, long *meta, long *n, long maxn){
  long *m;
  if(*n >= maxn || *off + op->bytes > cap) return 1;
  memcpy(buf + *off, op->packet, op->bytes);
  m = meta + *n * META;
  m[0] = *off; m[1] = op->bytes; m[2] = (long)op->granulepos; m[3] = op->e_o_s; m[4] = (long)op->packetno;
  *off += op->bytes; (*n)++;
  return 0;
}

/* pcm [ch][ns]; returns the packet count, or -1 */
long rds_encode(int ch, long rate, float quality, const float *pcm, long ns, unsigned char *buf, long cap,
                long *meta, long maxn){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  ogg_packet hdr[3], op;
  long pos = 0, off = 0, n = 0;
  int i, eos = 0, bad = 0;
  vorbis_info_init(&vi);
  if(vorbis_encode_init_vbr(&vi, ch, rate, quality)){ vorbis_info_clear(&vi); return -1; }
  vorbis_comment_init(&vc);
  vorbis_analysis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  vorbis_analysis_headerout(&vd, &vc, &hdr[0], &hdr[1], &hdr[2]);
  for(i = 0; i < 3; i++) bad |= keep(&hdr[i], buf, cap, &off, meta, &n, maxn);
  while(!eos && !bad){
    long todo = ns - pos < 1024 ? ns - pos : 1024;
    if(todo > 0){
      float **b = vorbis_analysis_buffer(&vd, (int)todo);
      for(i = 0; i < ch; i++) memcpy(b[i], pcm + (size_t)i*ns + pos, sizeof(float)*todo);
      vorbis_analysis_wrote(&vd, (int)todo);
      pos += todo;
    }else vorbis_analysis_wrote(&vd, 0);
    while(vorbis_analysis_blockout(&vd, &vb) == 1){
      vorbis_analysis(&vb, NULL);
      vorbis_bitrate_addblock(&vb);
      while(vorbis_bitrate_flushpacket(&vd, &op)){
        bad |= keep(&op, buf, cap, &off, meta, &n, maxn);
        if(op.e_o_s) eos = 1;
      }
    }
    if(todo <= 0) eos = 1;
  }
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return bad ? -1 : n;
}

static void to_packet(ogg_packet *op, const unsigned char *buf, const long *m){
  memset(op, 0, sizeof(*op));
  op->packet = (unsigned char*)buf + m[0]; op->bytes = m[1]; op->granulepos = m[2]; op->e_o_s = m[3];
  op->packetno = m[4]; op->b_o_s = (m[4] == 0);
}

/* examples/decoder_example.c:250-262 */
static int16_t s16_of(float x){
  int val = (int)floor(x * 32767.f + .5f);
  if(val > 32767) val = 32767;
  if(val < -32768) val = -32768;
  return (int16_t)val;
}

/* hdr: the 3 header packets (meta rows), audio: npkt audio packets.  out: float [ch][cap] or (s16) int16 [cap][ch];
 * NULL = count only.  Returns the samples per channel, or -1. */
long rds_stock_decode(const unsigned char *buf, const long *hdr, const long *audio, long npkt, int s16, void *out,
                      long cap){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  long produced = 0, k;
  int i;
  vorbis_info_init(&vi); vorbis_comment_init(&vc);
  for(k = 0; k < 3; k++){
    ogg_packet hp;
    to_packet(&hp, buf, hdr + k * META);
    if(vorbis_synthesis_headerin(&vi, &vc, &hp) < 0){ vorbis_comment_clear(&vc); vorbis_info_clear(&vi); return -1; }
  }
  vorbis_synthesis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  for(k = 0; k < npkt; k++){
    ogg_packet op; float **pcm; int got;
    to_packet(&op, buf, audio + k * META);
    if(vorbis_synthesis(&vb, &op) == 0) vorbis_synthesis_blockin(&vd, &vb);
    while((got = vorbis_synthesis_pcmout(&vd, &pcm)) > 0){
      long take = got, j;
      if(out){
        if(produced + take > cap) take = cap - produced;
        for(i = 0; i < vi.channels; i++)
          for(j = 0; j < take; j++){
            if(s16) ((int16_t*)out)[(produced + j) * vi.channels + i] = s16_of(pcm[i][j]);
            else ((float*)out)[(size_t)i * cap + produced + j] = pcm[i][j];
          }
      }
      produced += take;
      vorbis_synthesis_read(&vd, got);
    }
  }
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return produced;
}

/* ns streams on all host threads, samples counted only: stream s has npkt[s] audio packets from meta row
 * first[s]; returns the total samples per channel, or -1 */
long rds_stock_decode_many(int ns, const unsigned char *buf, const long *hdr, const long *meta, const long *first,
                           const long *npkt){
  long total = 0;
  int s, bad = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+:total) reduction(|:bad)
  for(s = 0; s < ns; s++){
    long r = rds_stock_decode(buf, hdr, meta + first[s] * META, npkt[s], 0, NULL, 0);
    if(r < 0) bad = 1; else total += r;
  }
  return bad ? -1 : total;
}

#ifdef VB200_DROPIN
typedef struct vb200md vb200md;
typedef void (*vb200md_sink)(void *user, int stream, const void *pcm, long samples);
vb200md *vb200md_open(int nstreams, ogg_packet hdr[3], int pcm_s16, int device);
int vb200md_packet(vb200md *m, int stream, const ogg_packet *op);
int vb200md_round(vb200md *m, vb200md_sink sink, void *user);
void vb200md_restart(vb200md *m, int stream);
void vb200md_close(vb200md *m);
int vb200md_channels(vb200md *m);
unsigned long long vb200md_launches(vb200md *m);
void vb200md_stats(vb200md *m, long *rounds, long *blocks, long *packets, double *device_s, double *host_s);

typedef struct { int s16, ch; long cap; void *out; long *len; int slot_of_stream_off; } md_out;

static void md_put(void *user, int stream, const void *pcm, long n){
  md_out *o = (md_out*)user;
  const int slot = stream + o->slot_of_stream_off;
  long at = o->len[slot], take = n, j;
  int c;
  if(o->out){
    if(at + take > o->cap) take = o->cap - at;
    for(c = 0; c < o->ch; c++)
      for(j = 0; j < take; j++){
        if(o->s16) ((int16_t*)o->out)[((size_t)slot * o->cap + at + j) * o->ch + c] = ((const int16_t*)pcm)[j * o->ch + c];
        else ((float*)o->out)[((size_t)slot * o->ch + c) * o->cap + at + j] = ((const float*)pcm)[(size_t)c * n + j];
      }
  }
  o->len[slot] += n;
}

/* ns streams through one driver.  sched [nrounds][ns]: packets fed to each stream before round r (after the
 * schedule: all that are left, one round).  restart >= 0: afterwards vb200md_restart(restart), all its packets
 * once more in one round, into slot ns of out / len.  out: float [ns+1][ch][cap] or int16 [ns+1][cap][ch]; NULL =
 * count only.  stats[0..5] = rounds, blocks, max launches of one round, launches of all rounds, device s, host s.
 * Returns 0 or < 0. */
long rds_md_run(int ns, const unsigned char *buf, const long *hdr, const long *meta, const long *first,
                const long *npkt, const int *sched, int nrounds, int s16, int device, int restart, void *out,
                long cap, long *len, double *stats){
  ogg_packet h[3];
  vb200md *m;
  md_out o;
  long *fed = (long*)calloc(ns, sizeof(long));
  long rounds = 0, blocks = 0, pk;
  unsigned long long lmax = 0, l0, lall = 0;
  int s, r, k, done = 0, rc = 0;
  double dev_s, host_s;
  for(k = 0; k < 3; k++) to_packet(&h[k], buf, hdr + k * META);
  m = vb200md_open(ns, h, s16, device);
  if(!m || !fed){ free(fed); return -1; }
  o.s16 = s16; o.ch = vb200md_channels(m); o.cap = cap; o.out = out; o.len = len; o.slot_of_stream_off = 0;
  for(s = 0; s <= ns; s++) len[s] = 0;
  for(r = 0; !done; r++){
    done = 1;
    for(s = 0; s < ns; s++){
      long want = r < nrounds ? sched[(size_t)r * ns + s] : npkt[s];
      for(k = 0; k < want && fed[s] < npkt[s]; k++, fed[s]++){
        ogg_packet op;
        to_packet(&op, buf, meta + (first[s] + fed[s]) * META);
        if(vb200md_packet(m, s, &op)){ rc = -1; goto out; }
      }
      if(fed[s] < npkt[s]) done = 0;
    }
    l0 = vb200md_launches(m);
    if((rc = vb200md_round(m, md_put, &o)) < 0) goto out;
    l0 = vb200md_launches(m) - l0;
    lall += l0;
    if(l0 > lmax) lmax = l0;
    rc = 0;
  }
  if(restart >= 0 && restart < ns){
    vb200md_restart(m, restart);
    for(pk = 0; pk < npkt[restart]; pk++){
      ogg_packet op;
      to_packet(&op, buf, meta + (first[restart] + pk) * META);
      if(vb200md_packet(m, restart, &op)){ rc = -1; goto out; }
    }
    o.slot_of_stream_off = ns - restart;
    if((rc = vb200md_round(m, md_put, &o)) < 0) goto out;
    rc = 0;
  }
out:
  vb200md_stats(m, &rounds, &blocks, &pk, &dev_s, &host_s);
  stats[0] = (double)rounds; stats[1] = (double)blocks; stats[2] = (double)lmax; stats[3] = (double)lall;
  stats[4] = dev_s; stats[5] = host_s;
  vb200md_close(m);
  free(fed);
  return rc;
}
#endif
