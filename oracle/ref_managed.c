/* ref_managed.c — bitrate-managed encoder runs for the tests, summarised per stream as (packet count, bytes,
 * FNV-1a hash of all packet bytes in order), the summary of ref_driver.c's ref_stock_encode_summary / ref_ms_encode.
 * TEST INFRASTRUCTURE ONLY.
 *
 *   ref_managed_stock_summary  ONE stock encoder from vorbis_encode_init (max / nominal / min bitrate, -1 = unset):
 *                              the reference's own API loop with vorbis_bitrate_addblock / flushpacket
 *   ref_ms_encode_managed      (-DVB200_DROPIN) N encoders of that configuration through the managed multi-stream
 *                              driver of vorbis_b200/host/vb200_mapping0.c (vb200ms_open_managed), fed in lockstep
 *
 * Both feed 1024-sample writes.  oracle/managed.py links this file with the objects oracle/Makefile compiles from
 * the unmodified reference sources.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"

#define CHUNK 1024

typedef struct { uint64_t *hash; long *bytes, *count; } mg_sum;

static void mg_sink(void *user, int stream, ogg_packet *op){
  mg_sum *s = (mg_sum*)user;
  long k;
  uint64_t h = s->hash[stream];
  for(k = 0; k < op->bytes; k++){ h ^= op->packet[k]; h *= 1099511628211ULL; }
  h ^= (uint64_t)op->bytes; h *= 1099511628211ULL;
  s->hash[stream] = h; s->bytes[stream] += op->bytes; s->count[stream]++;
}

/* pcm [ch][nsamples]; returns the number of blocks, or < 0 */
long ref_managed_stock_summary(int ch, long rate, long max_br, long nominal_br, long min_br, const float *pcm,
                               long nsamples, uint64_t *hash, long *bytes, long *count){
  vorbis_info vi;
  vorbis_dsp_state vd;
  vorbis_block vb;
  ogg_packet op;
  mg_sum sum;
  long pos = 0, blocks = 0;
  int i, done = 0;
  vorbis_info_init(&vi);
  if(vorbis_encode_init(&vi, ch, rate, max_br, nominal_br, min_br)){ vorbis_info_clear(&vi); return -1; }
  vorbis_analysis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  *hash = 1469598103934665603ULL; *bytes = 0; *count = 0;
  sum.hash = hash; sum.bytes = bytes; sum.count = count;
  while(!done){
    const long todo = nsamples - pos < CHUNK ? nsamples - pos : CHUNK;
    if(todo > 0){
      float **buf = vorbis_analysis_buffer(&vd, (int)todo);
      for(i = 0; i < ch; i++) memcpy(buf[i], pcm + (size_t)i*nsamples + pos, sizeof(float)*todo);
      vorbis_analysis_wrote(&vd, (int)todo);
      pos += todo;
    }else{
      vorbis_analysis_wrote(&vd, 0);
      done = 1;
    }
    while(vorbis_analysis_blockout(&vd, &vb) == 1){
      vorbis_analysis(&vb, NULL);
      vorbis_bitrate_addblock(&vb);
      while(vorbis_bitrate_flushpacket(&vd, &op)) mg_sink(&sum, 0, &op);
      blocks++;
    }
  }
  vorbis_block_clear(&vb);
  vorbis_dsp_clear(&vd);
  vorbis_info_clear(&vi);
  return blocks;
}

#ifdef VB200_DROPIN
typedef struct vb200ms vb200ms;
typedef void (*vb200ms_sink)(void *user, int stream, ogg_packet *op);
vb200ms *vb200ms_open_managed(int nstreams, int channels, long rate, long max_br, long nominal_br, long min_br, int device);
void vb200ms_close(vb200ms *m);
vorbis_dsp_state *vb200ms_state(vb200ms *m, int stream);
int vb200ms_round(vb200ms *m, vb200ms_sink sink, void *user);
unsigned long long vb200shim_launches(void);

/* pcm [nstreams][ch][nsamples]; returns the total number of blocks (or < 0), in *rounds the driver rounds that
 * processed blocks and in *launches the device kernel launches of the whole run */
long ref_ms_encode_managed(int nstreams, int ch, long rate, long max_br, long nominal_br, long min_br, int device,
                           const float *pcm, long nsamples, uint64_t *hash, long *bytes, long *count, long *rounds,
                           unsigned long long *launches){
  vb200ms *m = vb200ms_open_managed(nstreams, ch, rate, max_br, nominal_br, min_br, device);
  mg_sum sum;
  long pos = 0, blocks = 0;
  int i, c, r, done = 0;
  if(!m) return -1;
  for(i = 0; i < nstreams; i++){ hash[i] = 1469598103934665603ULL; bytes[i] = 0; count[i] = 0; }
  sum.hash = hash; sum.bytes = bytes; sum.count = count;
  *rounds = 0;
  *launches = vb200shim_launches();
  while(!done){
    const long todo = nsamples - pos < CHUNK ? nsamples - pos : CHUNK;
    for(i = 0; i < nstreams; i++){
      vorbis_dsp_state *vd = vb200ms_state(m, i);
      if(todo > 0){
        float **buf = vorbis_analysis_buffer(vd, (int)todo);
        for(c = 0; c < ch; c++) memcpy(buf[c], pcm + ((size_t)i*ch + c)*nsamples + pos, sizeof(float)*todo);
        vorbis_analysis_wrote(vd, (int)todo);
      }else vorbis_analysis_wrote(vd, 0);
    }
    if(todo > 0) pos += todo;
    else done = 1;
    while((r = vb200ms_round(m, mg_sink, &sum)) > 0){ blocks += r; (*rounds)++; }
    if(r < 0){ blocks = r; break; }
  }
  *launches = vb200shim_launches() - *launches;
  vb200ms_close(m);
  return blocks;
}
#endif
