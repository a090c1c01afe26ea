/* ref_encode_managed.c — the managed multi-stream driver with its entropy path chosen.  TEST INFRASTRUCTURE ONLY.
 *
 *   rep_ms_encode_managed   (-DVB200_DROPIN) ref_managed.c's ref_ms_encode_managed with the host entropy path forced
 *                           (host_entropy = 1), or left as the driver chooses it (0); reports the path it took, as
 *                           ref_encode_packets.c's rep_ms_encode does
 *
 * oracle/encode_managed.py links this file with the managed multi-stream driver and the drop-in objects.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"

#ifdef VB200_DROPIN
typedef struct vb200ms vb200ms;
typedef void (*vb200ms_sink)(void *user, int stream, ogg_packet *op);
vb200ms *vb200ms_open_managed(int nstreams, int channels, long rate, long max_br, long nominal_br, long min_br, int device);
void vb200ms_close(vb200ms *m);
vorbis_dsp_state *vb200ms_state(vb200ms *m, int stream);
int vb200ms_round(vb200ms *m, vb200ms_sink sink, void *user);
int vb200ms_entropy_on_device(vb200ms *m);
void vb200ms_set_host_entropy(vb200ms *m, int on);
unsigned long long vb200shim_launches(void);

typedef struct { uint64_t *hash; long *bytes, *count; } rem_sum;
static void rem_sink(void *user, int stream, ogg_packet *op){       /* the summary of ref_managed.c's mg_sink */
  rem_sum *s = (rem_sum*)user;
  long k;
  uint64_t h = s->hash[stream];
  for(k = 0; k < op->bytes; k++){ h ^= op->packet[k]; h *= 1099511628211ULL; }
  h ^= (uint64_t)op->bytes; h *= 1099511628211ULL;
  s->hash[stream] = h; s->bytes[stream] += op->bytes; s->count[stream]++;
}

/* pcm [nstreams][ch][nsamples] in 1024-sample writes; returns the total number of blocks (or < 0), in *rounds the
 * rounds that processed blocks, in *launches the device kernel launches of the run, in *on_device the path taken */
long rep_ms_encode_managed(int nstreams, int ch, long rate, long max_br, long nominal_br, long min_br, int device,
                           int host_entropy, const float *pcm, long nsamples, uint64_t *hash, long *bytes, long *count,
                           long *rounds, unsigned long long *launches, int *on_device){
  vb200ms *m = vb200ms_open_managed(nstreams, ch, rate, max_br, nominal_br, min_br, device);
  rem_sum sum;
  long pos = 0, blocks = 0;
  int i, c, r, done = 0;
  if(!m) return -1;
  vb200ms_set_host_entropy(m, host_entropy);
  *on_device = vb200ms_entropy_on_device(m);
  for(i = 0; i < nstreams; i++){ hash[i] = 1469598103934665603ULL; bytes[i] = 0; count[i] = 0; }
  sum.hash = hash; sum.bytes = bytes; sum.count = count;
  *rounds = 0;
  *launches = vb200shim_launches();
  while(!done){
    const long todo = nsamples - pos < 1024 ? nsamples - pos : 1024;
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
    while((r = vb200ms_round(m, rem_sink, &sum)) > 0){ blocks += r; (*rounds)++; }
    if(r < 0){ blocks = r; break; }
  }
  *launches = vb200shim_launches() - *launches;
  vb200ms_close(m);
  return blocks;
}
#endif
