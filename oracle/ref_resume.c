/* ref_resume.c — the unmodified reference's planner state after every vorbis_analysis_blockout.  TEST INFRASTRUCTURE
 * ONLY (oracle/resume.py links it with the stock reference objects that oracle/Makefile compiles).
 *
 *   ref_resume_capture  a stock VBR encoder on one stream, written in chunks of `chunk` samples then
 *                       vorbis_analysis_wrote(v, 0), with the blockout loop of examples/encoder_example.c after every
 *                       write.  Records the timeline it saw (as ref_bitrate.c's ref_stream_capture), its eof, the
 *                       timeline end after every write, and after every blockout that returned a block:
 *                       rec[k][0..11) = write index, base (the sum of movementW so far), ve->current, ve->cursor,
 *                       ve->curmark, v->pcm_current, v->centerW, v->W, v->lW, vb->nW, the block's blocktype.
 *                       Returns the number of blocks, or -1. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"
#include "codec_internal.h"
#include "envelope.h"

#define REC 11

long ref_resume_capture(int channels, long rate, double quality, const float *pcm, long nsamples, long chunk,
                        float *tl, long tl_cap, int64_t *tl_len, int64_t *eof_out, int64_t *write_end, long max_writes,
                        int64_t *rec, long maxn){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  ogg_packet h0, h1, h2;
  long pos = 0, nb = 0, shift = 0, len = 0, eof = 0, w = 0;
  int done = 0, i;
  if(chunk <= 0) chunk = nsamples > 0 ? nsamples : 1;
  vorbis_info_init(&vi);
  if(vorbis_encode_init_vbr(&vi, channels, rate, (float)quality)) return -1;
  vorbis_comment_init(&vc);
  vorbis_analysis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  vorbis_analysis_headerout(&vd, &vc, &h0, &h1, &h2);
  while(!done){
    const long todo = nsamples - pos < chunk ? nsamples - pos : chunk;
    private_state *b = vd.backend_state;
    if(todo > 0){
      float **buf = vorbis_analysis_buffer(&vd, (int)todo);
      for(i = 0; i < channels; i++) memcpy(buf[i], pcm + (size_t)i * nsamples + pos, sizeof(float) * todo);
      vorbis_analysis_wrote(&vd, (int)todo);
      pos += todo;
    }else vorbis_analysis_wrote(&vd, 0);
    {
      long k; int c;
      for(c = 0; c < channels; c++)
        for(k = 0; k < vd.pcm_current; k++)
          if(shift + k < tl_cap) tl[(size_t)c * tl_cap + shift + k] = vd.pcm[c][k];
      if(shift + vd.pcm_current > len) len = shift + vd.pcm_current;
      if(vd.eofflag > 0 && !eof) eof = shift + vd.eofflag;
    }
    if(w >= max_writes || nb >= maxn) return -1;
    write_end[w] = shift + vd.pcm_current;
    for(;;){
      const long pc_before = vd.pcm_current;
      int64_t *r;
      if(vorbis_analysis_blockout(&vd, &vb) != 1) break;
      shift += pc_before - vd.pcm_current;
      if(nb >= maxn) return -1;
      r = rec + (size_t)nb * REC;
      r[0] = w; r[1] = shift; r[2] = b->ve->current; r[3] = b->ve->cursor; r[4] = b->ve->curmark;
      r[5] = vd.pcm_current; r[6] = vd.centerW; r[7] = vd.W; r[8] = vd.lW; r[9] = vb.nW;
      r[10] = ((vorbis_block_internal *)vb.internal)->blocktype;
      nb++;
      vorbis_analysis(&vb, NULL);
    }
    w++;
    if(todo <= 0) done = 1;
  }
  *tl_len = len; *eof_out = eof;
  vorbis_block_clear(&vb);
  vorbis_dsp_clear(&vd);
  vorbis_comment_clear(&vc);
  vorbis_info_clear(&vi);
  return nb;
}
