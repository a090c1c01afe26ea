/* ref_bitrate.c — checkers of the device bitrate manager and of whole streams' packets.  TEST INFRASTRUCTURE ONLY.
 *
 *   ref_bitrate_info    ci->bi and the block sizes of an encoder opened from an rbr_config
 *   ref_bitrate_replay  the UNMODIFIED vorbis_bitrate_addblock / vorbis_bitrate_flushpacket of a real managed
 *                       vorbis_dsp_state on given packet lengths: packetblob[0..14] of each block are filled with
 *                       pseudo-random bits of those lengths; per block it returns bm->choice, the flushed packet's
 *                       length, whether its bytes are the kept blob's first bytes followed by zero bytes, and the
 *                       state after the block
 *   ref_stream_capture  a stock encoder (VBR quality or managed) on one stream through the API loop of
 *                       examples/encoder_example.c: the timeline and eof as ref_driver.c's ref_encode_capture records
 *                       them, and every audio packet with its granulepos, e_o_s and packetno
 *   (-DVB200_DROPIN, linked with the multi-stream driver)
 *   rbr_open_managed / rbr_ctx / rbr_close   a vb200ms_open_managed'd driver, whose context carries the setup and the
 *                                            entropy setup of the managed encoder
 *
 * oracle/bitrate.py links this file with the stock reference objects, and once more with the driver and the drop-in
 * objects.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"
#include "codec_internal.h"
#include "bitrate.h"

#include "vorbis_b200.h"

/* how an encoder is opened: mode 0 vorbis_encode_init_vbr(quality); 1 vorbis_encode_setup_managed(max, nominal, min),
 * then with rm2 != 0 OV_ECTL_RATEMANAGE2_SET with the reservoir bits, bias and average damping replaced, then
 * vorbis_encode_setup_init (what vorbis_encode_init does when rm2 == 0) */
typedef struct rbr_config {
  int32_t mode, channels;
  int64_t rate;
  double quality;
  int64_t max_br, nominal_br, min_br;
  int32_t rm2, pad;
  int64_t rm2_reservoir_bits;
  double rm2_bias, rm2_damp;
} rbr_config;

#ifndef VB200_DROPIN
static int rbr_open(const rbr_config *cf, vorbis_info *vi){
  vorbis_info_init(vi);
  if(cf->mode == 0){
    if(vorbis_encode_init_vbr(vi, cf->channels, cf->rate, (float)cf->quality)) goto bad;
    return 0;
  }
  if(vorbis_encode_setup_managed(vi, cf->channels, cf->rate, cf->max_br, cf->nominal_br, cf->min_br)) goto bad;
  if(cf->rm2){
    struct ovectl_ratemanage2_arg a;
    if(vorbis_encode_ctl(vi, OV_ECTL_RATEMANAGE2_GET, &a)) goto bad;
    a.bitrate_limit_reservoir_bits = cf->rm2_reservoir_bits;
    a.bitrate_limit_reservoir_bias = cf->rm2_bias;
    a.bitrate_average_damping = cf->rm2_damp;
    if(vorbis_encode_ctl(vi, OV_ECTL_RATEMANAGE2_SET, &a)) goto bad;
  }
  if(vorbis_encode_setup_init(vi)) goto bad;
  return 0;
bad:
  vorbis_info_clear(vi);
  return -1;
}

int ref_bitrate_info(const rbr_config *cf, vb200_bitrate_info *out, int32_t *bs){
  vorbis_info vi;
  codec_setup_info *ci;
  if(rbr_open(cf, &vi)) return -1;
  ci = (codec_setup_info*)vi.codec_setup;
  out->avg_rate = ci->bi.avg_rate; out->min_rate = ci->bi.min_rate; out->max_rate = ci->bi.max_rate;
  out->reservoir_bits = ci->bi.reservoir_bits; out->reservoir_bias = ci->bi.reservoir_bias;
  out->slew_damp = ci->bi.slew_damp;
  bs[0] = (int32_t)ci->blocksizes[0]; bs[1] = (int32_t)ci->blocksizes[1];
  vorbis_info_clear(&vi);
  return 0;
}

static uint8_t content_byte(uint64_t seed, long blk, int k, long j){
  uint64_t x = seed * 0x9E3779B97F4A7C15ULL ^ ((uint64_t)blk << 20) ^ ((uint64_t)k << 52) ^ (uint64_t)j;
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
  return (uint8_t)x;
}

/* nseq sequences of len[i] blocks, each from a fresh vorbis_bitrate_init state: W [total], bits [total][15];
 * per block choice, bytes, ok (1: the flushed packet is the kept blob's first bytes, then zero bytes) and the state
 * after it.  Returns 0, or -1 when the encoder cannot be opened or is not managed. */
int ref_bitrate_replay(const rbr_config *cf, uint64_t seed, int nseq, const int32_t *len, const int32_t *W,
                       const int32_t *bits, int32_t *choice, int64_t *bytes, int32_t *ok, vb200_bitrate_state *after){
  vorbis_info vi; vorbis_dsp_state vd; vorbis_block vb;
  private_state *b;
  long t = 0;
  int i, rc = 0;
  if(rbr_open(cf, &vi)) return -1;
  vorbis_analysis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  b = (private_state*)vd.backend_state;
  if(!b->bms.managed) rc = -1;
  for(i = 0; i < nseq && !rc; i++){
    int k;
    vorbis_bitrate_init(&vi, &b->bms);
    for(k = 0; k < len[i]; k++, t++){
      vorbis_block_internal *vbi = (vorbis_block_internal*)vb.internal;
      ogg_packet op;
      int c;
      long j;
      vb.W = W[t];
      for(c = 0; c < VB200_PACKETBLOBS; c++){
        oggpack_buffer *o = vbi->packetblob[c];
        const long nbits = bits[t * VB200_PACKETBLOBS + c];
        oggpack_reset(o);
        for(j = 0; j < nbits / 8; j++) oggpack_write(o, content_byte(seed, t, c, j), 8);
        if(nbits & 7) oggpack_write(o, content_byte(seed, t, c, j), (int)(nbits & 7));
      }
      vorbis_bitrate_addblock(&vb);
      choice[t] = b->bms.choice;
      after[t].avg_reservoir = b->bms.avg_reservoir;
      after[t].minmax_reservoir = b->bms.minmax_reservoir;
      after[t].avgfloat = b->bms.avgfloat;
      after[t].choice = b->bms.choice;
      after[t].pad = 0;
      if(vorbis_bitrate_flushpacket(&vd, &op) != 1){ rc = -1; break; }
      bytes[t] = op.bytes;
      {
        const long nb = bits[t * VB200_PACKETBLOBS + choice[t]];
        const long natural = (nb + 7) / 8;
        int good = 1;
        for(j = 0; j < op.bytes && good; j++){
          uint8_t want = 0;
          if(j < natural){
            want = content_byte(seed, t, choice[t], j);
            if(j == nb / 8 && (nb & 7)) want &= (uint8_t)((1u << (nb & 7)) - 1);
          }
          good = op.packet[j] == want;
        }
        ok[t] = good;
      }
    }
  }
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_info_clear(&vi);
  return rc;
}

/* pcm [ch][nsamples] through a fresh stock encoder in chunk-sample writes (0: 1024), then vorbis_analysis_wrote(0).
 * tl [ch][tl_cap]: v->pcm re-assembled in timeline samples (preamble, input, extrapolated tail); *tl_len, *eof as
 * ref_encode_capture reports them.  Audio packets back to back into out (cap bytes) with bytes, granulepos, e_o_s
 * and packetno each [maxn].  Returns the packet count, or < 0. */
long ref_stream_capture(const rbr_config *cf, const float *pcm, long nsamples, long chunk, float *tl, long tl_cap,
                        int64_t *tl_len, int64_t *eof_out, uint8_t *out, long cap, int64_t *bytes, int64_t *granulepos,
                        int32_t *eos, int64_t *packetno, long maxn){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  ogg_packet h0, h1, h2, op;
  long pos = 0, at = 0, np = 0, shift = 0, len = 0, eof = 0;
  int done = 0, i, rc = 0;
  if(chunk <= 0) chunk = 1024;
  if(rbr_open(cf, &vi)) return -1;
  vorbis_comment_init(&vc);
  vorbis_analysis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  vorbis_analysis_headerout(&vd, &vc, &h0, &h1, &h2);
  while(!done && !rc){
    const long todo = nsamples - pos < chunk ? nsamples - pos : chunk;
    if(todo > 0){
      float **buf = vorbis_analysis_buffer(&vd, (int)todo);
      for(i = 0; i < cf->channels; i++) memcpy(buf[i], pcm + (size_t)i * nsamples + pos, sizeof(float) * todo);
      vorbis_analysis_wrote(&vd, (int)todo);
      pos += todo;
    }else vorbis_analysis_wrote(&vd, 0);
    {
      long k; int c;
      for(c = 0; c < cf->channels; c++)
        for(k = 0; k < vd.pcm_current; k++)
          if(shift + k < tl_cap) tl[(size_t)c * tl_cap + shift + k] = vd.pcm[c][k];
      if(shift + vd.pcm_current > len) len = shift + vd.pcm_current;
      if(vd.eofflag > 0 && !eof) eof = shift + vd.eofflag;
    }
    while(!rc){
      const long pc_before = vd.pcm_current;
      if(vorbis_analysis_blockout(&vd, &vb) != 1) break;
      shift += pc_before - vd.pcm_current;
      vorbis_analysis(&vb, NULL);
      vorbis_bitrate_addblock(&vb);
      while(vorbis_bitrate_flushpacket(&vd, &op)){
        if(np >= maxn || at + op.bytes > cap){ rc = -2; break; }
        memcpy(out + at, op.packet, op.bytes);
        at += op.bytes;
        bytes[np] = op.bytes; granulepos[np] = op.granulepos; eos[np] = (int32_t)op.e_o_s; packetno[np] = op.packetno;
        np++;
        if(op.e_o_s) done = 1;
      }
    }
    if(todo <= 0) done = 1;
  }
  *tl_len = len; *eof_out = eof;
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return rc ? rc : np;
}
#endif

#ifdef VB200_DROPIN
typedef struct vb200ms vb200ms;
vb200ms *vb200ms_open_managed(int nstreams, int channels, long rate, long max_br, long nominal_br, long min_br, int device);
void vb200ms_close(vb200ms *m);
int vb200ms_entropy_on_device(vb200ms *m);
vb200_ctx *vb200ms_context(vb200ms *m);

void *rbr_open_managed(int ch, long rate, long max_br, long nominal_br, long min_br, int device){
  vb200ms *m = vb200ms_open_managed(1, ch, rate, max_br, nominal_br, min_br, device);
  if(m && !vb200ms_entropy_on_device(m)){ vb200ms_close(m); m = NULL; }
  return m;
}
void *rbr_ctx(void *m){ return vb200ms_context((vb200ms*)m); }
void rbr_close(void *m){ vb200ms_close((vb200ms*)m); }
#endif
