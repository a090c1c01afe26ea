/* ref_halfrate.c — half-rate decode through the UNMODIFIED reference sources.
 *
 * TEST INFRASTRUCTURE ONLY.  Compiled against the reference's headers and linked with the reference objects
 * oracle/Makefile builds (oracle/halfrate.py has the recipe):
 *   _ref/libvorbis_ref_halfrate.so     the stock reference (target `ref`'s objects)
 *   _ref/libvorbis_dropin_halfrate.so  the drop-in build, mapping0_inverse's mdct_backward bound to the CUDA
 *                                      shim (target `dropin`'s objects); compiled with -DVB200_DROPIN
 * refhs_encode runs the encoder API loop (as examples/encoder_example.c:210-235) and keeps every packet;
 * refhs_decode runs the decoder API loop on such packets (vorbis_synthesis, vorbis_synthesis_blockin,
 * vorbis_synthesis_pcmout), optionally after vorbis_synthesis_halfrate(&vi, 1) as ov_halfrate does.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"
#include "codec_internal.h"
#include "window.h"

#ifdef VB200_DROPIN
int vb200shim_attach(vorbis_dsp_state *vd, int device);
void vb200shim_detach(void);
#endif

static int keep(const ogg_packet *op, unsigned char *buf, long cap, long *off, long *sizes, int *n, int maxn){
  if(*n >= maxn || *off + op->bytes > cap) return -1;
  memcpy(buf + *off, op->packet, op->bytes);
  sizes[(*n)++] = op->bytes;
  *off += op->bytes;
  return 0;
}

/* pcm [ch][ns]; packets (3 headers, then audio) back to back in buf, their sizes in sizes[];
 * returns the packet count, or -1 (setup refused, buffers too small) */
int refhs_encode(int ch, long rate, float quality, const float *pcm, long ns,
                 unsigned char *buf, long cap, long *sizes, int maxn){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  ogg_packet hdr[3], op;
  long pos = 0, off = 0;
  int n = 0, i, eos = 0, bad = 0;
  vorbis_info_init(&vi);
  if(vorbis_encode_init_vbr(&vi, ch, rate, quality)){ vorbis_info_clear(&vi); return -1; }
  vorbis_comment_init(&vc);
  vorbis_analysis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  vorbis_analysis_headerout(&vd, &vc, &hdr[0], &hdr[1], &hdr[2]);
  for(i = 0; i < 3; i++) bad |= keep(&hdr[i], buf, cap, &off, sizes, &n, maxn);
  while(!eos && !bad){
    long todo = ns - pos < 1024 ? ns - pos : 1024;
    if(todo > 0){
      float **b = vorbis_analysis_buffer(&vd, (int)todo);
      for(i = 0; i < ch; i++) memcpy(b[i], pcm + (size_t)i*ns + pos, sizeof(float)*todo);
      vorbis_analysis_wrote(&vd, (int)todo);
      pos += todo;
    }else{
      vorbis_analysis_wrote(&vd, 0);
    }
    while(vorbis_analysis_blockout(&vd, &vb) == 1){
      vorbis_analysis(&vb, NULL);
      vorbis_bitrate_addblock(&vb);
      while(vorbis_bitrate_flushpacket(&vd, &op)){
        bad |= keep(&op, buf, cap, &off, sizes, &n, maxn);
        if(op.e_o_s) eos = 1;
      }
    }
    if(todo <= 0) eos = 1;
  }
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return bad ? -1 : n;
}

/* Decode npkt packets of refhs_encode.  halfrate: vorbis_synthesis_halfrate(&vi, 1) before
 * vorbis_synthesis_init; win0 / win1 (may be NULL) then receive the half windows the overlap-add uses,
 * _vorbis_window_get(b->window[w]-1) (lib/block.c:771-806), blocksizes[w]/4 floats each.
 * pcm_out [ch][pcm_cap]; Wseq[maxblocks] the block flags, *nblocks how many blocks were decoded.
 * Returns the samples produced per channel, or -1 (headers refused, half-rate refused, binding failed). */
long refhs_decode(const unsigned char *buf, const long *sizes, int npkt, int halfrate,
                  float *pcm_out, long pcm_cap, int32_t *Wseq, int maxblocks, int *nblocks,
                  float *win0, float *win1){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  long produced = 0, off = 0;
  int i, k, blocks = 0;
  vorbis_info_init(&vi); vorbis_comment_init(&vc);
  for(k = 0; k < npkt && k < 3; k++){
    ogg_packet hp;
    memset(&hp, 0, sizeof(hp));
    hp.packet = (unsigned char*)buf + off; hp.bytes = sizes[k]; hp.b_o_s = (k == 0); hp.packetno = k;
    off += sizes[k];
    if(vorbis_synthesis_headerin(&vi, &vc, &hp) < 0){ vorbis_comment_clear(&vc); vorbis_info_clear(&vi); return -1; }
  }
  if(halfrate && vorbis_synthesis_halfrate(&vi, 1)){ vorbis_comment_clear(&vc); vorbis_info_clear(&vi); return -1; }
  vorbis_synthesis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  if(halfrate){
    codec_setup_info *ci = (codec_setup_info*)vi.codec_setup;
    private_state *b = (private_state*)vd.backend_state;
    if(win0) memcpy(win0, _vorbis_window_get(b->window[0] - 1), sizeof(float)*(ci->blocksizes[0]/4));
    if(win1) memcpy(win1, _vorbis_window_get(b->window[1] - 1), sizeof(float)*(ci->blocksizes[1]/4));
  }
#ifdef VB200_DROPIN
  /* bind the decoder's own state after vorbis_synthesis_init, as an application of the shimmed library does */
  if(vb200shim_attach(&vd, 0)){
    vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
    return -1;
  }
#endif
  for(k = 3; k < npkt; k++){
    ogg_packet op; float **pcm; int got;
    memset(&op, 0, sizeof(op));
    op.packet = (unsigned char*)buf + off; op.bytes = sizes[k]; op.packetno = k; op.granulepos = -1;
    off += sizes[k];
    if(vorbis_synthesis(&vb, &op) == 0){
      if(Wseq && blocks < maxblocks) Wseq[blocks] = (int32_t)vb.W;
      vorbis_synthesis_blockin(&vd, &vb);
      blocks++;
    }
    while((got = vorbis_synthesis_pcmout(&vd, &pcm)) > 0){
      int take = got;
      if(produced + take > pcm_cap) take = (int)(pcm_cap - produced);
      for(i = 0; i < vi.channels; i++)
        if(take > 0) memcpy(pcm_out + (size_t)i*pcm_cap + produced, pcm[i], sizeof(float)*take);
      produced += take;
      vorbis_synthesis_read(&vd, got);
    }
  }
#ifdef VB200_DROPIN
  vb200shim_detach();
#endif
  if(nblocks) *nblocks = blocks < maxblocks ? blocks : maxblocks;
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return produced;
}
