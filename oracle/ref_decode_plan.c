/* ref_decode_plan.c — the stock decoder's state after every vorbis_synthesis_blockin.  TEST INFRASTRUCTURE ONLY.
 *
 *   rdsp_decode   the vorbis_synthesis -> vorbis_synthesis_blockin -> vorbis_synthesis_pcmout loop of
 *                 examples/decoder_example.c on the 3 header packets and npkt audio packets, at full rate or after
 *                 vorbis_synthesis_halfrate(vi, 1).  Per packet it records REC values:
 *                   status (what vorbis_synthesis returned), the block flag (-1 where dropped), the samples pcmout
 *                   returns, then v->granulepos, v->pcm_returned, v->pcm_current, v->sequence and b->sample_count
 *                   right after the blockin (as they stand where the packet was dropped);
 *                 and the PCM in pcmout order, float [ch][cap].  modebits: private_state.modebits.
 *
 * Packets live back to back in one byte buffer; meta rows are {offset, bytes, granulepos, e_o_s, packetno}.
 * oracle/Makefile links this file with the objects it compiles from the unmodified reference.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "codec_internal.h"

#define META 5
#define REC 8

static void to_packet(ogg_packet *op, const unsigned char *buf, const long *m){
  memset(op, 0, sizeof(*op));
  op->packet = (unsigned char*)buf + m[0]; op->bytes = m[1]; op->granulepos = m[2]; op->e_o_s = m[3];
  op->packetno = m[4]; op->b_o_s = (m[4] == 0);
}

/* returns the samples per channel, or -1 */
long rdsp_decode(const unsigned char *buf, const long *hdr, const long *audio, long npkt, int halfrate, float *out,
                 long cap, int64_t *rec, int *modebits){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  long produced = 0, k;
  int i;
  vorbis_info_init(&vi); vorbis_comment_init(&vc);
  for(k = 0; k < 3; k++){
    ogg_packet hp;
    to_packet(&hp, buf, hdr + k * META);
    if(vorbis_synthesis_headerin(&vi, &vc, &hp) < 0){ vorbis_comment_clear(&vc); vorbis_info_clear(&vi); return -1; }
  }
  if(halfrate && vorbis_synthesis_halfrate(&vi, 1)){ vorbis_comment_clear(&vc); vorbis_info_clear(&vi); return -1; }
  vorbis_synthesis_init(&vd, &vi);
  vorbis_block_init(&vd, &vb);
  *modebits = ((private_state*)vd.backend_state)->modebits;
  for(k = 0; k < npkt; k++){
    ogg_packet op; float **pcm; int got, st;
    int64_t *r = rec + k * REC;
    to_packet(&op, buf, audio + k * META);
    st = vorbis_synthesis(&vb, &op);
    if(st == 0) vorbis_synthesis_blockin(&vd, &vb);
    r[0] = st; r[1] = st == 0 ? vb.W : -1; r[2] = 0;
    r[3] = vd.granulepos; r[4] = vd.pcm_returned; r[5] = vd.pcm_current; r[6] = vd.sequence;
    r[7] = ((private_state*)vd.backend_state)->sample_count;
    while((got = vorbis_synthesis_pcmout(&vd, &pcm)) > 0){
      long j;
      r[2] += got;
      for(i = 0; i < vi.channels; i++)
        for(j = 0; j < got && produced + j < cap; j++) out[(size_t)i * cap + produced + j] = pcm[i][j];
      produced += got;
      vorbis_synthesis_read(&vd, got);
    }
  }
  vorbis_block_clear(&vb); vorbis_dsp_clear(&vd); vorbis_comment_clear(&vc); vorbis_info_clear(&vi);
  return produced;
}
