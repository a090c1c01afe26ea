/* vb_oracle_resume.c — the carried block planner restated in plain C (libvb_oracle_resume.so).  TEST INFRASTRUCTURE
 * ONLY: the CPU reference of k_env_marks_carry and k_plan_blocks_carry (vorbis_b200/csrc/vb200_streams.cuh).
 *
 * One call plans one stream's blocks on a buffer whose sample 0 is timeline sample c->base, the way repeated
 * vorbis_analysis_blockout calls do (lib/block.c:534-689) on a vorbis_dsp_state that has been carried along:
 *   - the marks are ve->mark as the reference keeps it: the carried window (what _ve_envelope_shift left, current/64 +
 *     VE_POST entries), then lib/envelope.c:254-264 replayed step by step over this call's trigger bits (the steps
 *     first = current/64 .. last-1 of the buffer, last = pcm_len/64 - VE_WIN, analysed by the caller with the carried
 *     envelope state); the device computes the same marks in closed form;
 *   - the cursor / curmark walk of _ve_envelope_search (:269-327), _ve_envelope_mark (:329-356) and the block sizes,
 *     with eofflag = eof - base (eof 0: no EOF yet);
 *   - after every block the re-basing of lib/block.c:654-686 and _ve_envelope_shift (lib/envelope.c:358-379).
 * At the end the carry holds the state of the stream's vorbis_dsp_state in the next buffer's coordinates and the mark
 * window the reference keeps.  Returns the number of blocks, or -1 when that window would not fit `cap` entries. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis_b200.h"

typedef struct vbo_carry {
  int64_t base;        /* timeline sample of this buffer's sample 0 (the sum of movementW) */
  int64_t kept;        /* v->pcm_current after the last block */
  int64_t centerW, cursor, curmark, current;
  int32_t W, lW, done, pad;
} vbo_carry;

void vbo_carry_init(int bs1, vbo_carry *c){
  memset(c, 0, sizeof(*c));
  c->centerW = c->cursor = bs1 / 2;                  /* _vds_shared_init; _ve_envelope_init (calloc) */
}

int vbo_plan_blocks_resume(int bs0_, int bs1_, vbo_carry *c, uint8_t *window, int cap, const uint8_t *ret, int count,
                           int64_t pcm_len, int64_t eof, int max_blocks, vb200_stream_block *plan){
  const long bs[2] = {bs0_, bs1_}, step = 64;
  const long first = c->current / step;
  long last = pcm_len / step - 4, j, nmark, i;
  long lW = c->lW, W = c->W, nW = 0;
  long centerW = c->centerW, cursor = c->cursor, curmark = c->curmark, shift = 0;
  long pcm_current = pcm_len, current;
  long eofflag = eof ? eof - c->base : 0;
  int nb = 0;
  int32_t *m;
  if(c->done) return 0;
  if(last < first) last = first;
  current = last * step;                             /* ve->current = last*searchstep */
  nmark = last + 4;
  m = calloc((size_t)nmark, sizeof(*m));
  for(i = 0; i < first + 2 && i < cap; i++) m[i] = window[i];
  for(j = first; j < first + count; j++){             /* lib/envelope.c:254-264 */
    const int r = ret[j - first];
    m[j + 2] = 0;
    if(r & 1){ m[j] = 1; m[j + 1] = 1; }
    if(r & 2){ m[j] = 1; if(j > 0) m[j - 1] = 1; }
  }
  while(nb < max_blocks){
    long bp = -1, centerNext, movementW;
    int blocktype;
    if(eofflag == -1) break;                          /* lib/block.c:547 */
    {
      const long testW = centerW + bs[W] / 4 + bs[1] / 2 + bs[0] / 4;
      for(j = cursor; j < current - step; j += step){ /* lib/envelope.c:269-327 */
        if(j >= testW){ bp = 1; break; }
        cursor = j;
        if(m[(j + shift) / step] && j > centerW){
          curmark = j;
          bp = j >= testW ? 1 : 0;
          break;
        }
      }
    }
    if(bp == -1){
      if(eofflag == 0) break;
      nW = 0;
    }else nW = bs[0] == bs[1] ? 0 : bp;
    centerNext = centerW + bs[W] / 4 + bs[nW] / 4;
    if(pcm_current < centerNext + bs[nW] / 2) break;
    if(W) blocktype = (!lW || !nW) ? 0 : 1;
    else{
      const long beginW = centerW - bs[0] / 2, endW = centerW + bs[0] / 2;
      int hit = curmark >= beginW && curmark < endW;
      for(i = beginW / step; !hit && i < endW / step; i++) hit = m[i + shift / step] != 0;
      blocktype = hit ? 0 : 1;
    }
    plan[nb].pos = (int32_t)(shift + centerW - bs[W] / 2);
    plan[nb].slot = 0;
    plan[nb].W = (int32_t)W; plan[nb].lW = (int32_t)lW; plan[nb].nW = (int32_t)nW; plan[nb].blocktype = blocktype;
    nb++;
    if(eofflag && centerW >= eofflag){ eofflag = -1; break; }
    movementW = centerNext - bs[1] / 2;
    if(movementW > 0){
      current -= movementW;                           /* _ve_envelope_shift */
      if(curmark >= 0) curmark -= movementW;
      cursor -= movementW;
      pcm_current -= movementW;
      shift += movementW;
      lW = W; W = nW; centerW = bs[1] / 2;
      if(eofflag){
        eofflag -= movementW;
        if(eofflag <= 0) eofflag = -1;
      }
    }
  }
  c->done = eofflag == -1;
  if(!c->done){
    const long keep = current / step + 2;            /* smallsize of _ve_envelope_shift */
    if(keep > cap){ free(m); return -1; }
    for(i = 0; i < cap; i++) window[i] = i < keep && m[i + shift / step] ? 1 : 0;
  }
  c->base += shift; c->kept = pcm_current;
  c->centerW = centerW; c->cursor = cursor; c->curmark = curmark; c->current = current;
  c->W = (int32_t)W; c->lW = (int32_t)lW;
  free(m);
  return nb;
}
