/* ref_headers.c — the reference's reading of three header packets.  TEST INFRASTRUCTURE ONLY.
 *
 *   rh_open     vorbis_synthesis_headerin on the identification (b_o_s), comment and setup packets, then
 *               vorbis_synthesis_init.  *rc = the first nonzero code (OV_*; a vorbis_synthesis_init failure is
 *               OV_EBADHEADER) or 0, and RH_HANGS where init would not return (a maptype-1 book of dimension 0 with
 *               entries: _book_maptype1_quantvals never ends for it).  On 0, *eimpl = what the decoder state shows
 *               the vb200 structs cannot describe (bit 0: not two modes of block flags 0 and 1; bit 1: a submap of
 *               either mode on a floor of type 0; bit 2: more than VB200_MAX_SUBMAPS submaps; bit 3: a book whose
 *               dimension is outside 1..127; bit 4: more codewords or value rows than VB200_HEADERS_MAX_*), and
 *               where that is 0 the handle carries vb200md_setup's vb200_setup and vb200md_entropy_new's vb200_entropy_setup (vorbis_b200/host/vb200_decode.c) of the decoder.
 *   rh_setup / rh_entropy / rh_modebits / rh_info / rh_close
 * oracle/Makefile links this file with the stock reference objects and the driver.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "codec_internal.h"
#include "backends.h"
#include "registry.h"
#include "misc.h"

#include "vorbis_b200.h"

#define RH_HANGS (-1000)

int vb200md_setup(vorbis_info *vi, vorbis_dsp_state *vd, vb200_setup *s);
vb200_entropy_setup *vb200md_entropy_new(vorbis_info *vi, vorbis_dsp_state *vd, int *err);
void vb200md_entropy_free(vb200_entropy_setup *es);

typedef struct {
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd;
  int init;
  vb200_setup s;
  vb200_entropy_setup *es;
} rh;

void rh_close(rh *h){
  if(!h) return;
  if(h->es) vb200md_entropy_free(h->es);
  if(h->init) vorbis_dsp_clear(&h->vd);
  vorbis_comment_clear(&h->vc);
  vorbis_info_clear(&h->vi);
  free(h);
}

static int rh_eimpl(rh *h){
  codec_setup_info *ci = (codec_setup_info*)h->vi.codec_setup;
  int why = 0, w, j, i;
  long rows = 0, values = 0;
  for(i = 0; i < ci->books; i++){
    const dec_codebook *db = ci->decbooks + i;
    /* the codewords md_book_codewords lists */
    const long n = !db->codelist ? 0 : db->codelengths ? (db->hi_max > 0 ? db->hi_max : 1) : db->entries;
    if(db->dim < 1 || db->dim > 127) why |= 8;
    rows += n;
    if(db->valuelist) values += n * db->dim;
  }
  if(rows > VB200_HEADERS_MAX_CODEWORDS || values > VB200_HEADERS_MAX_VALUES) why |= 16;
  if(ci->modes != 2 || ci->mode_param[0]->blockflag != 0 || ci->mode_param[1]->blockflag != 1) return why | 1;
  for(w = 0; w < 2; w++){
    vorbis_info_mapping0 *mp = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[w]->mapping];
    if(mp->submaps > VB200_MAX_SUBMAPS){ why |= 4; continue; }
    for(j = 0; j < mp->submaps; j++)
      if(ci->floor_type[mp->floorsubmap[j]] != 1) why |= 2;
  }
  return why;
}

rh *rh_open(const unsigned char *id, long id_bytes, const unsigned char *cm, long cm_bytes,
            const unsigned char *st, long st_bytes, int *rc, int *eimpl){
  rh *h = (rh*)calloc(1, sizeof(*h));
  const unsigned char *pk[3] = {id, cm, st};
  const long n[3] = {id_bytes, cm_bytes, st_bytes};
  codec_setup_info *ci;
  int k, e;
  *eimpl = 0;
  vorbis_info_init(&h->vi);
  vorbis_comment_init(&h->vc);
  for(k = 0; k < 3; k++){
    ogg_packet op;
    memset(&op, 0, sizeof(op));
    op.packet = (unsigned char*)pk[k]; op.bytes = n[k]; op.b_o_s = k == 0; op.packetno = k;
    if((*rc = vorbis_synthesis_headerin(&h->vi, &h->vc, &op)) != 0){ rh_close(h); return NULL; }
  }
  ci = (codec_setup_info*)h->vi.codec_setup;
  for(k = 0; k < ci->books; k++)
    if(ci->decbooks[k].maptype == 1 && ci->decbooks[k].dim == 0 && ci->decbooks[k].entries > 0){
      *rc = RH_HANGS; rh_close(h); return NULL;
    }
  if(vorbis_synthesis_init(&h->vd, &h->vi)){ *rc = OV_EBADHEADER; rh_close(h); return NULL; }
  h->init = 1;
  *rc = 0;
  if((*eimpl = rh_eimpl(h)) != 0) return h;
  if((e = vb200md_setup(&h->vi, &h->vd, &h->s)) != 0){ *rc = e; rh_close(h); return NULL; }
  h->es = vb200md_entropy_new(&h->vi, &h->vd, &e);
  if(!h->es){ *rc = e ? e : -1; rh_close(h); return NULL; }
  return h;
}

vb200_setup *rh_setup(rh *h){ return h->es ? &h->s : NULL; }
vb200_entropy_setup *rh_entropy(rh *h){ return h->es; }
int rh_modebits(rh *h){ return ((private_state*)h->vd.backend_state)->modebits; }
/* channels, rate, bitrate upper, nominal, lower */
void rh_info(rh *h, long *out){
  out[0] = h->vi.channels; out[1] = h->vi.rate; out[2] = h->vi.bitrate_upper; out[3] = h->vi.bitrate_nominal;
  out[4] = h->vi.bitrate_lower;
}
