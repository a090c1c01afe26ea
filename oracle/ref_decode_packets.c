/* ref_decode_packets.c — checkers of the device entropy decode.  TEST INFRASTRUCTURE ONLY.
 *
 *   rdp_encode_managed   the stock bitrate-managed encoder (vorbis_encode_init), packets kept as rds_encode keeps them
 *   rdp_ref_headers      each packet's block flag as vorbis_synthesis parses the header (lib/synthesis.c:37-82), -1
 *                        where it does not parse
 *   rdp_ref_staging      the reference's entropy half of mapping0_inverse (lib/mapping0.c:714-751: _floor_P[]->
 *                        inverse1, the nonzero propagation, _residue_P[]->inverse) into the staging rows of
 *                        vb200_decode_dsp, as vorbis_b200/host/vb200_decode.c's host path writes them
 *   (-DVB200_DROPIN, linked with the driver)
 *   rdp_open / rdp_ctx   a one-stream multi-stream decode driver, for its device context carrying the entropy setup
 *   rdp_md_run           rds_md_run with the host entropy path forced or not, reporting the path taken
 *
 * Packets live back to back in one byte buffer; meta[i] = {offset, bytes, granulepos, e_o_s, packetno}.
 * oracle/decode_packets.py links this file with the stock reference objects, and once more with the driver and the
 * drop-in objects.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vorbis/codec.h"
#include "vorbis/vorbisenc.h"
#include "codec_internal.h"
#include "backends.h"
#include "registry.h"

#include "vorbis_b200.h"

#define META 5

#ifdef VB200_DROPIN
typedef struct vb200md vb200md;
typedef void (*vb200md_sink)(void *user, int stream, const void *pcm, long samples);
vb200md *vb200md_open(int nstreams, ogg_packet hdr[3], int pcm_s16, int device);
int vb200md_packet(vb200md *m, int stream, const ogg_packet *op);
int vb200md_round(vb200md *m, vb200md_sink sink, void *user);
void vb200md_close(vb200md *m);
int vb200md_channels(vb200md *m);
unsigned long long vb200md_launches(vb200md *m);
void vb200md_stats(vb200md *m, long *rounds, long *blocks, long *packets, double *device_s, double *host_s);
int vb200md_entropy_on_device(vb200md *m);
void vb200md_set_host_entropy(vb200md *m, int on);
vb200_ctx *vb200md_context(vb200md *m);
#endif

static void to_packet(ogg_packet *op, const unsigned char *buf, const long *m){
  memset(op, 0, sizeof(*op));
  op->packet = (unsigned char*)buf + m[0]; op->bytes = m[1]; op->granulepos = m[2]; op->e_o_s = m[3];
  op->packetno = m[4]; op->b_o_s = (m[4] == 0);
}

static int keep(const ogg_packet *op, unsigned char *buf, long cap, long *off, long *meta, long *n, long maxn){
  long *m;
  if(*n >= maxn || *off + op->bytes > cap) return 1;
  memcpy(buf + *off, op->packet, op->bytes);
  m = meta + *n * META;
  m[0] = *off; m[1] = op->bytes; m[2] = (long)op->granulepos; m[3] = op->e_o_s; m[4] = (long)op->packetno;
  *off += op->bytes; (*n)++;
  return 0;
}

/* pcm [ch][ns] through vorbis_encode_init(ch, rate, max, nominal, min) (bit/s, -1 = unset); the packet count or -1 */
long rdp_encode_managed(int ch, long rate, long max_br, long nominal_br, long min_br, const float *pcm, long ns,
                        unsigned char *buf, long cap, long *meta, long maxn){
  vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb;
  ogg_packet hdr[3], op;
  long pos = 0, off = 0, n = 0;
  int i, eos = 0, bad = 0;
  vorbis_info_init(&vi);
  if(vorbis_encode_init(&vi, ch, rate, max_br, nominal_br, min_br)){ vorbis_info_clear(&vi); return -1; }
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

typedef struct { vorbis_info vi; vorbis_comment vc; vorbis_dsp_state vd; vorbis_block vb; } rdp_dec;

static int dec_open(rdp_dec *d, const unsigned char *buf, const long *hdr){
  int k;
  vorbis_info_init(&d->vi); vorbis_comment_init(&d->vc);
  for(k = 0; k < 3; k++){
    ogg_packet hp;
    to_packet(&hp, buf, hdr + k * META);
    if(vorbis_synthesis_headerin(&d->vi, &d->vc, &hp) < 0){ vorbis_comment_clear(&d->vc); vorbis_info_clear(&d->vi); return -1; }
  }
  vorbis_synthesis_init(&d->vd, &d->vi);
  vorbis_block_init(&d->vd, &d->vb);
  return 0;
}

static void dec_close(rdp_dec *d){
  vorbis_block_clear(&d->vb); vorbis_dsp_clear(&d->vd); vorbis_comment_clear(&d->vc); vorbis_info_clear(&d->vi);
}

/* lib/synthesis.c:37-82 up to the mapping: the block flag or -1 */
static int dec_header(rdp_dec *d, const unsigned char *pkt, long bytes){
  codec_setup_info *ci = (codec_setup_info*)d->vi.codec_setup;
  private_state *b = (private_state*)d->vd.backend_state;
  vorbis_block *vb = &d->vb;
  int mode;
  _vorbis_block_ripcord(vb);
  oggpack_readinit(&vb->opb, (unsigned char*)pkt, (int)bytes);
  if(oggpack_read(&vb->opb, 1) != 0) return -1;
  mode = oggpack_read(&vb->opb, b->modebits);
  if(mode == -1 || mode >= ci->modes || !ci->mode_param[mode]) return -1;
  vb->mode = mode;
  vb->W = ci->mode_param[mode]->blockflag;
  if(vb->W){
    vb->lW = oggpack_read(&vb->opb, 1);
    vb->nW = oggpack_read(&vb->opb, 1);
    if(vb->nW == -1) return -1;
  }else{ vb->lW = 0; vb->nW = 0; }
  vb->pcmend = ci->blocksizes[vb->W];
  return vb->W;
}

/* W [npkt]: the block flag of each packet (data + off[i], bytes[i]) or -1; returns 0 or -1 */
long rdp_ref_headers(const unsigned char *buf, const long *hdr, const unsigned char *data, const long *off,
                     const int *bytes, long npkt, int *W){
  rdp_dec d;
  long i;
  if(dec_open(&d, buf, hdr)) return -1;
  for(i = 0; i < npkt; i++) W[i] = dec_header(&d, data + off[i], bytes[i]);
  dec_close(&d);
  return 0;
}

/* packets whose header parses (W[i] >= 0): rows at coef_off[i] of res (zeroed, then decoded), posts
 * [i][ch][VB200_FLOOR1_STRIDE], present [i][ch] */
long rdp_ref_staging(const unsigned char *buf, const long *hdr, const unsigned char *data, const long *off,
                     const int *bytes, long npkt, const long *coef_off, float *res, int *posts, int *present){
  rdp_dec d;
  long i;
  if(dec_open(&d, buf, hdr)) return -1;
  for(i = 0; i < npkt; i++){
    codec_setup_info *ci = (codec_setup_info*)d.vi.codec_setup;
    private_state *b = (private_state*)d.vd.backend_state;
    vorbis_block *vb = &d.vb;
    vorbis_info_mapping0 *info;
    const int ch = d.vi.channels;
    float *pcmbundle[256];
    int zerobundle[256], nonzero[256];
    long n;
    int c, j;
    if(dec_header(&d, data + off[i], bytes[i]) < 0) continue;
    info = (vorbis_info_mapping0*)ci->map_param[ci->mode_param[vb->mode]->mapping];
    n = ci->blocksizes[vb->W];
    for(c = 0; c < ch; c++){
      const int fl = info->floorsubmap[info->chmuxlist[c]];
      int *memo = (int*)_floor_P[ci->floor_type[fl]]->inverse1(vb, b->flr[fl]);
      int *row = posts + ((size_t)i * ch + c) * VB200_FLOOR1_STRIDE;
      memset(row, 0, sizeof(int) * VB200_FLOOR1_STRIDE);
      nonzero[c] = present[(size_t)i * ch + c] = memo ? 1 : 0;
      if(memo) for(j = 0; j < ((vorbis_look_floor1*)b->flr[fl])->posts; j++) row[j] = memo[j];
      memset(res + coef_off[i] + (size_t)c * (n / 2), 0, sizeof(float) * (n / 2));
    }
    for(c = 0; c < info->coupling_steps; c++)
      if(nonzero[info->coupling_mag[c]] || nonzero[info->coupling_ang[c]])
        nonzero[info->coupling_mag[c]] = nonzero[info->coupling_ang[c]] = 1;
    for(c = 0; c < info->submaps; c++){
      int in_bundle = 0;
      for(j = 0; j < ch; j++)
        if(info->chmuxlist[j] == c){
          zerobundle[in_bundle] = nonzero[j] ? 1 : 0;
          pcmbundle[in_bundle++] = res + coef_off[i] + (size_t)j * (n / 2);
        }
      _residue_P[ci->residue_type[info->residuesubmap[c]]]->inverse(vb, b->residue[info->residuesubmap[c]],
                                                                   pcmbundle, zerobundle, in_bundle);
    }
  }
  dec_close(&d);
  return 0;
}

#ifdef VB200_DROPIN
/* a one-stream driver on the headers: its device context carries the driver's entropy setup */
void *rdp_open(const unsigned char *buf, const long *hdr, int device){
  ogg_packet h[3];
  int k;
  for(k = 0; k < 3; k++) to_packet(&h[k], buf, hdr + k * META);
  return vb200md_open(1, h, 0, device);
}
void *rdp_ctx(void *m){ return vb200md_context((vb200md*)m); }
int rdp_on_device(void *m){ return vb200md_entropy_on_device((vb200md*)m); }
void rdp_close(void *m){ vb200md_close((vb200md*)m); }

typedef struct { int s16, ch; long cap; void *out; long *len; } rdp_out;

static void rdp_put(void *user, int stream, const void *pcm, long n){
  rdp_out *o = (rdp_out*)user;
  long at = o->len[stream], take = n, j;
  int c;
  if(o->out){
    if(at + take > o->cap) take = o->cap - at;
    for(c = 0; c < o->ch; c++)
      for(j = 0; j < take; j++){
        if(o->s16) ((int16_t*)o->out)[((size_t)stream * o->cap + at + j) * o->ch + c] = ((const int16_t*)pcm)[j * o->ch + c];
        else ((float*)o->out)[((size_t)stream * o->ch + c) * o->cap + at + j] = ((const float*)pcm)[(size_t)c * n + j];
      }
  }
  o->len[stream] += n;
}

/* ns streams through one driver on the schedule sched [nrounds][ns] (then all that are left, one round);
 * host_entropy forces the host path.  out: float [ns][ch][cap] or int16 [ns][cap][ch].  stats[0..6] = rounds,
 * blocks, max launches of one round, launches, device s, host s, entropy on the device.  Returns 0 or < 0. */
long rdp_md_run(int ns, const unsigned char *buf, const long *hdr, const long *meta, const long *first,
                const long *npkt, const int *sched, int nrounds, int s16, int device, int host_entropy, void *out,
                long cap, long *len, double *stats){
  ogg_packet h[3];
  vb200md *m;
  rdp_out o;
  long *fed = (long*)calloc(ns, sizeof(long));
  long rounds = 0, blocks = 0, pk;
  unsigned long long lmax = 0, l0, lall = 0;
  int s, r, k, done = 0, rc = 0;
  double dev_s, host_s;
  for(k = 0; k < 3; k++) to_packet(&h[k], buf, hdr + k * META);
  m = vb200md_open(ns, h, s16, device);
  if(!m || !fed){ free(fed); if(m) vb200md_close(m); return -1; }
  vb200md_set_host_entropy(m, host_entropy);
  o.s16 = s16; o.ch = vb200md_channels(m); o.cap = cap; o.out = out; o.len = len;
  for(s = 0; s < ns; s++) len[s] = 0;
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
    if((rc = vb200md_round(m, rdp_put, &o)) < 0) goto out;
    l0 = vb200md_launches(m) - l0;
    lall += l0;
    if(l0 > lmax) lmax = l0;
    rc = 0;
  }
out:
  vb200md_stats(m, &rounds, &blocks, &pk, &dev_s, &host_s);
  stats[0] = (double)rounds; stats[1] = (double)blocks; stats[2] = (double)lmax; stats[3] = (double)lall;
  stats[4] = dev_s; stats[5] = host_s; stats[6] = vb200md_entropy_on_device(m);
  vb200md_close(m);
  free(fed);
  return rc;
}
#endif
