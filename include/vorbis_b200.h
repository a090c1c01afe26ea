/* vorbis_b200.h — C ABI of the CUDA per-block DSP path of libvorbis.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / C++ types.
 * Every entry point names the reference interface it replaces (paths relative
 * to the xiph/vorbis tree, libvorbis 1.3.7).  The reference-side binding a
 * libvorbis maintainer would add (a replacement `mapping0_exportbundle`) is
 * shown in INTEGRATION.md and implemented in vorbis_b200/host/.
 *
 * Conventions
 *   - return 0 on success, a negative OV_* style code on failure (never abort;
 *     lib/mapping0.c:498 returns -1, include/vorbis/codec.h:217-233 OV_*);
 *     vb200_last_error() gives a thread-local message.
 *   - N  = block size in samples (vorbis_block.pcmend), n = N/2 spectral lines.
 *   - W  = block-size flag (0 short, 1 long), as vorbis_block.W.
 *   - batches are homogeneous in W; vectors are laid out [block][channel][...]
 *     contiguous fp32 (the reference's vb->pcm[ch][N] stacked block-major).
 *   - functions ending in _dev take DEVICE pointers and a cudaStream_t passed
 *     as void* (NULL = legacy default stream) and are asynchronous;
 *     the others take HOST pointers, copy in/out and synchronise.
 *   - a context keeps grow-only device scratch: use one context per host thread
 *     (the reference is single threaded per vorbis_dsp_state as well, SURVEY §8b);
 *     the host-pointer entry points serialise on a per-context mutex.  _dev calls
 *     that use that scratch (Phase A, encode_dsp, encode_dsp_managed,
 *     encode_streams, encode_streams_managed, envelope_search, encode_entropy,
 *     encode_entropy_managed) may be issued on different CUDA streams: each waits
 *     (on the device, via an event) for the previous such call of the same
 *     context, so they never share
 *     the scratch in time.  Growing the scratch re-allocates (cudaFree/cudaMalloc
 *     synchronise the device): the first call at a new maximum size is not
 *     asynchronous.
 */
#ifndef VORBIS_B200_H
#define VORBIS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VB200_OK        0
#define VB200_EFAULT  (-129)   /* OV_EFAULT: CUDA/runtime failure            */
#define VB200_EIMPL   (-130)   /* OV_EIMPL : configuration not supported      */
#define VB200_EINVAL  (-131)   /* OV_EINVAL: bad argument                     */

#define VB200_P_BANDS        17   /* lib/psy.h:28  */
#define VB200_P_LEVELS        8   /* lib/psy.h:29  */
#define VB200_P_NOISECURVES   3   /* lib/psy.h:31  */
#define VB200_EHMER_MAX      56   /* lib/masking.h:43 */
#define VB200_COMPAND_LEVELS 40   /* lib/psy.h:33  */
#define VB200_PACKETBLOBS    15   /* lib/codec_internal.h:28 */
#define VB200_MAX_CHANNELS  255
#define VB200_VE_BANDS        7   /* lib/envelope.h:29 */
#define VB200_MAX_COUPLING  256

/* One psychoacoustic lookup == vorbis_look_psy + the vorbis_info_psy scalars
 * the per-block code reads (lib/psy.h:35-65, 96-114).  Built by the
 * reference's _vp_psy_init (lib/psy.c:266); we only consume it.            */
typedef struct vb200_psy_setup {
  int32_t n;                      /* vorbis_look_psy.n  (= blocksize/2)      */
  int32_t blockflag;              /* vorbis_info_psy.blockflag               */
  float   ath_adjatt;
  float   ath_maxatt;
  float   tone_masteratt[VB200_P_NOISECURVES];
  float   tone_abs_limit;
  float   noisemaxsupp;
  int32_t noisewindowfixed;
  float   noisecompand[VB200_COMPAND_LEVELS];
  float   max_curve_dB;
  int32_t normal_p;
  int32_t normal_start;
  int32_t normal_partition;
  double  normal_thresh;
  int32_t firstoc;
  int32_t shiftoc;
  int32_t eighth_octave_lines;
  int32_t total_octave_lines;
  float   m_val;
  const float   *ath;             /* [n]                                      */
  const int32_t *octave;          /* [n]   (reference: long)                  */
  const int32_t *bark;            /* [n]   packed ((lo-1)<<16)+(hi-1)         */
  const float   *tonecurves;      /* [P_BANDS][P_LEVELS][EHMER_MAX+2]         */
  const float   *noiseoffset;     /* [P_NOISECURVES][n]                       */
} vb200_psy_setup;

/* Floor 1 configuration of one block size: vorbis_info_floor1 (lib/backends.h:64-91).  The sorted /
 * forward / reverse indices and the decode neighbours of vorbis_look_floor1
 * (lib/codec_internal.h:138-155, built by floor1_look lib/floor1.c:180-259) are re-derived from
 * postlist by the context.                                                                    */
#define VB200_VIF_POSIT 63
#define VB200_FLOOR1_STRIDE (VB200_VIF_POSIT + 2)   /* ints per row in every posts array of this API */
#define VB200_MAX_SUBMAPS 4                          /* libvorbis' encoder setups use 1 or 2 (5.1: LFE) */
typedef struct vb200_floor1_setup {
  int32_t posts;                          /* vorbis_look_floor1.posts (<= VIF_POSIT+2); 0 = absent */
  int32_t postlist[VB200_VIF_POSIT + 2];
  int32_t mult;                           /* 1..4 */
  int32_t n;                              /* spectral lines this floor spans (postlist[1])  */
  float   maxover, maxunder, maxerr;
  float   twofitweight, twofitatten;
} vb200_floor1_setup;

/* Residue partition classification parameters of one submap: vorbis_info_residue0 (lib/backends.h:103-118)
 * + the residue type (codec_setup_info.residue_type).  Only what res{0,1,2}_class read.              */
typedef struct vb200_residue_setup {
  int32_t type;                           /* 0, 1 or 2; -1 = not provided                          */
  int32_t begin, end;                     /* in samples (type 2: interleaved samples of the bundle) */
  int32_t grouping;                       /* samples per partition                                  */
  int32_t partitions;                     /* number of partition classes                            */
  int32_t classmetric1[64];
  int32_t classmetric2[64];
} vb200_residue_setup;

/* Everything the kernels need from codec_setup_info / private_state
 * (lib/codec_internal.h:59-133) for one (channels, rate, quality) setup.    */
typedef struct vb200_setup {
  int32_t channels;
  int32_t rate;
  int32_t blocksizes[2];          /* codec_setup_info.blocksizes              */
  int32_t n_psy;                  /* 0 (decode/transform only) or 4           */
  vb200_psy_setup psy[4];         /* private_state.psy[blocktype+2*W]         */
  /* vorbis_info_psy_global (lib/psy.h:67-85) */
  float   ampmax_att_per_sec;
  int32_t coupling_pointlimit[2][VB200_PACKETBLOBS];
  int32_t coupling_prepointamp[VB200_PACKETBLOBS];
  int32_t coupling_postpointamp[VB200_PACKETBLOBS];
  int32_t sliding_lowpass[2][VB200_PACKETBLOBS];
  /* vorbis_info_mapping0 coupling (lib/backends.h:127-141), per W           */
  int32_t coupling_steps[2];
  int32_t coupling_mag[2][VB200_MAX_COUPLING];
  int32_t coupling_ang[2][VB200_MAX_COUPLING];
  /* optional half-window tables, vwin[] of lib/window.c:23-2096 for
   * blocksizes[0] and [1] (blocksize/2 floats each); NULL = compute from the
   * closed form of doc/04-codec.tex:320                                     */
  const float *window[2];
  /* floors of mode W (lib/mapping0.c:499-506): channel i uses floor1[W][chmux[W][i]], i.e. the
   * floor of its submap (vorbis_info_mapping0.chmuxlist / floorsubmap, lib/backends.h:127-141).
   * posts == 0: not provided (the floor entry points then return -1)                          */
  int32_t submaps[2];
  uint8_t chmux[2][VB200_MAX_CHANNELS + 1];
  vb200_floor1_setup floor1[2][VB200_MAX_SUBMAPS];
  /* envelope / block-switch detector: vorbis_info_psy_global.preecho_thresh, postecho_thresh,
   * stretch_penalty, preecho_minenergy (lib/psy.h:67-85), read by _ve_amp (lib/envelope.c:88-213) */
  float   preecho_thresh[VB200_VE_BANDS];
  float   postecho_thresh[VB200_VE_BANDS];
  float   stretch_penalty;
  float   preecho_minenergy;
  /* residue of submap sm of mode W: residue_param[ mapping.residuesubmap[sm] ] (lib/mapping0.c:663) */
  vb200_residue_setup residue[2][VB200_MAX_SUBMAPS];
} vb200_setup;

/* Per-block inputs of mapping0_forward that are not PCM (lib/mapping0.c:230-252) */
typedef struct vb200_block_desc {
  int32_t lW;                     /* vorbis_block.lW                          */
  int32_t nW;                     /* vorbis_block.nW                          */
  int32_t blocktype;              /* vorbis_block_internal.blocktype (0/1)    */
  float   ampmax;                 /* vorbis_block_internal.ampmax on entry    */
} vb200_block_desc;

typedef struct vb200_ctx vb200_ctx;

/* ---- context ---------------------------------------------------------- */
/* replaces the lookup building of _vds_shared_init (lib/block.c:170-294):
 * mdct_init, drft_init are recomputed here from the block sizes; the psy
 * lookups and windows are uploaded as given.                                */
int  vb200_ctx_create(const vb200_setup *setup, int device, vb200_ctx **out);
void vb200_ctx_destroy(vb200_ctx *ctx);
int  vb200_device_count(void);
const char *vb200_last_error(void);
/* host copies of the tables the context derived itself (for parity tests):
 * which: 0 mdct trig (N+N/4), 1 mdct bitrev (N/4 int32), 2 window (N/2),
 * 3 fft twiddles (N).  Returns element count or <0.                         */
int  vb200_ctx_table(vb200_ctx *ctx, int W, int which, void *dst, int cap);
/* kernels launched through this context since creation (bench evidence)     */
uint64_t vb200_launch_count(vb200_ctx *ctx);
/* measurement aid: when on, the Phase-A entry points bracket each of their three
 * kernels (transform, ampmax, psy) with CUDA events on the launching stream;
 * vb200_phaseA_kernel_ms returns the durations of the last call (ms3[3]).       */
int  vb200_set_profiling(vb200_ctx *ctx, int on);
int  vb200_phaseA_kernel_ms(vb200_ctx *ctx, float *ms3);
/* same for the last vb200_encode_dsp_dev call: transform, ampmax, psy, floor1_fit, floor1_render,
 * couple_quantize_normalize (+ nonzero propagation)                                            */
int  vb200_encode_dsp_kernel_ms(vb200_ctx *ctx, float *ms6);
/* development aid: with env VB200_PHASE_TIMING set, the psy kernel adds the SM cycles each of
 * its 11 barrier-delimited phases took (thread 0 of every CTA) into a 16-slot counter array;
 * with env VB200_FLOOR1_TIMING set, the floor-1 fit adds its per-phase cycles and per-row counts
 * (summed over its warps, layout in tools/floor1_phase_timing.py) into the same array.          */
int  vb200_debug_phase_cycles(vb200_ctx *ctx, unsigned long long *out16, int reset);

/* ---- transforms (SURVEY §8 a2-a5) ------------------------------------- */
/* mdct_forward, lib/mdct.c:492: in [nvec][N] -> out [nvec][N/2]            */
int vb200_mdct_forward_dev (vb200_ctx*, int W, int nvec, const float *d_in, float *d_out, void *stream);
int vb200_mdct_forward     (vb200_ctx*, int W, int nvec, const float *in,   float *out);
/* mdct_backward, lib/mdct.c:396: in [nvec][N/2] -> out [nvec][N]; in half-rate mode
 * (vb200_synthesis_halfrate) the transform of size N/2: in [nvec][N/4] -> out [nvec][N/2] */
int vb200_mdct_backward_dev(vb200_ctx*, int W, int nvec, const float *d_in, float *d_out, void *stream);
int vb200_mdct_backward    (vb200_ctx*, int W, int nvec, const float *in,   float *out);
/* _vorbis_apply_window, lib/window.c:2102: in place on [nvec][N];
 * lW/nW are per-vector int32 arrays (host) or NULL for W=0                  */
int vb200_apply_window     (vb200_ctx*, int W, int nvec, const int32_t *lW, const int32_t *nW, float *data);
/* drft_forward, lib/smallft.c:1231: in place on [nvec][N], FFTPACK layout   */
int vb200_drft_forward     (vb200_ctx*, int W, int nvec, float *data);

/* ---- psychoacoustic stages, stage-isolated (SURVEY §8 a8-a10) --------- */
/* look = blocktype + 2*W selects vb200_setup.psy[look]                      */
/* _vp_noisemask, lib/psy.c:706: logmdct [nvec][n] -> noise [nvec][n]       */
int vb200_noisemask        (vb200_ctx*, int look, int nvec, const float *logmdct, float *noise);
/* _vp_tonemask, lib/psy.c:754: logfft [nvec][n], specmax per vector         */
int vb200_tonemask         (vb200_ctx*, int look, int nvec, const float *logfft,
                            const float *global_specmax, const float *local_specmax, float *tone);
/* _vp_offset_and_mix, lib/psy.c:779: writes logmask, scales mdct in place   */
int vb200_offset_and_mix   (vb200_ctx*, int look, int nvec, int offset_select,
                            const float *noise, const float *tone,
                            float *mdct, const float *logmdct, float *logmask);

/* ---- encode Phase A: the per-channel loops of mapping0_forward
 *      (lib/mapping0.c:254-470): window, MDCT, FFT, log spectra, ampmax,
 *      noise mask, tone mask, offset_and_mix(select 1).
 * pcm     [nblocks][ch][N]   un-windowed block PCM (vb->pcm), read-only
 * desc    [nblocks]
 * mdct    [nblocks][ch][n]   gmdct after the AoTuV-M1 scaling (mapping0.c:463)
 * logmdct [nblocks][ch][n]   input of floor1_fit (mapping0.c:500)
 * logmask [nblocks][ch][n]   input of floor1_fit
 * ampmax_out [nblocks]       vorbis_block_internal.ampmax on exit (mapping0.c:576)
 * Optional taps (may be NULL): noise, tone, logfft [nblocks][ch][n], raw mdct. */
typedef struct vb200_phaseA_io {
  const float *pcm;
  const vb200_block_desc *desc;
  float *mdct;
  float *logmdct;
  float *logmask;
  float *ampmax_out;
  float *tap_noise;
  float *tap_tone;
  float *tap_logfft;
  float *tap_mdct_raw;
} vb200_phaseA_io;
int vb200_analysis_phaseA_dev(vb200_ctx*, int W, int nblocks, const vb200_phaseA_io *d_io, void *stream);
int vb200_analysis_phaseA    (vb200_ctx*, int W, int nblocks, const vb200_phaseA_io *io);

/* Stream mode: `nstreams` streams of `blocks_per_stream` consecutive blocks
 * (block index = stream*blocks_per_stream + k).  desc[].ampmax is ignored;
 * the ampmax chain of vorbis_analysis_blockout (lib/block.c:626-628,
 * lib/psy.c:837-848) is evaluated on the device between the transform and
 * the psy kernel, starting from `ampmax0[stream]` (NULL = -9999).           */
int vb200_analysis_phaseA_streams_dev(vb200_ctx*, int W, int nstreams, int blocks_per_stream,
                                      const vb200_phaseA_io *d_io, const float *d_ampmax0, void *stream);

/* ---- PCM ingest fused into Phase A (SURVEY §8 f4) -----------------------------------------
 * Each stream's PCM is ONE contiguous buffer; block k of a stream is the N samples that start
 * at sample k*hop - exactly what vorbis_analysis_blockout copies out of v->pcm (lib/block.c:630-643;
 * hop = N/2 for a run of equal-size blocks), so the 50 % overlap is never duplicated in memory.
 *   fmt VB200_PCM_F32_PLANAR : float [stream][ch][stream_stride]
 *   fmt VB200_PCM_S16_INTERLEAVED : int16 [stream][stream_stride][ch], converted sample/32768.f
 *       as examples/encoder_example.c:196-201 does
 * io->pcm is ignored; everything else as vb200_analysis_phaseA_streams_dev (ampmax chain on device,
 * d_ampmax0 may be NULL).  stream_stride counts samples per channel; it and hop must be multiples
 * of 4 for the float format.                                                                 */
#define VB200_PCM_F32_PLANAR       1
#define VB200_PCM_S16_INTERLEAVED  2
int vb200_analysis_phaseA_pcmstream_dev(vb200_ctx*, int W, int nstreams, int blocks_per_stream,
                                        const void *d_pcm, int fmt, int64_t stream_stride, int hop,
                                        const vb200_phaseA_io *d_io, const float *d_ampmax0, void *stream);

/* ---- floor 1 on the device (SURVEY §8 f1) ---------------------------------------------------
 * Rows are (block, channel) pairs.  floor_sel = -1: rows are laid out [block][channel] like the
 * Phase A outputs and row r uses the floor of channel r % channels; floor_sel >= 0: every row uses
 * floor1[W][floor_sel] (what one reference call with one vorbis_look_floor1 does).
 * All posts arrays are [rows][VB200_FLOOR1_STRIDE] int32; entries past the floor's posts are 0.
 *
 * floor1_fit (lib/floor1.c:576-729): logmdct, logmask [rows][n] -> posts exactly as the reference
 * returns them (unused posts carry predicted|0x8000); fit_nonzero[rows] = 0 where the reference
 * returns NULL (silent channel; the row of posts is then all 0).                               */
int vb200_floor1_fit_dev(vb200_ctx*, int W, int floor_sel, int nrows, const float *d_logmdct,
                         const float *d_logmask, int32_t *d_posts, int32_t *d_fit_nonzero, void *stream);
int vb200_floor1_fit    (vb200_ctx*, int W, int floor_sel, int nrows, const float *logmdct,
                         const float *logmask, int32_t *posts, int32_t *fit_nonzero);
/* the part of floor1_encode that is not bit packing (lib/floor1.c:765-832, 919-945): quantise the
 * posts to the multiplier, apply the prediction/flag pass, render the integer floor curve.
 * posts is updated in place to what the reference leaves in post[]; ilogmask [rows][n] is the curve
 * (all zero and nonzero = 0 where fit_nonzero is 0).                                            */
int vb200_floor1_render_dev(vb200_ctx*, int W, int floor_sel, int nrows, int32_t *d_posts,
                            const int32_t *d_fit_nonzero, int32_t *d_ilogmask, int32_t *d_nonzero,
                            void *stream);
int vb200_floor1_render    (vb200_ctx*, int W, int floor_sel, int nrows, int32_t *posts,
                            const int32_t *fit_nonzero, int32_t *ilogmask, int32_t *nonzero);

/* ---- encode Phase B: _vp_couple_quantize_normalize, lib/psy.c:1014 ----
 * mdct  [nblocks][ch][n]  (Phase A output)
 * iwork [nblocks][ch][n]  in: ilogmask from floor1_encode (0..1023 dB index,
 *                         mapping0.c:617), out: quantised residue ints
 * nonzero [nblocks][ch]   in/out                                            */
int vb200_couple_quantize_normalize_dev(vb200_ctx*, int W, int blocktype, int blobno, int nblocks,
                                        const float *d_mdct, int32_t *d_iwork, int32_t *d_nonzero, void *stream);
int vb200_couple_quantize_normalize    (vb200_ctx*, int W, int blocktype, int blobno, int nblocks,
                                        const float *mdct, int32_t *iwork, int32_t *nonzero);

/* ---- residue partition classification (SURVEY §8 f3): res1_class / res2_class (lib/res0.c:745-778)
 * -> _01class (:412-474) / _2class (:479-532), called per submap as mapping0_forward does (:660-672).
 * iwork   [nblocks][ch][n] quantised residue (what vb200_couple_quantize_normalize leaves)
 * nonzero [nblocks][ch]
 * classes [nblocks][ch][class_stride] int32 partition classes (the reference's partword):
 *   residue type 0/1: row of channel c holds partword of that channel, valid where nonzero[c] (the
 *     reference compacts the used channels of a submap: partword[u] = row of the u-th used channel);
 *   residue type 2: ONE vector per submap, stored in the row of the submap's first channel, valid if any
 *     channel of the submap is nonzero (the reference then classifies the whole bundle, :769-778).
 *   Rows that are not valid and entries past partvals = (end-begin)/grouping are 0.
 * class_stride >= vb200_residue_partvals(ctx, W) (the largest partvals over the mode's submaps).    */
int vb200_residue_partvals(vb200_ctx*, int W);
int vb200_residue_classify_dev(vb200_ctx*, int W, int nblocks, const int32_t *d_iwork, const int32_t *d_nonzero,
                               int32_t *d_classes, int class_stride, void *stream);
int vb200_residue_classify    (vb200_ctx*, int W, int nblocks, const int32_t *iwork, const int32_t *nonzero,
                               int32_t *classes, int class_stride);

/* ---- the whole per-block encode DSP of mapping0_forward in ONE call ---------------------------
 * lib/mapping0.c:230-646 with the bit packing and the residue backend left to the caller:
 *   window, MDCT, FFT, log spectra, ampmax (:254-346)  ->  noise / tone masks, offset_and_mix(1)
 *   (:366-470)  ->  floor1_fit (:500)  ->  the non-bit-packing part of floor1_encode (:617)
 *   ->  _vp_couple_quantize_normalize (:631-646)
 * for un-managed bitrate (only blob `blobno` = PACKETBLOBS/2 is produced, :592-594).  The float
 * spectra never leave the device: per stereo long block 4 KB of int16 PCM go in and 8.4 KB come
 * back (posts, nonzero, quantised residue) instead of 16 KB + 24.6 KB for Phase A alone.
 *
 * Blocks are `nstreams` x `blocks_per_stream`, block index = stream*blocks_per_stream + k.
 *   pcm_fmt VB200_PCM_F32_BLOCKS      float [nblocks][ch][N]  (vb->pcm as blockout leaves it)
 *           VB200_PCM_F32_PLANAR      float [stream][ch][stream_stride], block k starts at k*hop
 *           VB200_PCM_S16_INTERLEAVED int16 [stream][stream_stride][ch], sample/32768.f
 *   desc[nblocks]      lW, nW, blocktype of every block (psy look = blocktype + 2W, :250)
 *   independent != 0   desc[].ampmax is each block's ampmax on entry (what one vorbis_analysis
 *                      call sees); == 0: the decay chain of vorbis_analysis_blockout
 *                      (lib/block.c:626-628) runs per stream from ampmax0[stream] (NULL = -9999)
 * Outputs (what floor1_encode's bit packer and the residue backend consume):
 *   posts   [nblocks][ch][VB200_FLOOR1_STRIDE]  post[] as floor1_encode leaves it (:765-832)
 *   nonzero [nblocks][ch]                       after the coupling propagation (lib/psy.c:1203)
 *   iwork   [nblocks][ch][n]                    quantised, coupled residue ints
 *   ampmax_out [nblocks]                        vorbis_block_internal.ampmax on exit (:576)
 *   mdct, logmdct, logmask [nblocks][ch][n]     optional (NULL = stay in device scratch)
 * iwork_fmt VB200_IWORK_S16 halves the largest output: the residue leaves as int16, saturated to
 * [-32768,32767]; overflow[block] counts the values of that block that were clipped (0 for any
 * realistic signal: |mdct|/floor would have to exceed 32767) - a caller that sees a non-zero
 * count re-runs that block with VB200_IWORK_S32.                                                */
#define VB200_PCM_F32_BLOCKS       0
#define VB200_IWORK_S32            0
#define VB200_IWORK_S16            1
typedef struct vb200_encode_io {
  const void *pcm;
  int32_t pcm_fmt;
  int32_t hop;
  int64_t stream_stride;
  const vb200_block_desc *desc;
  const float *ampmax0;
  int32_t independent;
  int32_t iwork_fmt;              /* VB200_IWORK_S32 (0) or VB200_IWORK_S16 */
  int32_t *posts;
  int32_t *nonzero;
  void    *iwork;                 /* int32 or int16 [nblocks][ch][n], see iwork_fmt */
  float *ampmax_out;
  float *mdct;
  float *logmdct;
  float *logmask;
  int32_t *overflow;              /* VB200_IWORK_S16 only: [nblocks] values that did not fit */
  int32_t *classes;               /* optional [nblocks][ch][class_stride]: vb200_residue_classify of the residue */
  int64_t class_stride;
} vb200_encode_io;
/* every pointer in *d_io is a device pointer; the struct itself is host memory */
int vb200_encode_dsp_dev(vb200_ctx*, int W, int nstreams, int blocks_per_stream, int blobno,
                         const vb200_encode_io *d_io, void *stream);
/* host buffers (pinned memory makes the copies asynchronous); whole streams are cut into chunks
 * that rotate over four device buffer sets: all H2D copies on one stream, all D2H copies on
 * another, the kernels of consecutive chunks on two compute streams, ordered by events         */
int vb200_encode_dsp    (vb200_ctx*, int W, int nstreams, int blocks_per_stream, int blobno,
                         const vb200_encode_io *io);

/* ---- bitrate-managed mode (SURVEY §8 a12) ------------------------------------------------------
 * What mapping0_forward does when vorbis_bitrate_managed(vb) (lib/mapping0.c:507-573, 596-646):
 * Phase A as above, then besides the middle mask (offset_select 1) the low-noise and the
 * high-noise masks (_vp_offset_and_mix selections 2 and 0, lib/psy.c:779-835), a floor1_fit on
 * each (only where the middle fit exists), the twelve floor1_interpolate_fit curves in between
 * (lib/floor1.c:731-757; a curve exists only where both of its ends do), and for EVERY one of the
 * VB200_PACKETBLOBS curves k: the floor render (floor1_encode minus the bits, :765-945) and
 * _vp_couple_quantize_normalize with blob k's coupling parameters and sliding low-pass.
 * Same vb200_encode_io as vb200_encode_dsp with blob-major outputs:
 *   posts   [VB200_PACKETBLOBS][nblocks*ch][VB200_FLOOR1_STRIDE]   (all zero where the curve is NULL)
 *   nonzero [VB200_PACKETBLOBS][nblocks*ch]
 *   iwork   [VB200_PACKETBLOBS][nblocks*ch][n]                     (iwork_fmt must be VB200_IWORK_S32)
 * classes / overflow must be NULL.  The host keeps what it keeps in un-managed mode: the bits of
 * floor1_encode, residue coding, and the bitrate manager's choice among the 15 packets.          */
int vb200_encode_dsp_managed_dev(vb200_ctx*, int W, int nstreams, int blocks_per_stream,
                                 const vb200_encode_io *d_io, void *stream);
int vb200_encode_dsp_managed    (vb200_ctx*, int W, int nstreams, int blocks_per_stream,
                                 const vb200_encode_io *io);

/* ---- envelope / block-switch detector (SURVEY §8 f2) -----------------------------------------
 * The analysis loop of _ve_envelope_search (lib/envelope.c:232-267): for steps j = first_step ..
 * first_step+nsteps-1 of every stream and every channel, _ve_amp (:88-213) on the 128 samples that
 * start at sample 64*j - squared-sine window, mdct_forward(128), near-DC spreading, the seven band
 * amplitudes, their pre-/post-echo deltas against the 17-deep amplitude history - and the stretch
 * logic that couples the channels.  Everything that vorbis_analysis_blockout then does with the
 * result (cursor / curmark walk, :269-327) only reads the marks and stays on the host.
 *
 * pcm     stream PCM, VB200_PCM_F32_PLANAR [stream][ch][stream_stride] or VB200_PCM_S16_INTERLEAVED
 *         [stream][stream_stride][ch]; 64*(first_step+nsteps-1)+128 <= stream_stride
 * state   [nstreams][VB200_VE_STATE_WORDS(ch)] 32-bit words, in/out: word 0 = envelope_lookup.stretch,
 *         then envelope_filter_state[ch*VE_BANDS] with the reference's own layout (lib/envelope.h:32-42:
 *         ampbuf[17], ampptr, nearDC[15], nearDC_acc, nearDC_partialacc, nearptr) so that a binding
 *         can copy ve->filter in and out verbatim; all zero = a fresh vorbis_dsp_state
 * ret     [nstreams][nsteps] the loop's `ret` per step: bit 0 (and 2) pre-echo, bit 1 post-echo
 * vb200_envelope_apply_marks (plain C, no CUDA) replays lib/envelope.c:254-264 on a mark array.   */
#define VB200_VE_FILTER_WORDS 36
#define VB200_VE_STATE_WORDS(ch) (1 + VB200_VE_FILTER_WORDS * VB200_VE_BANDS * (ch))
int vb200_envelope_search_dev(vb200_ctx*, int nstreams, const void *d_pcm, int pcm_fmt, int64_t stream_stride,
                              int first_step, int nsteps, int32_t *d_state, uint8_t *d_ret, void *stream);
int vb200_envelope_search    (vb200_ctx*, int nstreams, const void *pcm, int pcm_fmt, int64_t stream_stride,
                              int first_step, int nsteps, int32_t *state, uint8_t *ret);
void vb200_envelope_apply_marks(const uint8_t *ret, int first_step, int nsteps, int32_t *mark);
/* many streams with DIFFERENT amounts of new data in one call (the multi-stream driver of
 * vorbis_b200/host/vb200_mapping0.c): stream s analyses steps 0 .. steps_per_stream[s]-1 (<= nsteps) of its
 * buffer; ret [nstreams][nsteps], entries past a stream's own count are left untouched.  Host pointers.   */
int vb200_envelope_search_var(vb200_ctx*, int nstreams, const void *pcm, int pcm_fmt, int64_t stream_stride,
                              int nsteps, const int32_t *steps_per_stream, int32_t *state, uint8_t *ret);

/* ---- block planning: what vorbis_analysis_blockout decides per block (SURVEY §8 a15) ----------------
 * lib/block.c:556-615 (nW from the envelope marks, blocktype) with the cursor / curmark walk of
 * _ve_envelope_search (lib/envelope.c:269-327) and _ve_envelope_mark (:329-356), replayed per stream
 * on the stream's timeline buffer: sample 0 is v->pcm[][0] of a fresh vorbis_dsp_state, i.e. the
 * blocksizes[1]/2 samples of (pre-extrapolated) preamble, then the caller's PCM, then - after EOF -
 * the extrapolated tail of vorbis_analysis_wrote(v,0).
 *   mark   [nstreams][mark_stride] int32, mark[j] = envelope_lookup.mark of the 64-sample step j counted
 *          from sample 0 (vb200_envelope_search + vb200_envelope_apply_marks over the whole timeline)
 *   nsteps steps analysed (the reference's `last` = pcm_len/64 - 4 when the whole timeline was searched)
 *   pcm_len[nstreams]  samples present per stream (v->pcm_current without any shift)
 *   eof    [nstreams]  v->eofflag in timeline samples (preamble + samples written) or 0: no EOF yet
 *   plan   [nstreams][max_blocks] blocks in stream order; nblocks[nstreams] how many (the stream stops
 *          where vorbis_analysis_blockout would return 0)
 * block sizes: blocksizes[0]/4 must be a multiple of 64 (the envelope search step).               */
typedef struct vb200_stream_block {
  int32_t pos;        /* first sample of the block on the timeline (centerW - blocksizes[W]/2) */
  int32_t slot;       /* index of the block among the blocks of its size in the whole call */
  int32_t W, lW, nW;  /* vb->W, vb->lW, vb->nW */
  int32_t blocktype;  /* vorbis_block_internal.blocktype (psy look = blocktype + 2W) */
} vb200_stream_block;
int vb200_plan_blocks(vb200_ctx*, int nstreams, const int32_t *mark, int64_t mark_stride, int nsteps,
                      const int64_t *pcm_len, const int64_t *eof, int max_blocks,
                      vb200_stream_block *plan, int32_t *nblocks);

/* ---- whole streams in ONE call (SURVEY §8 a12 + a15): envelope search, block planning, then the
 * per-block encode DSP of both block sizes with the ampmax decay chain carried along each stream
 * across sizes (lib/block.c:626-628).  The blocks of size W of all streams form one batch; block
 * `slot` of that batch writes posts[W][slot], nonzero[W][slot], iwork[W][slot], ampmax_out[W][slot].
 *   pcm       timeline buffers (see vb200_plan_blocks), VB200_PCM_F32_PLANAR [stream][ch][stream_stride]
 *             or VB200_PCM_S16_INTERLEAVED [stream][stream_stride][ch]
 *   cap[W]    capacity (blocks) of the size-W outputs; count[W] (host, out) blocks produced
 *   plan / nblocks as vb200_plan_blocks (device pointers for the _dev form)
 * Un-managed bitrate (blob `blobno`).  Streams start fresh (zero envelope state, ampmax -9999).   */
typedef struct vb200_streams_io {
  const void *pcm;
  int32_t pcm_fmt;
  int32_t max_blocks;
  int64_t stream_stride;
  const int64_t *pcm_len;      /* [nstreams] */
  const int64_t *eof;          /* [nstreams] or NULL (no EOF anywhere) */
  vb200_stream_block *plan;    /* [nstreams][max_blocks] out */
  int32_t *nblocks;            /* [nstreams] out */
  int32_t cap[2];
  int32_t count[2];            /* out (host) */
  int32_t *posts[2];           /* [cap][ch][VB200_FLOOR1_STRIDE] */
  int32_t *nonzero[2];         /* [cap][ch] */
  int32_t *iwork[2];           /* [cap][ch][blocksizes[W]/2] */
  float   *ampmax_out[2];      /* [cap] */
} vb200_streams_io;
int vb200_encode_streams_dev(vb200_ctx*, int nstreams, int blobno, vb200_streams_io *d_io, void *stream);
int vb200_encode_streams    (vb200_ctx*, int nstreams, int blobno, vb200_streams_io *io);
/* Bitrate-managed whole streams: the same envelope search, plan, transforms and ampmax chain, then per size the
 * psy stage and every step of vb200_encode_dsp_managed (three masks and fits, twelve interpolated curves, floor
 * render and couple/quantise/normalise of all VB200_PACKETBLOBS curves).  Same vb200_streams_io; the curve
 * outputs are blob-major with cap[W] blocks from one curve to the next, so their layout is fixed before count[W]
 * is known:
 *   posts[W]      [VB200_PACKETBLOBS][cap[W]*ch][VB200_FLOOR1_STRIDE]   (all zero where the curve is NULL)
 *   nonzero[W]    [VB200_PACKETBLOBS][cap[W]*ch]
 *   iwork[W]      [VB200_PACKETBLOBS][cap[W]*ch][blocksizes[W]/2]        int32
 *   ampmax_out[W] [cap[W]]
 * Block `slot` of curve k is row k*cap[W]*ch + slot*ch + channel; rows past count[W] of a curve are not
 * written.  count[] and the error when count > cap as vb200_encode_streams.  The host form makes one
 * synchronous H2D - compute - D2H round trip (no chunk pipeline) and copies back count[W] blocks of every
 * curve into the same cap-strided host layout.  Device scratch per size besides that of vb200_encode_streams:
 * the psy stage's noise and tone taps and the low-/high-noise mask (3 x count*ch*blocksizes[W]/2 floats), the
 * three fits' flags (3 x count*ch) and the curves' present flags (VB200_PACKETBLOBS x cap*ch), int32.          */
int vb200_encode_streams_managed_dev(vb200_ctx*, int nstreams, vb200_streams_io *d_io, void *stream);
int vb200_encode_streams_managed    (vb200_ctx*, int nstreams, vb200_streams_io *io);

/* ---- decode: mdct_backward (lib/mapping0.c:792-795) fused with the windowed
 *      overlap-add of vorbis_synthesis_blockin (lib/block.c:767-823).
 * `nstreams` independent streams x `ch` channels, each `nblk` blocks long.
 * Wseq  [nstreams][nblk] int32 block-size flags
 * coef_off [nstreams][nblk] int64 offset (floats) of block k's spectra inside
 *       `coef`; channel c of that block is at coef_off + c*n_k
 * pcm_off  [nstreams][nblk] int64 offset (floats) into each channel's output
 *       where the samples finished by block k go (k=0 finishes nothing)
 * pcm   [nstreams][ch][pcm_stride]
 * Half-rate mode (vb200_synthesis_halfrate): the same coef layout (channel stride n_k), of which the
 * first n_k/2 lines of every channel are read; the IMDCT runs at N_k/2, the overlap-add uses the
 * half windows of the halved sizes and block k finishes (N_{k-1}/4 + N_k/4)/2 samples
 * (lib/block.c:735-842); pcm_off and pcm_stride count half-rate samples.                 */
int vb200_synthesis_dev(vb200_ctx*, int nstreams, int nblk, const int32_t *d_Wseq,
                        const int64_t *d_coef_off, const float *d_coef,
                        const int64_t *d_pcm_off, float *d_pcm, int64_t pcm_stride, void *stream);
/* same, but the finished samples leave as interleaved int16 [stream][pcm_stride][ch]:
 * floor(x*32767.f+.5f) clipped to [-32768,32767] (examples/decoder_example.c:250-262)          */
int vb200_synthesis_s16_dev(vb200_ctx*, int nstreams, int nblk, const int32_t *d_Wseq,
                            const int64_t *d_coef_off, const float *d_coef,
                            const int64_t *d_pcm_off, int16_t *d_pcm16, int64_t pcm_stride, void *stream);
int vb200_synthesis    (vb200_ctx*, int nstreams, int nblk, const int32_t *Wseq,
                        const int64_t *coef_off, const float *coef, int64_t coef_len,
                        const int64_t *pcm_off, float *pcm, int64_t pcm_stride);
/* vorbis_synthesis_halfrate, lib/synthesis.c:166-174: flag != 0 turns half-rate decode on for the
 * decode entry points of this context (mdct_backward, synthesis[_s16], decode_dsp; host and _dev forms).
 * window[w] = the half-window of block size blocksizes[w]/2 (blocksizes[w]/4 floats), i.e. what
 * _vorbis_window_get(b->window[w]-1) returns; NULL = closed form (not bit-exact, as for vb200_setup.window).
 * The tables are built on the first call that turns the mode on; later calls do not read `window`.
 * Returns VB200_EINVAL when flag != 0 and blocksizes[0] <= 64 (the reference returns -1 there).
 * Takes effect for calls issued after it returns; encode entry points ignore it.                     */
int vb200_synthesis_halfrate(vb200_ctx*, int flag, const float *const window[2]);

/* ---- decode: channel de-coupling of mapping0_inverse (lib/mapping0.c:754-779).
 * res [nblocks][ch][n] residue vectors as left by the residue backend; every coupling step
 * (magnitude, angle) -> (left, right) is undone in place, last step first.  Elementwise.  */
int vb200_decouple_dev(vb200_ctx*, int W, int nblocks, float *d_res, void *stream);
int vb200_decouple    (vb200_ctx*, int W, int nblocks, float *res);

/* ---- decode: floor1_inverse2 (lib/floor1.c:1041-1086), the floor curve multiplied into the spectrum.
 * data [rows][n] in place; posts [rows][VB200_FLOOR1_STRIDE] = fit_value[] as floor1_inverse1 returns it
 * (:962-1039; unused posts carry bit 15); present[rows] = 0 where floor1_inverse1 returned NULL (the row
 * is zeroed, :1084).  Rows and floor_sel as for vb200_floor1_fit.                                        */
int vb200_floor1_inverse2_dev(vb200_ctx*, int W, int floor_sel, int nrows, const int32_t *d_posts,
                              const int32_t *d_present, float *d_data, void *stream);
int vb200_floor1_inverse2    (vb200_ctx*, int W, int floor_sel, int nrows, const int32_t *posts,
                              const int32_t *present, float *data);

/* ---- decode: everything of mapping0_inverse after the entropy decoders (lib/mapping0.c:754-795) plus
 * the overlap-add of vorbis_synthesis_blockin, in one call: channel de-coupling, floor multiply,
 * mdct_backward, windowed overlap-add.  Layout as vb200_synthesis; `res` holds the residue vectors as
 * the residue backend leaves them and is modified in place; posts / present are
 * [nstreams][nblk][ch][VB200_FLOOR1_STRIDE] and [nstreams][nblk][ch].  pcm_s16 != 0: the finished
 * samples leave as interleaved int16 (as vb200_synthesis_s16_dev), else planar float.
 * Half-rate mode: de-coupling and the floor multiply still cover all n lines, so `res` is left exactly
 * as at full rate (lib/mapping0.c:754-790); the rest is vb200_synthesis in half-rate mode.               */
int vb200_decode_dsp_dev(vb200_ctx*, int nstreams, int nblk, const int32_t *d_Wseq, const int64_t *d_coef_off,
                         float *d_res, const int32_t *d_posts, const int32_t *d_present,
                         const int64_t *d_pcm_off, void *d_pcm, int pcm_s16, int64_t pcm_stride, void *stream);
int vb200_decode_dsp    (vb200_ctx*, int nstreams, int nblk, const int32_t *Wseq, const int64_t *coef_off,
                         float *res, int64_t res_len, const int32_t *posts, const int32_t *present,
                         const int64_t *pcm_off, void *pcm, int pcm_s16, int64_t pcm_stride);

/* ---- decode resumed across calls: vb200_decode_dsp for a decoder that receives its packets over time.
 * The overlap state that vorbis_synthesis_blockin keeps between blocks (lib/block.c:767-823) lives in a
 * carry, one entry per (stream, channel):
 *   tail [nstreams][ch][blocksizes[1]/2]  the right half of that channel's last IMDCT (n_W/2 floats used;
 *                                         n_W/4 in half-rate mode)
 *   W    [nstreams][ch]                   that block's size flag, -1 = nothing decoded yet
 * A new decoder starts with every W = -1.  Stream s decodes count[s] <= nblk blocks (count NULL: nblk);
 * the Wseq, coef_off, pcm_off, posts and present entries of blocks past count[s] are not read and those
 * blocks write nothing, and a stream with count[s] = 0 leaves its carry as it was.  Where the carried W is
 * >= 0, block 0 overlap-adds onto the carried tail and finishes (N_W'/4 + N_W/4) samples (halved in half-rate
 * mode) at pcm_off[s][0], W' the carried flag; where it is -1, block 0 only primes, as in vb200_decode_dsp.
 * After the call the carry holds the last decoded block of every stream that decoded one.
 * Contract: cutting a stream's blocks into any sequence of calls that pass the carry along gives the PCM of
 * one vb200_decode_dsp call over all of them, bit for bit.  A carry is only valid in the mode (full or half
 * rate) that produced it.  Otherwise layout and arguments as vb200_decode_dsp.  Two kernel launches.
 * _dev: every pointer is device memory except `carry` itself, a host struct holding device pointers; the
 * values of count and of the carried W are used as they are (as Wseq in vb200_decode_dsp_dev).
 * Host form: the carry's arrays are host memory, copied in and back out.  Returns VB200_EINVAL for a null
 * pointer, count[s] outside [0, nblk], a carried W outside {-1, 0, 1} or a counted Wseq entry outside {0, 1}. */
typedef struct vb200_decode_carry {
  float   *tail;
  int32_t *W;
} vb200_decode_carry;
int vb200_decode_dsp_resume_dev(vb200_ctx*, int nstreams, int nblk, const int32_t *d_count, const int32_t *d_Wseq,
                                const int64_t *d_coef_off, float *d_res, const int32_t *d_posts,
                                const int32_t *d_present, const int64_t *d_pcm_off, void *d_pcm, int pcm_s16,
                                int64_t pcm_stride, const vb200_decode_carry *carry, void *stream);
int vb200_decode_dsp_resume    (vb200_ctx*, int nstreams, int nblk, const int32_t *count, const int32_t *Wseq,
                                const int64_t *coef_off, float *res, int64_t res_len, const int32_t *posts,
                                const int32_t *present, const int64_t *pcm_off, void *pcm, int pcm_s16,
                                int64_t pcm_stride, vb200_decode_carry *carry);

/* ---- decode: the entropy half of mapping0_inverse (lib/mapping0.c:714-751) on the device.
 * What floor1_inverse1 (lib/floor1.c:955-1039) and the residue inverse of types 1 and 2 (lib/res0.c:651-711,
 * 812-864) read, in a plain form registered on a context with vb200_decode_entropy_setup.
 *
 * vb200_codebook: one codebook as vorbis_book_decode sees it.  Codeword i has length length[i] (1..32) and the
 * bits bits[i], the first bit of the stream in bit 0 (what oggpack_read(length[i]) returns when the codeword is
 * next); vorbis_book_decode returns entry[i] for it, and the residue adds value[i*dim .. i*dim+dim) (NULL for a
 * book without a value mapping).  used == 0: a book with no codelist, for which vorbis_book_decode returns -1
 * and the residue adds read nothing (lib/codebook.c:389-403, 428-443, 472-495).                               */
typedef struct vb200_codebook {
  int32_t dim;                     /* elements per vector, 1..127                    */
  int32_t used;                    /* codewords                                      */
  const uint8_t  *length;          /* [used]                                         */
  const uint32_t *bits;            /* [used]                                         */
  const int32_t  *entry;           /* [used]                                         */
  const float    *value;           /* [used][dim] or NULL                            */
} vb200_codebook;

/* the decode fields of vorbis_info_floor1 (lib/backends.h:60-68); the posts and mult come from the context's
 * vb200_floor1_setup of the same (W, submap) */
typedef struct vb200_floor_decode {
  int32_t type;                    /* the floor type; only 1 is taken (else VB200_EIMPL) */
  int32_t partitions;              /* 0..31                                          */
  int32_t partitionclass[31];      /* 0..15                                          */
  int32_t class_dim[16];           /* 1..8                                           */
  int32_t class_subs[16];          /* 0..3                                           */
  int32_t class_book[16];          /* read where class_subs > 0                      */
  int32_t class_subbook[16][8];    /* -1 = none                                      */
} vb200_floor_decode;

/* the decode fields of vorbis_info_residue0 (lib/backends.h:103-118) with its stage books laid out as res0_look
 * lays them out (lib/res0.c:274-299): stagebook[class][s] for the ilog(secondstages) stages of each class, -1
 * where a stage bit is clear */
typedef struct vb200_residue_decode {
  int32_t type;                    /* 1 or 2 (0: VB200_EIMPL); -1 = submap not used  */
  int32_t begin, end, grouping;
  int32_t partitions;              /* classes, 1..64                                 */
  int32_t partvals;                /* partitions ^ dim(groupbook)                    */
  int32_t groupbook;
  int32_t stagebook[64][8];
} vb200_residue_decode;

typedef struct vb200_entropy_setup {
  int32_t nbooks;
  const vb200_codebook *books;     /* [nbooks], ci->decbooks                         */
  int32_t modebits;                /* bits of the mode number (private_state.modebits) */
  vb200_floor_decode   floor[2][VB200_MAX_SUBMAPS];     /* [W][submap], submaps[W] used */
  vb200_residue_decode residue[2][VB200_MAX_SUBMAPS];
} vb200_entropy_setup;

/* Copies everything and builds the device lookup tables.  Returns VB200_EINVAL for inconsistent input (a code
 * that is not a complete prefix code, except the single-entry length-1 book; a book index out of range; a
 * residue range or grouping that does not fit the block; partition counts that do not match the floor's posts)
 * and VB200_EIMPL for residue type 0 or a floor that is not type 1.  Replaces an earlier registration.  After it,
 * no value read from a packet can index outside a table or a row.                                             */
int vb200_decode_entropy_setup(vb200_ctx*, const vb200_entropy_setup*);

/* The entropy half of mapping0_inverse for nblocks packets, into the staging layout of vb200_decode_dsp:
 *   Wseq [nblocks]        block flag of each packet (its header already parsed by the caller)
 *   pkt_off [nblocks] int64, pkt_bytes [nblocks] int32: packet i is data[pkt_off[i] .. pkt_off[i]+pkt_bytes[i])
 *   res  at coef_off[i] + c*n_W/2: channel c's residue vector, zeroed and then decoded (n_W/2 floats)
 *   posts [nblocks][ch][VB200_FLOOR1_STRIDE]: fit_value as floor1_inverse1 returns it, zeros past the posts
 *         and in absent rows; present [nblocks][ch]: 0 where floor1_inverse1 returned NULL.
 * Decoding starts at bit 1 + modebits + (W ? 2 : 0).  Damaged and truncated packets decode as the reference
 * decodes them.  One kernel launch.  Host form: data_bytes and res_len give the sizes of data and res; returns
 * VB200_EINVAL for a null pointer, a packet outside data, a Wseq entry outside {0, 1} or a row outside res.  */
int vb200_decode_entropy_dev(vb200_ctx*, int nblocks, const int32_t *d_Wseq, const int64_t *d_pkt_off,
                             const int32_t *d_pkt_bytes, const uint8_t *d_data, const int64_t *d_coef_off,
                             float *d_res, int32_t *d_posts, int32_t *d_present, void *stream);
int vb200_decode_entropy    (vb200_ctx*, int nblocks, const int32_t *Wseq, const int64_t *pkt_off,
                             const int32_t *pkt_bytes, const uint8_t *data, int64_t data_bytes,
                             const int64_t *coef_off, float *res, int64_t res_len, int32_t *posts, int32_t *present);

/* vb200_decode_dsp_resume from the packets: the entropy decode fused in front of the de-coupling and floor
 * multiply, then the IMDCT and overlap-add.  Arguments as vb200_decode_dsp_resume with the packets (pkt_off,
 * pkt_bytes, data, indexed like Wseq) in place of posts / present; res is scratch laid out by coef_off.
 * Contract: the PCM and the carry equal vb200_decode_entropy followed by vb200_decode_dsp_resume, bit for bit,
 * at full and half rate.  Two kernel launches.  Needs a registered vb200_decode_entropy_setup (else
 * VB200_EINVAL).  _dev: checks its pointers only.  Host form: res_len floats of scratch are allocated on the
 * device; returns VB200_EINVAL as vb200_decode_dsp_resume does and for a packet outside data (data_bytes).   */
int vb200_decode_packets_resume_dev(vb200_ctx*, int nstreams, int nblk, const int32_t *d_count,
                                    const int32_t *d_Wseq, const int64_t *d_coef_off, float *d_res,
                                    const int64_t *d_pkt_off, const int32_t *d_pkt_bytes, const uint8_t *d_data,
                                    const int64_t *d_pcm_off, void *d_pcm, int pcm_s16, int64_t pcm_stride,
                                    const vb200_decode_carry *carry, void *stream);
int vb200_decode_packets_resume    (vb200_ctx*, int nstreams, int nblk, const int32_t *count, const int32_t *Wseq,
                                    const int64_t *coef_off, int64_t res_len, const int64_t *pkt_off,
                                    const int32_t *pkt_bytes, const uint8_t *data, int64_t data_bytes,
                                    const int64_t *pcm_off, void *pcm, int pcm_s16, int64_t pcm_stride,
                                    vb200_decode_carry *carry);

/* ---- whole streams from packets: what a stock decoder's vorbis_synthesis -> vorbis_synthesis_blockin ->
 * vorbis_synthesis_pcmout loop (examples/decoder_example.c) returns, for many streams in one call, on the device:
 * the packet headers, the drops, the entropy decode, mapping0_inverse's DSP, the overlap-add and blockin's sample
 * bookkeeping (lib/block.c:741-751, 835-941), with the PCM packed in stream order.
 *   npkt  [nstreams]: stream s passes npkt[s] (0..max_packets) packets, info[s*max_packets + k] for k < npkt[s]:
 *         data[offset .. offset+bytes) with granulepos, e_o_s and packetno as an ogg_packet carries them; choice is
 *         not read.  The layout vb200_encode_streams_packets returns, so its info and data can be passed straight in.
 *   carry [nstreams][vb200_decode_streams_carry_bytes], device memory in both forms: one decoder's state per stream
 *         (the overlap tail of every channel, the last block flag, v->sequence, v->granulepos, b->sample_count, and
 *         the mode, full or half rate, it belongs to).  vb200_decode_streams_carry_init is vorbis_synthesis_restart
 *         for nstreams consecutive carries (pass one stream's slot to restart that stream); it is synchronous.
 *   pcm_base [nstreams + 1] int64: stream s returns n_s = pcm_base[s+1] - pcm_base[s] samples at pcm + pcm_base[s]*ch,
 *         planar float [ch][n_s], or with pcm_s16 interleaved int16 [n_s][ch] converted as decoder_example does
 *         (floor(x*32767.f+.5f) clipped).  The samples are those the pcmout loop returns after each blockin, in order.
 *   out   [nstreams][max_packets]: packet k of stream s (entries past npkt[s] are not written).
 * The packet header is parsed as vorbis_synthesis parses it (lib/synthesis.c:41-71), with the mode layout of the
 * entropy setup: modes 0 and 1 have block flags 0 and 1.  A packet whose type bit is not 0 (an empty packet too) is
 * dropped as OV_ENOTAUDIO, a mode number >= 2 or a long block without its nW bit as OV_EBADPACKET; a dropped packet
 * changes nothing, so the next one sees a packetno gap as the stock decoder does.  Truncated and damaged packets
 * past the header decode as the reference decodes them.
 * When pcm_base[nstreams]*ch > pcm_cap (elements), no PCM is written and every carry stays as it was; pcm_base and
 * out are still filled, and the host form returns VB200_EINVAL.  sum(npkt[s]) * ((blocksizes[1]/2) >> halfrate)
 * samples per channel never overflow.
 * Contract: any cut of a stream's packets into calls that pass the carry along gives the PCM, out and pcm_base of
 * one call, byte for byte (calls with no packets for some streams included); fed a stock decoder's packets the
 * result is that decoder's pcmout sequence, bit for bit.  Full rate, and half rate after vb200_synthesis_halfrate.
 * Needs a registered vb200_decode_entropy_setup (else VB200_EINVAL).  Five kernel launches per call, whatever
 * nstreams and the packet counts: header parse, per-stream plan, prefix scan, entropy decode + DSP, synthesis.
 * Device scratch (arena of its own, carved once per call): nstreams*max_packets*(ch*blocksizes[1]/2 floats of
 * residue + 48 bytes of tables) + nstreams*48 bytes.
 * _dev: every pointer is device memory; checks its pointers only.  Host form: host buffers except the carry;
 * returns VB200_EINVAL for null pointers, max_packets < 1, npkt[s] outside [0, max_packets], a packet outside
 * data (data_bytes), and a carry of the other rate mode (or not written by carry_init).                         */
typedef struct vb200_decoded_packet {
  int64_t pcm_offset;   /* first sample of this packet's PCM within stream s's output of this call */
  int64_t granulepos;   /* v->granulepos after this packet's blockin; -1 = not known */
  int32_t samples;      /* what vorbis_synthesis_pcmout returns after this packet's blockin */
  int32_t status;       /* 0, or VB200_ENOTAUDIO / VB200_EBADPACKET where vorbis_synthesis rejects it (dropped) */
} vb200_decoded_packet;
#define VB200_ENOTAUDIO  (-135)   /* OV_ENOTAUDIO  */
#define VB200_EBADPACKET (-136)   /* OV_EBADPACKET */
struct vb200_packet_info;         /* defined with vb200_encode_streams_packets below */
int vb200_decode_streams_carry_bytes(vb200_ctx*);
int vb200_decode_streams_carry_init (vb200_ctx*, int nstreams, void *d_carry);
int vb200_decode_streams_packets_dev(vb200_ctx*, int nstreams, int max_packets, const int32_t *d_npkt,
                                     const struct vb200_packet_info *d_info, const uint8_t *d_data, void *d_carry,
                                     int pcm_s16, void *d_pcm, int64_t pcm_cap, int64_t *d_pcm_base,
                                     vb200_decoded_packet *d_out, void *stream);
int vb200_decode_streams_packets    (vb200_ctx*, int nstreams, int max_packets, const int32_t *npkt,
                                     const struct vb200_packet_info *info, const uint8_t *data, int64_t data_bytes,
                                     void *d_carry, int pcm_s16, void *pcm, int64_t pcm_cap, int64_t *pcm_base,
                                     vb200_decoded_packet *out);

/* ---- sample ranges from packets: random access into many streams without decoding them whole (what vorbisfile's
 * ov_pcm_seek + ov_read give one stream, without Ogg pages).  The inputs are those of vb200_decode_streams_packets:
 * each stream given from its first packet, so vb200_encode_streams_packets' info and data go straight in; header
 * packets passed in are dropped as OV_ENOTAUDIO.  Modes, floors and residue types are limited as there, and a
 * registered vb200_decode_entropy_setup is needed (else VB200_EINVAL).  Full rate, and half rate after
 * vb200_synthesis_halfrate.
 *
 * vb200_decode_streams_index[_dev]: the bookkeeping alone.  length[s] = the samples a fresh-carry
 * vb200_decode_streams_packets call returns for stream s; out[s*max_packets + k] = its vb200_decoded_packet for
 * packet k (pcm_offset, samples, granulepos, status), byte for byte.  No PCM, no carry, no residue scratch; two
 * kernel launches (header parse, plan).  Device scratch (arena of its own with the ranges call, carved once per
 * call): nstreams*max_packets*40 + nstreams*80 bytes.
 *
 * vb200_decode_ranges[_dev]: request r is samples [start, start + length) of stream `stream`'s output, counted as a
 * fresh-carry vb200_decode_streams_packets call counts them (every pcmout sample, after the front and end trims).
 * Its samples equal that slice bit for bit, for every stream that call accepts (dropped, truncated and empty
 * packets, packetno gaps, beginning trims, granulepos on every packet or on page-final packets only).  Requests may
 * come in any order, name one stream several times and overlap.  Only the blocks that finish the range's samples
 * are decoded, after the one block before them, which primes the overlap.
 *   pcm   float planar [nreq][ch][out_stride], or with pcm_s16 interleaved int16 [nreq][out_stride][ch] converted
 *         as decoder_example does.  Row r holds got[r] samples from index 0 and zeros after them.
 *   got   [nreq]: min(length, max(0, length_s - start)), so 0 for a start at or past the stream's end; or
 *         VB200_EINVAL for a request whose stream, start or length is out of range (the _dev form checks them per
 *         request) or that needs more blocks than its scratch holds (below).  Such a row is all zero.
 * Capacity: a request's scratch is fixed by out_stride: (out_stride << halfrate) / (blocksizes[0]/2) + 3 blocks and
 * ch * (2 * (out_stride << halfrate) + 3 * blocksizes[1]/2) floats of residue, rounded up to a multiple of 64.  That
 * holds every range of a stream whose blocks return all the samples they finish away from its ends; a crafted stream
 * (a packetno gap followed by a granulepos far behind the count) can need more, which gives got[r] = VB200_EINVAL
 * and nothing written out of bounds.  A larger out_stride serves such a request.  Device scratch (arena of its own,
 * carved once per call): nreq*(blocks*40 + 12 bytes + residue floats*4 bytes).  Three kernel launches per call
 * (plan, entropy decode + DSP, synthesis) whatever nreq and nstreams are, after a memset of the output rows.  The
 * plan of a request walks its stream's packets from the first to the range's end, so its cost does not grow with
 * other streams or with packets past the range.
 * _dev: every pointer is device memory; asynchronous; checks its pointers, max_packets >= 1, nreq >= 0 and
 * out_stride >= 0 only.  Host forms: host buffers; return VB200_EINVAL for null pointers, nreq < 0, max_packets < 1,
 * npkt[s] outside [0, max_packets], a packet outside data (data_bytes), a request's stream outside [0, nstreams),
 * start < 0 or length outside [0, out_stride].                                                                  */
typedef struct vb200_pcm_range {
  int64_t start;
  int32_t stream;
  int32_t length;       /* 0 .. out_stride */
} vb200_pcm_range;
int vb200_decode_streams_index_dev(vb200_ctx*, int nstreams, int max_packets, const int32_t *d_npkt,
                                   const struct vb200_packet_info *d_info, const uint8_t *d_data,
                                   int64_t *d_length, vb200_decoded_packet *d_out, void *stream);
int vb200_decode_streams_index    (vb200_ctx*, int nstreams, int max_packets, const int32_t *npkt,
                                   const struct vb200_packet_info *info, const uint8_t *data, int64_t data_bytes,
                                   int64_t *length, vb200_decoded_packet *out);
int vb200_decode_ranges_dev(vb200_ctx*, int nstreams, int max_packets, const int32_t *d_npkt,
                            const struct vb200_packet_info *d_info, const uint8_t *d_data,
                            int nreq, const vb200_pcm_range *d_req, int pcm_s16, void *d_pcm, int32_t out_stride,
                            int32_t *d_got, void *stream);
int vb200_decode_ranges    (vb200_ctx*, int nstreams, int max_packets, const int32_t *npkt,
                            const struct vb200_packet_info *info, const uint8_t *data, int64_t data_bytes,
                            int nreq, const vb200_pcm_range *req, int pcm_s16, void *pcm, int32_t out_stride,
                            int32_t *got);

/* ---- encode: the entropy coding of mapping0_forward (lib/mapping0.c:596-687) on the device, un-managed bitrate.
 * What floor1_encode (lib/floor1.c:753-921) and the residue class / forward of types 1 and 2 (lib/res0.c:534-648,
 * 725-809) read, registered on a context with vb200_encode_entropy_setup.
 *
 * vb200_enc_codebook: one codebook as the encoder uses it (codec_setup_info.fullbooks).  Entry i has the codeword
 * codeword[i] of length[i] bits (0 = unused entry), written LSb first as oggpack_write(codeword[i], length[i])
 * writes it; minval / delta / quantvals are the integer lattice of a residue stage book (book->minval, ->delta,
 * ->quantvals; 0 for books without a value mapping).                                                           */
typedef struct vb200_enc_codebook {
  int32_t dim;
  int32_t entries;
  const uint8_t  *length;          /* [entries] c->lengthlist                        */
  const uint32_t *codeword;        /* [entries] book->codelist                       */
  int32_t minval, delta, quantvals;
} vb200_enc_codebook;

/* floor[W][submap] and residue[W][submap] carry exactly the fields the encoder reads; their layout is the decoder's
 * (stagebook[class][stage] as res0_look lays out partbooks, -1 where the stage bit is clear).  The struct shares
 * its name with the function that registers it, so C callers name it `struct vb200_encode_entropy_setup`. */
struct vb200_encode_entropy_setup {
  int32_t nbooks;
  const vb200_enc_codebook *books; /* [nbooks]                                       */
  int32_t modebits;                /* private_state.modebits                         */
  vb200_floor_decode   floor[2][VB200_MAX_SUBMAPS];
  vb200_residue_decode residue[2][VB200_MAX_SUBMAPS];
};

/* Copies and uploads everything.  Returns VB200_EINVAL for a book index out of range, a stage book with dim > 8,
 * quantvals <= 0 or a lattice larger than its entries, a codeword longer than 32 bits, a residue range that does
 * not fit the block or differs from the context's vb200_residue_setup (which classifies), a floor class with
 * class_dim > 8 or class_subs > 3, floor partitions that do not give the floor's posts; VB200_EIMPL for residue
 * type 0 or a floor that is not type 1.  Unused entries (length 0) are legal.  Replaces an earlier registration. */
int vb200_encode_entropy_setup(vb200_ctx*, const struct vb200_encode_entropy_setup*);

/* Worst-case bytes of one packet of block size W under the registered setup, a multiple of 4: the header, per
 * channel 1 + 2*ilog(quant_q-1) bits and the longest class and sub-book codewords of every partition, and per
 * residue stage the longest phrase codeword per partition word plus grouping/dim times the longest codeword of
 * the stage's class books per partition.  < 0: no setup registered (VB200_EINVAL).                              */
int vb200_encode_packet_bound(vb200_ctx*, int W);

/* The packets of nblocks blocks of size W (what mapping0_forward writes into packetblob[PACKETBLOBS/2]): packet
 * type bit, mode W in modebits bits, lW / nW for long blocks, the floor of every channel, then classification and
 * residue per submap.  byte-identical to the reference.
 *   desc    [nblocks]          lW / nW of every block (blocktype and ampmax are not read)
 *   posts   [nblocks][ch][VB200_FLOOR1_STRIDE], nonzero [nblocks][ch], iwork [nblocks][ch][n] int32: exactly
 *           what vb200_encode_dsp returns (a silent channel is an all-zero posts row); iwork is not modified.
 * _dev: block b goes to data + b*pkt_stride and pkt_bits[b] is its length in bits; pkt_stride must be a multiple
 *       of 4 and >= vb200_encode_packet_bound(W).  Two kernel launches (classification, then the coder).
 * Host form: packets back to back, block b at data + pkt_off[b] (int64 bytes), (pkt_bits[b] + 7) / 8 bytes long;
 *       only the packet bytes and the per-block counts are copied back.  If they do not fit data_cap bytes it returns
 *       VB200_EINVAL with pkt_bits filled (as count > cap does for vb200_encode_streams).  Four kernel launches.
 * Without a registered setup, all of these return VB200_EINVAL.                                                  */
int vb200_encode_entropy_dev(vb200_ctx*, int W, int nblocks, const vb200_block_desc *d_desc, const int32_t *d_posts,
                             const int32_t *d_nonzero, const int32_t *d_iwork, int64_t pkt_stride, int32_t *d_pkt_bits,
                             uint8_t *d_data, void *stream);
int vb200_encode_entropy    (vb200_ctx*, int W, int nblocks, const vb200_block_desc *desc, const int32_t *posts,
                             const int32_t *nonzero, const int32_t *iwork, int64_t *pkt_off, int32_t *pkt_bits,
                             uint8_t *data, int64_t data_cap);

/* PCM in, packets out: vb200_encode_dsp's chain, then classification and entropy coding, in one synchronous round
 * trip (host buffers; no chunk pipeline).  io as for vb200_encode_dsp except that posts, nonzero, iwork, classes,
 * overflow, mdct, logmdct and logmask must be NULL (they stay in device scratch) and iwork_fmt must be
 * VB200_IWORK_S32; io->ampmax_out is filled.  Packed output as vb200_encode_entropy.  Launches: those of
 * vb200_encode_dsp on one batch plus four.  A caller with device buffers chains vb200_encode_dsp_dev and
 * vb200_encode_entropy_dev on one stream instead; there is no fused _dev form.                                   */
int vb200_encode_packets(vb200_ctx*, int W, int nstreams, int blocks_per_stream, int blobno, const vb200_encode_io *io,
                         int64_t *pkt_off, int32_t *pkt_bits, uint8_t *data, int64_t data_cap);

/* Bitrate-managed: all VB200_PACKETBLOBS packets of every block (what mapping0_forward writes into packetblob[0..14]
 * when vorbis_bitrate_managed), byte-identical to the reference; the bitrate manager then picks one of them.
 *   posts / nonzero / iwork  blob-major as vb200_encode_dsp_managed / vb200_encode_streams_managed write them: block b
 *           of curve k is row k*blob_blocks*ch + b*ch + channel, blob_blocks >= nblocks (nblocks for
 *           vb200_encode_dsp_managed, cap[W] for vb200_encode_streams_managed); rows past nblocks of a curve are never
 *           read.  A NULL curve (all-zero posts rows) codes as silent floors.
 * _dev: packet (k, b) goes to data + (k*nblocks + b)*pkt_stride and pkt_bits[k*nblocks + b] is its length in bits;
 *       pkt_stride as for vb200_encode_entropy_dev (the bound holds for every curve).  Two kernel launches
 *       (classification of all curves, then the coder); the scratch does not grow with the curve count.
 * vb200_encode_packets_managed: PCM in, packets out in one synchronous round trip; io as for vb200_encode_dsp_managed
 *       with posts, nonzero, iwork, classes, overflow and the spectra NULL; io->ampmax_out is filled.  Packet (k, b)
 *       at data + pkt_off[k*nblocks + b], (pkt_bits[k*nblocks + b] + 7) / 8 bytes; when they do not fit data_cap it
 *       returns VB200_EINVAL with pkt_bits filled.  Launches: those of vb200_encode_dsp_managed plus four.
 * VB200_EINVAL without a registered setup, for blob_blocks < nblocks, a bad pkt_stride and null pointers.       */
int vb200_encode_entropy_managed_dev(vb200_ctx*, int W, int nblocks, int64_t blob_blocks,
                                     const vb200_block_desc *d_desc, const int32_t *d_posts, const int32_t *d_nonzero,
                                     const int32_t *d_iwork, int64_t pkt_stride, int32_t *d_pkt_bits, uint8_t *d_data,
                                     void *stream);
int vb200_encode_packets_managed(vb200_ctx*, int W, int nstreams, int blocks_per_stream, const vb200_encode_io *io,
                                 int64_t *pkt_off, int32_t *pkt_bits, uint8_t *data, int64_t data_cap);

/* ---- the bitrate manager on the device: vorbis_bitrate_addblock (lib/bitrate.c:73-227), replayed exactly.
 * vb200_bitrate_info is bitrate_manager_info (lib/bitrate.h:41-50), what a binding reads from ci->bi.
 * vb200_bitrate_setup registers it on the context, which derives what vorbis_bitrate_init derives
 * (lib/bitrate.c:28-56) from it, the context's rate and its block sizes: avg/min/max_bitsper, short_per_long and
 * desired_fill.  reservoir_bits <= 0 is the un-managed case: the setup is kept, and every call below that manages
 * the rate returns VB200_EINVAL for it.  Replaces an earlier registration.                                      */
typedef struct vb200_bitrate_info {
  int64_t avg_rate;                /* bits/s; <= 0: no average target */
  int64_t min_rate;
  int64_t max_rate;
  int64_t reservoir_bits;
  double  reservoir_bias;
  double  slew_damp;
} vb200_bitrate_info;
/* The part of bitrate_manager_state (lib/bitrate.h:25-39) that changes from block to block. */
typedef struct vb200_bitrate_state {
  int64_t avg_reservoir;
  int64_t minmax_reservoir;
  double  avgfloat;
  int32_t choice;                  /* the last block's choice */
  int32_t pad;
} vb200_bitrate_state;
int vb200_bitrate_setup(vb200_ctx*, const vb200_bitrate_info*);
/* plain host code: the state vorbis_bitrate_init leaves (both reservoirs at desired_fill, avgfloat 7, choice 0) */
int vb200_bitrate_init(vb200_ctx*, vb200_bitrate_state *state);
/* The choice for count[s] blocks of each of nstreams streams, in stream order, one thread per stream:
 *   W        [nstreams][max_blocks]                      block-size flag of each block
 *   pkt_bits [nstreams][max_blocks][VB200_PACKETBLOBS]   the 15 packets' lengths in bits as the coder reports them
 *                                                        (rounded up to whole bytes, as oggpack_bytes does)
 *   state    [nstreams]                                  read and written in place
 *   choice   [nstreams][max_blocks]  the packet kept (bm->choice); bytes [nstreams][max_blocks] its final length:
 *            cut to maxsize bytes when even packet 0 is too large, padded with zero bytes up to minsize when the
 *            minimum demands it.
 * Entries past count[s] are neither read nor written.  Contract: cutting a stream's blocks into any sequence of
 * calls that carry the state along gives the result of one call.  One kernel launch.  VB200_EINVAL without a
 * managed vb200_bitrate_setup, for a null pointer, max_blocks < 1 or (host form) count[s] outside [0, max_blocks]. */
int vb200_bitrate_addblocks_dev(vb200_ctx*, int nstreams, int max_blocks, const int32_t *d_count, const int32_t *d_W,
                                const int32_t *d_pkt_bits, vb200_bitrate_state *d_state, int32_t *d_choice,
                                int32_t *d_bytes, void *stream);
int vb200_bitrate_addblocks    (vb200_ctx*, int nstreams, int max_blocks, const int32_t *count, const int32_t *W,
                                const int32_t *pkt_bits, vb200_bitrate_state *state, int32_t *choice, int32_t *bytes);

/* ---- whole streams to packets: what the vorbis_analysis_blockout -> vorbis_analysis -> vorbis_bitrate_addblock ->
 * vorbis_bitrate_flushpacket loop of a stock encoder hands its caller, for many fresh streams in one call.
 * vb200_encode_streams[_managed]_dev, vb200_encode_entropy[_managed]_dev per block size, then on the device: the
 * per-size bit counts moved into stream order through the plan, (managed) the chooser along every stream from
 * vorbis_bitrate_init's state, an offset scan over the final lengths and a gather of each kept packet from its
 * strided slot.  Only the plan, nblocks, info and the packed bytes are copied back.
 *   io    as for vb200_encode_streams, host buffers, with posts, nonzero, iwork and ampmax_out NULL (they stay in
 *         device scratch); plan, nblocks and count[] are returned as there
 *   info  [nstreams][max_blocks]: packet k of stream s is data[offset .. offset+bytes), streams back to back in
 *         stream order; e_o_s, granulepos and packetno as vorbis_bitrate_flushpacket sets them (lib/bitrate.c:
 *         229-252) from vorbis_analysis_blockout (lib/block.c:311, 618-619, 645-687): packetno = 3 + k, granulepos =
 *         the block's centre on the timeline minus blocksizes[1]/2, clipped at eof, e_o_s on the block whose centre
 *         reaches eof (never where eof is 0 or NULL); choice = the packet kept (VB200_PACKETBLOBS/2 un-managed).
 *         Entries past nblocks[s] are zero but for offset.
 * When the packets do not fit data_cap bytes: VB200_EINVAL with info filled (as vb200_encode_packets).  VB200_EINVAL
 * also without a registered vb200_encode_entropy_setup, (managed) without a managed vb200_bitrate_setup, and for null
 * pointers.  Launches: those of the streams call, two per block size with blocks, then three (un-managed) or four.
 * Device scratch of this call family, besides the staging of the streams call's io (posts, nonzero, iwork of cap[W]
 * blocks, times VB200_PACKETBLOBS managed): per block size, curves x count[W] x (vb200_encode_packet_bound(W) + 4)
 * bytes of strided packets and bit counts (curves = 1, or VB200_PACKETBLOBS managed), which dominates; then per
 * (stream, block) 4 x (curves + 3) + 8 + sizeof(vb200_packet_info) bytes, and data_cap bytes for the packed output.
 * Callers size their calls by that; nothing is cut into chunks.                                                  */
typedef struct vb200_packet_info {
  int64_t offset;
  int64_t granulepos;
  int32_t bytes;
  int32_t e_o_s;
  int32_t packetno;
  int32_t choice;
} vb200_packet_info;
int vb200_encode_streams_packets        (vb200_ctx*, int nstreams, int blobno, vb200_streams_io *io,
                                         vb200_packet_info *info, uint8_t *data, int64_t data_cap);
int vb200_encode_streams_packets_managed(vb200_ctx*, int nstreams, vb200_streams_io *io,
                                         vb200_packet_info *info, uint8_t *data, int64_t data_cap);

/* ---- whole streams to packets in pieces: the same calls with a carried per-stream encoder state, for PCM that arrives
 * over time.  The carry is [nstreams][vb200_encode_carry_bytes] bytes; each begins with a vb200_encode_carry head that
 * callers may read, the rest is opaque: the planner state of vorbis_analysis_blockout and the envelope search
 * (lib/block.c:534-689, lib/envelope.c:215-374: W, lW, centerW, ve->cursor, ve->curmark, ve->current and the eof
 * state), the envelope detector's VB200_VE_STATE_WORDS(ch) words, the window of ve->mark that _ve_envelope_shift keeps,
 * the ampmax chain (g->ampmax and the previous block's vbi->ampmax) and a vb200_bitrate_state.
 *   mark_steps  capacity of the mark window in 64-sample steps; <= 0 takes the default, (3*blocksizes[1]/2 +
 *               blocksizes[0]/4)/64 + 8, which holds every window a call leaves unless max_blocks cut it short.  A call
 *               cut by max_blocks keeps the marks of everything it analysed beyond the last block: about
 *               (pcm_len - consumed)/64 + 2 steps.  A call whose window would not fit returns VB200_EINVAL and leaves
 *               the carry as it was.
 *   vb200_encode_carry_init writes fresh carries: a fresh vorbis_dsp_state (base 0, packetno 3) and, when a managed
 *   vb200_bitrate_setup is registered, vorbis_bitrate_init's state (initialise after the setup for the managed form).
 * Per call, stream s passes timeline samples [base, base + pcm_len[s]) in io->pcm (the layouts of vb200_streams_io):
 * the samples the carry kept (the previous call's base + pcm_len minus the new base), then the new ones.  A stream with
 * no new data passes just what it kept.  eof[s] is in timeline samples (v->eofflag plus base), and is given only in
 * calls whose buffer ends at the end of the timeline (with the extrapolated tail of vorbis_analysis_wrote(v,0)); 0
 * before.  A stream whose carry is done is skipped and emits nothing.  LPC pre- and post-extrapolation stay with the
 * caller: the timeline is the one described at vb200_plan_blocks.
 * Output as vb200_encode_streams_packets: info and data hold this call's packets only, with absolute granulepos and
 * continuing packetno; plan[].pos is relative to this call's buffer (so int32 suffices for streams longer than 2^31
 * samples).  max_blocks may cut a call short; the carry records where planning stopped.
 * Contract: (a) a fresh carry with the whole timeline in one call gives vb200_encode_streams_packets[_managed]'s output;
 * (b) cutting a stream's timeline into any sequence of calls, at any sample, including calls with no new samples and
 * calls cut by max_blocks, gives the packets and infos of one call, byte for byte; (c) hence, fed the timeline of a
 * stock encoder written in chunks, the result is that encoder's packets, granulepos, e_o_s and packetno.
 * Errors: those of vb200_encode_streams_packets[_managed]; VB200_EINVAL for a null carry, a carry of another channel
 * count, block-size setup or mark capacity than stream 0's, (managed) a carry initialised before a managed
 * vb200_bitrate_setup, pcm_len[s] below what the carry kept, eof[s] at or before base, and a mark window overflow.  On any error the carries are left as they were.  The launches are those of the
 * fresh calls.  Device scratch: that of the fresh calls plus the carries and nstreams x (the steps analysed) bytes.  */
typedef struct vb200_encode_carry {
  int64_t base;        /* timeline sample where the next call's buffer for this stream starts (the sum of movementW) */
  int64_t granulepos;  /* the last packet's granulepos (0 before the first) */
  int32_t packetno;    /* the next packet's number (v->sequence) */
  int32_t done;        /* the e_o_s packet has been emitted */
} vb200_encode_carry;
int vb200_encode_carry_bytes(vb200_ctx*, int mark_steps);
int vb200_encode_carry_init (vb200_ctx*, int nstreams, int mark_steps, void *carry);
int vb200_encode_streams_packets_resume        (vb200_ctx*, int nstreams, int blobno, vb200_streams_io *io,
                                                void *carry, vb200_packet_info *info, uint8_t *data, int64_t data_cap);
int vb200_encode_streams_packets_managed_resume(vb200_ctx*, int nstreams, vb200_streams_io *io,
                                                void *carry, vb200_packet_info *info, uint8_t *data, int64_t data_cap);

/* ---- raw PCM to packets: the _resume calls fed the caller's PCM instead of a timeline.  The LPC pre-extrapolation of
 * vorbis_analysis_wrote (lib/block.c:426-466, 525: order 16 over all P samples written when more than blocksizes[1]
 * have been, time-reversed, predicting the blocksizes[1]/2 preamble samples; the guard P > 32) and its post-
 * extrapolation at the end (:474-514: order 32 over the timeline [eof - n, eof), n = min(eof - base, blocksizes[1]),
 * primed with the 32 samples before eof, predicting 3*blocksizes[1] samples; the guard eof - base > 64) run on the
 * device, bit for bit.  The carry is [nstreams][vb200_encode_pcm_carry_bytes] bytes; each begins with a readable
 * vb200_pcm_carry, the rest is opaque: an encode carry and, per channel, the 16 preamble coefficients with their 16
 * prime samples and the 32 tail coefficients with their 32 prime samples (filters, not samples: every call rebuilds
 * the preamble or tail part of its timeline by replaying vorbis_lpc_predict from them).  mark_steps as for
 * vb200_encode_carry_init; vb200_encode_pcm_carry_init after a managed vb200_bitrate_setup for the managed form.
 * Per call, stream s passes in io->pcm the input samples from its carry's raw_base: the ones it kept (written -
 * raw_base), then this call's new ones; pcm_len[s] counts both.
 * The write rule: one call is one vorbis_analysis_wrote(v, new) followed by the blockout loop of encoder_example.c,
 * run until it returns 0 (or max_blocks blocks).  A call with no new samples is a drain call.  A call with end[s]
 * nonzero is vorbis_analysis_wrote(v, 0): it brings no new samples, and the carry must be drained (the last call
 * planned fewer than max_blocks blocks for the stream).  Hence the packets, granulepos, e_o_s and packetno equal a
 * stock encoder's fed the same writes; more generally they equal those of any stock encoder whose writes cross
 * blocksizes[1] samples at the same count P (the write that does so fixes the preamble; the end's base is the drained
 * planner's and does not depend on the cuts).  Streams without a preamble yet plan nothing.
 *   pcm_fmt  VB200_PCM_F32_PLANAR [stream][ch][stream_stride] or VB200_PCM_S16_INTERLEAVED [stream][stream_stride][ch]
 *            (read as x/32768.f, as encoder_example.c converts)
 *   plan, nblocks, cap, count and the outputs as vb200_encode_streams_packets_resume; plan[].pos is relative to the
 *            call's timeline buffer, which starts at enc.base (the input starts at timeline sample blocksizes[1]/2).
 * Errors (VB200_EINVAL, every carry left as it was): those of the _resume calls, a pcm_fmt other than the two,
 * pcm_len[s] below the kept samples or above stream_stride, an end call with new samples, an end on an undrained
 * carry, a second end, and samples after the end.  Launches: four (the preamble filters, the timelines up to eof, the
 * tail filters, the tails) plus those of the _resume call, whatever the stream count.  Device scratch: that of the
 * _resume calls plus the input and nstreams x channels x (the longest timeline passed) floats.  Host pointers only. */
typedef struct vb200_pcm_carry {
  vb200_encode_carry enc;  /* the encode carry's head (base in timeline samples, granulepos, packetno, done) */
  int64_t raw_base;        /* input sample where the next call's buffer starts: max(0, enc.base - blocksizes[1]/2) */
  int64_t written;         /* input samples written so far */
  int32_t ended;           /* vorbis_analysis_wrote(v, 0) has been made */
  int32_t drained;         /* the last call planned fewer than max_blocks blocks for this stream (1 when fresh) */
} vb200_pcm_carry;
int vb200_encode_pcm_carry_bytes(vb200_ctx*, int mark_steps);
int vb200_encode_pcm_carry_init (vb200_ctx*, int nstreams, int mark_steps, void *carry);
typedef struct vb200_pcm_io {
  const void *pcm;
  int32_t pcm_fmt;
  int32_t max_blocks;
  int64_t stream_stride;
  const int64_t *pcm_len;      /* [nstreams] input samples from raw_base: the kept ones, then this call's new ones */
  const int32_t *end;          /* [nstreams] or NULL: nonzero = this call is vorbis_analysis_wrote(v, 0) */
  vb200_stream_block *plan;    /* [nstreams][max_blocks] out */
  int32_t *nblocks;            /* [nstreams] out */
  int32_t cap[2];
  int32_t count[2];            /* out */
} vb200_pcm_io;
int vb200_encode_pcm_packets        (vb200_ctx*, int nstreams, int blobno, vb200_pcm_io *io, void *carry,
                                     vb200_packet_info *info, uint8_t *data, int64_t data_cap);
int vb200_encode_pcm_packets_managed(vb200_ctx*, int nstreams, vb200_pcm_io *io, void *carry,
                                     vb200_packet_info *info, uint8_t *data, int64_t data_cap);
/* The stage call of those kernels: per row r, vorbis_lpc_from_data(data[r][0 .. n[r]), order) (lib/lpc.c:60-130), then
 * vorbis_lpc_predict of `count` samples continuing the window, primed with its last `order` samples (:132-159).
 * order 16 or 32; order <= n[r] <= data_stride; out_stride >= count.  coeff [nrows][order] and out [nrows][out_stride]
 * (the first count of each row written).  No guard: a row of silence takes the reference's epsilon exit.          */
int vb200_lpc_extrapolate(vb200_ctx*, int nrows, int order, const float *data, int64_t data_stride,
                          const int32_t *n, int32_t count, float *coeff, float *out, int64_t out_stride);

/* ---- device memory helpers for non-CUDA hosts (C callers) -------------- */
int  vb200_malloc_device(vb200_ctx*, size_t bytes, void **dptr);
int  vb200_free_device  (vb200_ctx*, void *dptr);
int  vb200_memcpy_h2d   (vb200_ctx*, void *dptr, const void *src, size_t bytes);
int  vb200_memcpy_d2h   (vb200_ctx*, void *dst, const void *dptr, size_t bytes);
int  vb200_synchronize  (vb200_ctx*);

#ifdef __cplusplus
}
#endif
#endif /* VORBIS_B200_H */
