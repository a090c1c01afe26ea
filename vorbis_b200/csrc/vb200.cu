// vb200.cu — kernels (__global__) and the C ABI of include/vorbis_b200.h.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false
//        -Xcompiler -fPIC -shared   (see __graft_entry__.build()).
// No torch, no oracle/ dependency: this is the product library.
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "vorbis_b200.h"
#include "vb200_tables.h"
#include "vb200_kernels.cuh"
#include "vb200_cqn.cuh"
#include "vb200_psy3.cuh"
#include "vb200_floor1.cuh"
#include "vb200_env.cuh"
#include "vb200_res.cuh"
#include "vb200_streams.cuh"
#include "vb200_managed.cuh"
#include "vb200_entropy_enc.cuh"
#include "vb200_bitrate.cuh"
#include "vb200_decode_streams.cuh"
#include "vb200_decode_ranges.cuh"
#include "vb200_lpc.cuh"
#include "vb200_pcm.cuh"
#include "vb200_ogg.cuh"
#include "vb200_ogg_ranges.cuh"
#include "vb200_headers.h"
#include "vb200_ogg_group.cuh"
#include "vb200_ogg_mux.cuh"
#include "floor1_db_table.h"

using namespace vb200;

// ======================================================================== //
// error plumbing
static thread_local std::string g_err;
static int fail(int code, const char *what, cudaError_t e = cudaSuccess) {
  g_err = what;
  if (e != cudaSuccess) { g_err += ": "; g_err += cudaGetErrorString(e); }
  return code;
}
#define CU(call)                                                         \
  do {                                                                   \
    cudaError_t e_ = (call);                                             \
    if (e_ != cudaSuccess) return fail(VB200_EFAULT, #call, e_);         \
  } while (0)

extern "C" const char *vb200_last_error(void) { return g_err.c_str(); }

// ======================================================================== //
// context
// a grow-only device buffer, freed with the context
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
};

constexpr int STAGE_SLOTS = 16;      // device buffers one host form may stage (HostIO)
constexpr int ENC_SETS = 4;          // buffer sets of the pipelined host forms (HostPipe)

struct vb200_ctx {
  int device = 0;
  int sm_count = 132;
  vb200_setup setup;                 // scalar copy (pointers not used after create)
  HostXform hx[2];
  XformDev dx[2];
  WinDev dwin;
  // half-rate decode (vb200_synthesis_halfrate): transforms at blocksizes[w]/2 and the half windows of those
  // sizes, built and uploaded the first time the mode is enabled
  bool halfrate = false, hs_built = false;
  HostXform hx_hs[2];
  XformDev dx_hs[2];
  WinDev dwin_hs;
  int n_psy = 0;
  HostPsyFlow hflow[4];
  PsyDev dpsy[4];
  std::vector<void *> owned;         // device allocations freed at destroy
  std::atomic<uint64_t> launches{0};
  // Device scratch: one arena (a grow-only buffer, cut into regions by carve()) per owning call family.  An arena
  // is carved at most once per call, and the arenas one call uses at the same time are different arenas.
  //   stage[]   HostIO: the device copies of a host form's inputs and outputs; nothing else uses it
  //   cycles    the debug cycle counters (VB200_PHASE_TIMING, VB200_FLOOR1_TIMING), kept between calls
  //   phaseA    phaseA_dev_common: log spectrum, row and block maxima
  //   enc       the encode chain of vb200_encode_dsp_dev and vb200_encode_packets
  //   set[]     HostPipe, one per buffer set, for both pipelined host forms: a chunk's copies and its intermediates
  //             (vb200_encode_dsp: its chain; vb200_analysis_phaseA: its maxima and the taps the caller asks for)
  //   mgd       vb200_encode_dsp_managed_dev
  //   plan      block planning: vb200_plan_blocks, and the envelope state, marks and plan tables of
  //             vb200_encode_streams[_managed]_dev
  //   chain     the chains of vb200_encode_streams[_managed]_dev, sized by the plan
  //   env_scratch  vb200_envelope_search[_dev] (c->env holds the detector's tables)
  //   coder     the entropy coder: residue classes and the per-CTA residue copies
  //   pack      the host forms of the entropy coder: packet offsets and the packed bytes
  //   spk       vb200_encode_streams_packets[_managed]: strided packets and bit counts of both sizes, the stream-order
  //             tables, offsets, packet infos and the packed bytes
  //   brc       the host form of vb200_bitrate_addblocks
  //   dsk       vb200_decode_streams_packets[_dev]: the packet headers, the block tables, the per-stream plan and the
  //             residue scratch, sized by nstreams x max_packets
  //   ptl       vb200_encode_pcm_packets[_managed][_dev]: the planar float timelines [nstreams][ch][tl_stride], the
  //             carries unpacked, the LPC jobs, and the posts / nonzero / iwork of cap[] blocks that the streams
  //             packets path writes
  //   drg       vb200_decode_streams_index[_dev]: the packet headers, the per-stream plan tables and fresh heads,
  //             sized by nstreams x max_packets; vb200_decode_ranges[_dev]: the per-request block tables and residue
  //             scratch, sized by nreq and out_stride; vb200_ogg_ranges[_dev]: the same and the per-request packet
  //             scratch, sized by nreq and pkt_cap
  DevBuf stage[STAGE_SLOTS], cycles, phaseA, enc, set[ENC_SETS], mgd, plan, chain, env_scratch, coder, pack,
      spk, brc, dsk, ptl, drg;
  const ResDev *d_res[2] = {nullptr, nullptr};        // [VB200_MAX_SUBMAPS] residue class parameters per block size
  int res_partvals[2] = {0, 0};
  EnvDev env;                        // envelope detector tables (N = 128 transform, windows, thresholds)
  int grid_div = 1;                  // see grid_for
  cudaStream_t s_split[2] = {nullptr, nullptr};       // vb200_encode_dsp_dev: two concurrent half-batches
  cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
  // HostPipe: two compute streams and one stream per copy direction, ordered by events per buffer set (see there)
  cudaStream_t s_enc[3] = {nullptr, nullptr, nullptr};   // compute 0, compute 1, host->device
  cudaStream_t s_d2h = nullptr;
  cudaEvent_t ev_h2d[ENC_SETS] = {}, ev_cmp[ENC_SETS] = {}, ev_d2h[ENC_SETS] = {};
  bool psy_carveout_set = false;     // the generic psy kernel's shared-memory carve-out is set for this context
  // The *_dev entry points keep their intermediates in per-context scratch: two calls in flight on different
  // user streams would share it.  Every such call waits for the previous one's event and records its own.
  cudaEvent_t ev_scratch = nullptr;
  bool scratch_busy = false;
  const float *d_fromdB = nullptr;
  const int *d_mag[2] = {nullptr, nullptr}, *d_ang[2] = {nullptr, nullptr};
  const Floor1Dev *d_floor[2] = {nullptr, nullptr};   // [VB200_MAX_SUBMAPS] per block size
  const unsigned char *d_chmux[2] = {nullptr, nullptr};
  cudaStream_t s_main = nullptr;
  // vb200_decode_entropy_setup: the device tables of the entropy decoders (ent.books == nullptr: none registered)
  EntDev ent{};
  std::vector<void *> ent_owned;
  // vb200_encode_entropy_setup: the tables of the entropy coder (eent.books == nullptr: none registered)
  EncEntDev eent{};
  std::vector<void *> eent_owned;
  // vb200_bitrate_setup: what vorbis_bitrate_init derives (br_set: registered; br_managed: reservoir_bits > 0)
  bool br_set = false, br_managed = false;
  BitrateDev br{};
  std::mutex mu;
  // optional per-kernel timing of the last Phase-A call (bench roofline evidence)
  bool profiling = false;
  cudaEvent_t ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
};

static int scratch_begin(vb200_ctx *c, cudaStream_t st) {
  if (c->scratch_busy) CU(cudaStreamWaitEvent(st, c->ev_scratch, 0));
  return 0;
}
static int scratch_end(vb200_ctx *c, cudaStream_t st) {
  CU(cudaEventRecord(c->ev_scratch, st));
  c->scratch_busy = true;
  return 0;
}

// a device copy of src[count] in *dst, freed with the tables of `owned`
template <class T>
static int upload(std::vector<void *> &owned, const T *src, size_t count, const T **dst) {
  void *d = nullptr;
  size_t bytes = sizeof(T) * (count ? count : 1);
  CU(cudaMalloc(&d, bytes));
  owned.push_back(d);
  if (count) CU(cudaMemcpy(d, src, sizeof(T) * count, cudaMemcpyHostToDevice));
  *dst = reinterpret_cast<const T *>(d);
  return 0;
}

static int ensure_buf(DevBuf &b, size_t bytes, void **out) {
  if (b.cap < bytes) {
    if (b.p) CU(cudaFree(b.p));
    b.p = nullptr; b.cap = 0;
    CU(cudaMalloc(&b.p, bytes));
    b.cap = bytes;
  }
  *out = b.p;
  return 0;
}

// One call's regions of an arena.  carve() runs the layout twice: first to sum the sizes, then, once the arena
// holds that sum, to hand out the pointers.  Every region starts on a 256-byte boundary, as a cudaMalloc'd buffer
// does: the int4 / short4 loads of k_pack_s16 and the floor fit's four-lines-per-load path rely on it.
struct Carve {
  char *base;
  size_t off;
  template <class T> T *take(size_t n) {
    T *p = base ? (T *)(base + off) : nullptr;
    off += (sizeof(T) * n + 255) & ~(size_t)255;
    return p;
  }
};

template <class F> static int carve(DevBuf &arena, F &&layout) {
  Carve sizes{nullptr, 0};
  layout(sizes);
  void *p; int rc;
  if ((rc = ensure_buf(arena, sizes.off, &p))) return rc;
  Carve place{(char *)p, 0};
  layout(place);
  return 0;
}

extern "C" int vb200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

static bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

// mdct_init (and the window / FFT tables) of one block size: host tables into h, device copies into d
static int xform_upload(vb200_ctx *c, int N, const float *window, HostXform &h, XformDev &d) {
  build_xform(h, N, window);
  memset(&d, 0, sizeof(d));
  d.N = h.N; d.log2n = h.log2n; d.nst = h.log2n - 6; d.nf = h.nf; d.scale = h.scale;
  for (int i = 0; i < h.nf && i < 8; i++) d.fac[i] = h.fac[i];
  for (size_t i = 0; i < h.stage_off.size() && i < 8; i++) d.stage_off[i] = h.stage_off[i];
  int rc;
  if ((rc = upload(c->owned, h.trig.data(), h.trig.size(), &d.trig))) return rc;
  if ((rc = upload(c->owned, h.bitrev.data(), h.bitrev.size(), &d.bitrev))) return rc;
  const float *tw = nullptr;
  if ((rc = upload(c->owned, h.stage_tw.data(), h.stage_tw.size(), &tw))) return rc;
  d.stage_tw = reinterpret_cast<const float2 *>(tw);
  if ((rc = upload(c->owned, h.win.data(), h.win.size(), &d.win))) return rc;
  return upload(c->owned, h.wa.data(), h.wa.size(), &d.wa);
}

extern "C" void vb200_ctx_destroy(vb200_ctx *c);
// everything of vb200_ctx_create that can fail after the context exists; the caller destroys *c on failure
static int ctx_build(vb200_ctx *c, const vb200_setup *s, int device) {
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  CU(cudaStreamCreateWithFlags(&c->s_main, cudaStreamNonBlocking));
  for (auto &st : c->s_enc) CU(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking));
  for (auto &e : c->ev_h2d) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto &e : c->ev_cmp) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto &e : c->ev_d2h) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto &st : c->s_split) CU(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  CU(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&c->ev_scratch, cudaEventDisableTiming));
  for (auto &e : c->ev_join) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));

  for (int w = 0; w < 2; w++) {
    int rc;
    if ((rc = xform_upload(c, s->blocksizes[w], s->window[w], c->hx[w], c->dx[w]))) return rc;
    c->dwin.N[w] = c->hx[w].N;
    c->dwin.win[w] = c->dx[w].win;
  }
  for (int w = 0; w < 2; w++) {      // residue classification parameters (lib/backends.h:103-118)
    ResDev hr[VB200_MAX_SUBMAPS];
    memset(hr, 0, sizeof(hr));
    for (int sm = 0; sm < VB200_MAX_SUBMAPS; sm++) {
      const vb200_residue_setup &r = s->residue[w][sm];
      ResDev &d = hr[sm];
      d.type = -1;
      if (r.type < 0 || r.grouping <= 0) continue;         // not provided (zero-initialised setups: grouping 0)
      if (r.type > 2 || r.begin < 0 || r.end < r.begin || r.partitions < 1 || r.partitions > 64)
        return fail(VB200_EINVAL, "residue setup");
      d.type = r.type; d.begin = r.begin; d.end = r.end; d.grouping = r.grouping; d.partitions = r.partitions;
      d.partvals = (r.end - r.begin) / r.grouping;
      d.scale = (float)(100. / r.grouping);
      for (int k = 0; k < 64; k++) { d.cm1[k] = r.classmetric1[k]; d.cm2[k] = r.classmetric2[k]; }
      if (d.partvals > c->res_partvals[w]) c->res_partvals[w] = d.partvals;
    }
    int rc;
    if ((rc = upload(c->owned, hr, (size_t)VB200_MAX_SUBMAPS, &c->d_res[w]))) return rc;
  }
  {
    // envelope detector lookups, _ve_envelope_init (lib/envelope.c:31-74)
    HostXform h;
    build_xform(h, ENV_N, nullptr);
    EnvDev &E = c->env;
    memset(&E, 0, sizeof(E));
    XformDev &d = E.X;
    d.N = h.N; d.log2n = h.log2n; d.nst = h.log2n - 6; d.nf = h.nf; d.scale = h.scale;
    for (size_t i = 0; i < h.stage_off.size() && i < 8; i++) d.stage_off[i] = h.stage_off[i];
    int rc;
    if ((rc = upload(c->owned, h.trig.data(), h.trig.size(), &d.trig))) return rc;
    if ((rc = upload(c->owned, h.bitrev.data(), h.bitrev.size(), &d.bitrev))) return rc;
    const float *tw = nullptr;
    if ((rc = upload(c->owned, h.stage_tw.data(), h.stage_tw.size(), &tw))) return rc;
    d.stage_tw = reinterpret_cast<const float2 *>(tw);
    float win[ENV_N];
    for (int i = 0; i < ENV_N; i++) {
      win[i] = (float)std::sin(i / (ENV_N - 1.) * M_PI);
      win[i] = win[i] * win[i];
    }
    if ((rc = upload(c->owned, win, (size_t)ENV_N, &E.win))) return rc;
    static const int B[VB200_VE_BANDS] = {2, 4, 6, 9, 13, 17, 22}, En[VB200_VE_BANDS] = {4, 5, 6, 8, 8, 8, 8};
    float bwin[VB200_VE_BANDS * 8] = {0};
    for (int j = 0; j < VB200_VE_BANDS; j++) {
      float total = 0.f;
      for (int i = 0; i < En[j]; i++) {
        bwin[j * 8 + i] = (float)std::sin((i + .5) / En[j] * M_PI);
        total = total + bwin[j * 8 + i];
      }
      E.total[j] = (float)(1. / (double)total);
      E.begin[j] = B[j]; E.end[j] = En[j];
      E.preecho[j] = s->preecho_thresh[j]; E.postecho[j] = s->postecho_thresh[j];
    }
    if ((rc = upload(c->owned, bwin, (size_t)VB200_VE_BANDS * 8, &E.bwin))) return rc;
    E.stretch_penalty = s->stretch_penalty; E.minenergy = s->preecho_minenergy;
  }
  {
    int rc;
    if ((rc = upload(c->owned, VB_FLOOR1_FROMDB, (size_t)256, &c->d_fromdB))) return rc;
    for (int w = 0; w < 2; w++) {                      // the map was checked by vb200_ctx_create
      if ((rc = upload(c->owned, (const int *)s->coupling_mag[w], (size_t)s->coupling_steps[w], &c->d_mag[w]))) return rc;
      if ((rc = upload(c->owned, (const int *)s->coupling_ang[w], (size_t)s->coupling_steps[w], &c->d_ang[w]))) return rc;
    }
  }
  c->n_psy = s->n_psy;
  for (int i = 0; i < s->n_psy; i++) {
    const vb200_psy_setup &p = s->psy[i];
    if (!p.ath || !p.octave || !p.bark || !p.tonecurves || !p.noiseoffset)
      return fail(VB200_EINVAL, "psy lookup tables missing");
    if (p.n != s->blocksizes[i >> 1] / 2) return fail(VB200_EINVAL, "psy n != blocksize/2");
    HostPsyFlow &f = c->hflow[i];
    build_psy_flow(f, p);
    PsyDev &d = c->dpsy[i];
    memset(&d, 0, sizeof(d));
    d.n = p.n; d.total = p.total_octave_lines; d.linesper = p.eighth_octave_lines;
    d.firstoc = p.firstoc; d.shiftoc = p.shiftoc;
    d.noisewindowfixed = p.noisewindowfixed;
    d.bark_first_extra = f.bark_first_extra; d.fixed_first_extra = f.fixed_first_extra;
    d.nruns = (int)f.run_lo.size(); d.ngrp = (int)f.grp.size() / 4; d.tail_lin0 = f.tail_lin0;
    d.ath_adjatt = p.ath_adjatt; d.ath_maxatt = p.ath_maxatt; d.tone_abs_limit = p.tone_abs_limit;
    d.noisemaxsupp = p.noisemaxsupp; d.max_curve_dB = p.max_curve_dB; d.m_val = p.m_val;
    for (int j = 0; j < 3; j++) d.tone_masteratt[j] = p.tone_masteratt[j];
    int rc;
    if ((rc = upload(c->owned, p.ath, p.n, &d.ath))) return rc;
    if ((rc = upload(c->owned, p.octave, p.n, &d.octave))) return rc;
    if ((rc = upload(c->owned, p.bark, p.n, &d.bark))) return rc;
    if ((rc = upload(c->owned, p.tonecurves, (size_t)VB200_P_BANDS * VB200_P_LEVELS * (VB200_EHMER_MAX + 2),
                     &d.tonecurves))) return rc;
    if ((rc = upload(c->owned, p.noiseoffset, (size_t)VB200_P_NOISECURVES * p.n, &d.noiseoffset))) return rc;
    if ((rc = upload(c->owned, p.noisecompand, (size_t)VB200_COMPAND_LEVELS, &d.noisecompand))) return rc;
    if ((1 << f.linesper_log2) != p.eighth_octave_lines)
      return fail(VB200_EIMPL, "eighth_octave_lines must be a power of two (lib/psy.h:108)");
    const int *dr = nullptr, *dg = nullptr, *dc = nullptr, *ds = nullptr;
    if ((rc = upload(c->owned, f.runinfo.data(), f.runinfo.size(), &dr))) return rc;
    if ((rc = upload(c->owned, f.grp.data(), f.grp.size(), &dg))) return rc;
    if ((rc = upload(c->owned, f.cls_run.data(), f.cls_run.size(), &dc))) return rc;
    if ((rc = upload(c->owned, f.slot_rng.data(), f.slot_rng.size(), &ds))) return rc;
    d.runinfo = reinterpret_cast<const int4 *>(dr);
    d.grps = reinterpret_cast<const int4 *>(dg);
    d.cls_run = reinterpret_cast<const int2 *>(dc);
    d.slot_rng = reinterpret_cast<const int2 *>(ds);
    d.linesper_log2 = f.linesper_log2;
    { const int *drr = nullptr, *dlg = nullptr;
      if ((rc = upload(c->owned, f.runrec.data(), f.runrec.size(), &drr))) return rc;
      if ((rc = upload(c->owned, f.long_grp.data(), f.long_grp.size(), &dlg))) return rc;
      d.runrec = reinterpret_cast<const int4 *>(drr); d.long_grp = dlg; d.nlong = (int)f.long_grp.size(); }
    { const short *db = nullptr; if ((rc = upload(c->owned, f.bin_grp.data(), f.bin_grp.size(), &db))) return rc; d.bin_grp = db; }
    if (p.eighth_octave_lines > 32) return fail(VB200_EIMPL, "eighth_octave_lines > 32");
    if (p.total_octave_lines >= 2048) return fail(VB200_EIMPL, "total_octave_lines >= 2048");
    { const int *dco = nullptr; if ((rc = upload(c->owned, f.cls_off.data(), f.cls_off.size(), &dco))) return rc; d.cls_off = dco; }
    d.max_cls_len = 0;
    for (size_t k = 0; k + 1 < f.cls_off.size(); k++) d.max_cls_len = std::max(d.max_cls_len, f.cls_off[k + 1] - f.cls_off[k]);
  }
  // floor 1 lookups: what floor1_look (lib/floor1.c:205-253) derives from the post list
  for (int w = 0; w < 2; w++) {
    Floor1Dev hf[VB200_MAX_SUBMAPS];
    memset(hf, 0, sizeof(hf));
    if (s->submaps[w] < 0 || s->submaps[w] > VB200_MAX_SUBMAPS) return fail(VB200_EINVAL, "submaps");
    for (int sm = 0; sm < VB200_MAX_SUBMAPS; sm++) {
      const vb200_floor1_setup &f = s->floor1[w][sm];
      Floor1Dev &d = hf[sm];
      if (f.posts == 0) continue;
      const int P = f.posts;
      if (P < 2 || P > VB200_VIF_POSIT + 2) return fail(VB200_EINVAL, "floor1 posts");
      if (f.mult < 1 || f.mult > 4) return fail(VB200_EINVAL, "floor1 mult");
      if (f.n < 1 || f.n > s->blocksizes[w] / 2 || f.postlist[0] != 0 || f.postlist[1] != f.n)
        return fail(VB200_EINVAL, "floor1 post list must start 0, n with n <= blocksize/2");
      for (int i = 0; i < P; i++) {
        if (f.postlist[i] < 0 || f.postlist[i] > f.n) return fail(VB200_EINVAL, "floor1 post out of range");
        for (int j = 0; j < i; j++)
          if (f.postlist[j] == f.postlist[i]) return fail(VB200_EINVAL, "floor1 posts must be distinct");
      }
      d.posts = P; d.n = f.n; d.mult = f.mult;
      d.maxover = f.maxover; d.maxunder = f.maxunder; d.maxerr = f.maxerr;
      d.twofitweight = f.twofitweight; d.twofitatten = f.twofitatten;
      d.int_thresh = f.maxover == (float)(int)f.maxover && f.maxunder == (float)(int)f.maxunder &&
                     fabsf(f.maxover) < 65536.f && fabsf(f.maxunder) < 65536.f;
      d.maxover_i = d.int_thresh ? (int)f.maxover : 0;
      d.maxunder_i = d.int_thresh ? (int)f.maxunder : 0;
      int order[VB200_VIF_POSIT + 2];
      for (int i = 0; i < P; i++) order[i] = i;
      std::sort(order, order + P, [&](int x, int y) { return f.postlist[x] < f.postlist[y]; });
      for (int i = 0; i < P; i++) {
        d.postlist[i] = (short)f.postlist[i];
        d.fwd[i] = (short)order[i];
        d.rev[order[i]] = (short)i;
        d.sorted[i] = (short)f.postlist[order[i]];
      }
      for (int i = 0; i < P - 2; i++) {                 // nearest already-coded posts on both sides
        int lo = 0, hi = 1, lx = 0, hx = f.n;
        const int cur = f.postlist[i + 2];
        for (int j = 0; j < i + 2; j++) {
          const int x = f.postlist[j];
          if (x > lx && x < cur) { lo = j; lx = x; }
          if (x < hx && x > cur) { hi = j; hx = x; }
        }
        d.lo[i] = (short)lo; d.hi[i] = (short)hi;
        d.prcp[i] = 1.f / (float)(hx - lx);             // render_point's divisor for post i+2 is static
      }
      {                                                 // dependency levels of the prediction passes
        int level[VB200_VIF_POSIT + 2], nl = 0, w = 0;
        level[0] = level[1] = -1;
        for (int i = 2; i < P; i++) {
          const int a = level[d.lo[i - 2]], b = level[d.hi[i - 2]];
          level[i] = (a > b ? a : b) + 1;
          if (level[i] + 1 > nl) nl = level[i] + 1;
        }
        d.nlevels = nl;
        for (int lv = 0; lv < nl; lv++) {
          d.lvl_start[lv] = (unsigned char)w;
          for (int i = 2; i < P; i++) if (level[i] == lv) d.lvl_order[w++] = (unsigned char)i;
        }
        d.lvl_start[nl] = (unsigned char)w;
      }
    }
    for (int k = 0; k < s->channels; k++) {
      const int sm = s->chmux[w][k];
      if (sm >= VB200_MAX_SUBMAPS) return fail(VB200_EINVAL, "chmux");
    }
    int rc;
    if ((rc = upload(c->owned, hf, (size_t)VB200_MAX_SUBMAPS, &c->d_floor[w]))) return rc;
    if ((rc = upload(c->owned, (const unsigned char *)s->chmux[w], (size_t)VB200_MAX_CHANNELS + 1, &c->d_chmux[w]))) return rc;
  }
  return 0;
}


extern "C" int vb200_ctx_create(const vb200_setup *s, int device, vb200_ctx **out) {
  if (!s || !out) return fail(VB200_EINVAL, "null argument");
  for (int w = 0; w < 2; w++)
    if (!pow2(s->blocksizes[w]) || s->blocksizes[w] < 64 || s->blocksizes[w] > 8192)
      return fail(VB200_EINVAL, "block sizes must be powers of two in [64,8192] (lib/info.c:227-228)");
  if (s->blocksizes[0] > s->blocksizes[1]) return fail(VB200_EINVAL, "blocksizes[0] > blocksizes[1]");
  if (s->n_psy != 0 && s->n_psy != 4) return fail(VB200_EIMPL, "n_psy must be 0 or 4");
  if (s->channels < 1 || s->channels > VB200_MAX_CHANNELS) return fail(VB200_EINVAL, "channels");
  // mapping0_unpack's checks (lib/mapping0.c:110-118): every kernel that couples or decouples indexes the block's
  // channel rows with these, so a map the stock decoder refuses gets no context
  for (int w = 0; w < 2; w++) {
    if (s->coupling_steps[w] < 0 || s->coupling_steps[w] > VB200_MAX_COUPLING) return fail(VB200_EINVAL, "coupling_steps");
    for (int k = 0; k < s->coupling_steps[w]; k++) {
      const int m = s->coupling_mag[w][k], a = s->coupling_ang[w][k];
      if (m < 0 || a < 0 || m == a || m >= s->channels || a >= s->channels) return fail(VB200_EINVAL, "coupling map");
    }
  }
  int ndev = 0;
  CU(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(VB200_EINVAL, "no such CUDA device");
  CU(cudaSetDevice(device));
  vb200_ctx *c = new vb200_ctx();
  c->device = device;
  c->setup = *s;
  const int rc = ctx_build(c, s, device);
  if (rc) { vb200_ctx_destroy(c); return rc; }      // streams, events and every table uploaded so far are released
  *out = c;
  return 0;
}

extern "C" void vb200_ctx_destroy(vb200_ctx *c) {
  if (!c) return;
  cudaSetDevice(c->device);
  for (void *p : c->owned) cudaFree(p);
  for (auto &st : c->s_split) if (st) cudaStreamDestroy(st);
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  for (auto &e : c->ev_join) if (e) cudaEventDestroy(e);
  for (auto &st : c->s_enc) if (st) cudaStreamDestroy(st);
  if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
  for (auto &e : c->ev_h2d) if (e) cudaEventDestroy(e);
  for (auto &e : c->ev_cmp) if (e) cudaEventDestroy(e);
  for (auto &e : c->ev_d2h) if (e) cudaEventDestroy(e);
  if (c->s_main) cudaStreamDestroy(c->s_main);
  for (auto &e : c->ev) if (e) cudaEventDestroy(e);
  if (c->ev_scratch) cudaEventDestroy(c->ev_scratch);
  for (void *p : c->ent_owned) cudaFree(p);
  for (void *p : c->eent_owned) cudaFree(p);
  delete c;                                            // the arenas free themselves (DevBuf)
}

extern "C" int vb200_ctx_table(vb200_ctx *c, int W, int which, void *dst, int cap) {
  if (!c || W < 0 || W > 1 || !dst) return VB200_EINVAL;
  const HostXform &h = c->hx[W];
  const void *src = nullptr; size_t cnt = 0, el = 4;
  switch (which) {
    case 0: src = h.trig.data(); cnt = h.trig.size(); break;
    case 1: src = h.bitrev.data(); cnt = h.bitrev.size(); break;
    case 2: src = h.win.data(); cnt = h.win.size(); break;
    case 3: src = h.wa.data(); cnt = h.wa.size(); break;
    default: return VB200_EINVAL;
  }
  if ((size_t)cap < cnt) return VB200_EINVAL;
  memcpy(dst, src, cnt * el);
  return (int)cnt;
}

extern "C" uint64_t vb200_launch_count(vb200_ctx *c) { return c ? c->launches.load() : 0; }

extern "C" int vb200_set_profiling(vb200_ctx *c, int on) {
  if (!c) return fail(VB200_EINVAL, "null context");
  CU(cudaSetDevice(c->device));
  if (on) for (auto &e : c->ev) if (!e) CU(cudaEventCreate(&e));
  c->profiling = on != 0;
  return 0;
}

// dev aid: per-phase cycle sums of k_phaseA_psy3 (its DBG instance) accumulated while VB200_PHASE_TIMING is set,
// and of k_floor1_fit (its DBG instance) while VB200_FLOOR1_TIMING is set
extern "C" int vb200_debug_phase_cycles(vb200_ctx *c, unsigned long long *out16, int reset) {
  if (!c || !out16) return fail(VB200_EINVAL, "null argument");
  CU(cudaSetDevice(c->device));
  void *p; int rc;
  if ((rc = ensure_buf(c->cycles, 16 * sizeof(unsigned long long), &p))) return rc;
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out16, p, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  if (reset) CU(cudaMemset(p, 0, 16 * sizeof(unsigned long long)));
  return 0;
}

extern "C" int vb200_phaseA_kernel_ms(vb200_ctx *c, float *ms3) {
  if (!c || !ms3 || !c->ev[0]) return fail(VB200_EINVAL, "profiling not enabled");
  CU(cudaSetDevice(c->device));
  CU(cudaEventSynchronize(c->ev[3]));
  for (int i = 0; i < 3; i++) CU(cudaEventElapsedTime(ms3 + i, c->ev[i], c->ev[i + 1]));
  return 0;
}

extern "C" int vb200_encode_dsp_kernel_ms(vb200_ctx *c, float *ms6) {
  if (!c || !ms6 || !c->ev[0]) return fail(VB200_EINVAL, "profiling not enabled");
  CU(cudaSetDevice(c->device));
  CU(cudaEventSynchronize(c->ev[6]));
  for (int i = 0; i < 6; i++) CU(cudaEventElapsedTime(ms6 + i, c->ev[i], c->ev[i + 1]));
  return 0;
}

// ======================================================================== //
// kernels

// config 2: batched mdct_forward.  One CTA per vector (grid-stride), the vector
// staged in shared memory with 128-bit coalesced loads.
template <int NC>
__global__ void __launch_bounds__(256)
k_mdct_forward(XformDev X, int nvec, const float *__restrict__ in, float *__restrict__ out) {
  extern __shared__ __align__(16) float sm[];
  const int N = NC ? NC : X.N, tid = threadIdx.x, nt = blockDim.x;
  // two input buffers: the NEXT vector of this CTA travels global -> shared with cp.async (LDGSTS, no registers)
  // while this one is transformed; the padded hand-over buffer keeps the bit-reverse gather conflict free
  float *sx[2] = {sm, sm + N};
  float *sw = sm + 2 * N, *pad = sm + 3 * N;
  auto stage = [&](float *dst, int v) {
    const float *src = in + (size_t)v * N;
    const unsigned d = smem_u32(dst);
    for (int i = tid; i < (N >> 2); i += nt) cp_async16(d + 16u * (unsigned)i, src + 4 * i);
    cp_async_commit();
  };
  int v = blockIdx.x, buf = 0;
  if (v < nvec) stage(sx[0], v);
  for (; v < nvec; v += gridDim.x, buf ^= 1) {
    cp_async_wait_all();
    __syncthreads();
    if (v + (int)gridDim.x < nvec) stage(sx[buf ^ 1], v + gridDim.x);
    dev_mdct_forward<NC>(X, sx[buf], sw, out + (size_t)v * (N >> 1), tid, nt, pad);
    __syncthreads();
  }
}

template <int NC>
__global__ void __launch_bounds__(256)
k_mdct_backward(XformDev X, int nvec, const float *__restrict__ in, float *__restrict__ out) {
  extern __shared__ __align__(16) float sm[];
  const int N = NC ? NC : X.N, n2 = N >> 1, tid = threadIdx.x, nt = blockDim.x;
  float *sin_ = sm, *so = sm + n2;         // n2 coefficients, N outputs
  for (int v = blockIdx.x; v < nvec; v += gridDim.x) {
    const float4 *src = reinterpret_cast<const float4 *>(in + (size_t)v * n2);
    for (int i = tid; i < (n2 >> 2); i += nt) reinterpret_cast<float4 *>(sin_)[i] = __ldg(src + i);
    __syncthreads();
    dev_mdct_backward<NC>(X, sin_, so, tid, nt);
    float4 *dst = reinterpret_cast<float4 *>(out + (size_t)v * N);
    for (int i = tid; i < (N >> 2); i += nt) dst[i] = reinterpret_cast<float4 *>(so)[i];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
k_apply_window(WinDev Wd, int W, int nvec, const int *__restrict__ lW, const int *__restrict__ nW,
               float *__restrict__ data) {
  const int N = Wd.N[W];
  for (int v = blockIdx.x; v < nvec; v += gridDim.x) {
    const int l = lW ? lW[v] : 0, r = nW ? nW[v] : 0;
    float *d = data + (size_t)v * N;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      bool z;
      const float g = dev_window_gain(Wd, W, l, r, i, z);
      d[i] = z ? 0.f : d[i] * g;
    }
  }
}

__global__ void __launch_bounds__(256)
k_drft_forward(XformDev X, int nvec, float *__restrict__ data) {
  extern __shared__ __align__(16) float sm[];
  const int N = X.N, tid = threadIdx.x, nt = blockDim.x;
  float *sa = sm, *sb = sm + fft_buf_floats(N);
  for (int v = blockIdx.x; v < nvec; v += gridDim.x) {
    float4 *g = reinterpret_cast<float4 *>(data + (size_t)v * N);
    for (int i = tid; i < (N >> 2); i += nt) reinterpret_cast<float4 *>(sa)[i] = g[i];
    __syncthreads();
    const float *r = dev_drft_forward<0>(X, sa, sb, tid, nt);
    float *gs = data + (size_t)v * N;
    for (int i = tid; i < N; i += nt) gs[i] = r[fft_idx(i)];
    __syncthreads();
  }
}

// ---- Phase A, kernel 1: per (block, channel) window + MDCT + FFT + log spectrum.
// Reads 4N bytes of PCM, writes mdct (2N), logfft (2N) and one local_ampmax.
// (first per-channel loop of mapping0_forward, lib/mapping0.c:254-360)
// where a row's N samples come from: block layout (fmt 0), or a contiguous per-stream buffer
// from which block k is the window starting at k*hop (lib/block.c:630-643), float planar or
// interleaved int16 (examples/encoder_example.c:196-201)
struct PcmSrc {
  const void *base;
  int fmt;                 // 0 blocks [row][N] f32, VB200_PCM_F32_PLANAR, VB200_PCM_S16_INTERLEAVED
  int bps, hop;
  long long stride;        // samples per channel per stream
  const int2 *blk_src;     // optional [blocks]: (stream, first sample) of every block instead of (blk / bps, k * hop)
};

// stream and first sample of block `blk`: equal-size runs (k * hop) or the planner's table
__device__ __forceinline__ void blk_origin(const PcmSrc &src, int blk, long long &st, long long &off) {
  if (src.blk_src) { const int2 o = __ldg(src.blk_src + blk); st = o.x; off = o.y; }
  else { const int s = blk / src.bps; st = s; off = (long long)(blk - s * src.bps) * src.hop; }
}

// the FFT ping-pong buffer is idle during the MDCT: it takes the padded fly output
__device__ __forceinline__ float *mdct_pad_buffer(float *sf) {
#ifdef VB200_NO_FLY_PAD
  (void)sf; return nullptr;
#else
  return sf;
#endif
}

#ifndef XF_MINB
#define XF_MINB 5
#endif
template <int NC>
__global__ void __launch_bounds__(256, XF_MINB)
k_phaseA_transform(XformDev X, WinDev Wd, int W, int ch, int nrows,
                   PcmSrc src, const vb200_block_desc *__restrict__ desc,
                   float *__restrict__ mdct, float *__restrict__ logfft, float *__restrict__ lmax) {
  extern __shared__ __align__(16) float sm[];
  __shared__ float s_red[8];
  const int N = NC ? NC : X.N, n = N >> 1, tid = threadIdx.x, nt = blockDim.x;
  float *sx = sm, *sw = sm + fft_buf_floats(N), *sf = sw + N;   // sx and sf double as the padded FFT ping-pong buffers
  const float scale = 4.f / (float)N;
  const float scale_dB = add345(todB_dev(scale));
  // The raw samples of the NEXT row travel global -> shared with cp.async (16-byte LDGSTS, no registers)
  // while this row is transformed; the window is applied on the shared -> shared pass that follows.
  // mode 0: nothing staged (unaligned source or channel layout without a vector path): direct loads
  // mode 1: N floats staged;  mode 2: N stereo int16 frames staged (this row keeps its channel)
  float *sraw = sf + fft_buf_floats(N);
  auto stage = [&](int r) -> int {
    const int b2 = r / ch, c = r - b2 * ch;
    const char *g = nullptr;
    int mode = 0;
    if (src.fmt == VB200_PCM_S16_INTERLEAVED) {
      long long st, off; blk_origin(src, b2, st, off);
      g = reinterpret_cast<const char *>(reinterpret_cast<const short *>(src.base) + (st * src.stride + off) * ch);
      mode = ch == 2 ? 2 : 0;
    } else {
      const float *pf = reinterpret_cast<const float *>(src.base);
      if (src.fmt == VB200_PCM_F32_PLANAR) {
        long long st, off; blk_origin(src, b2, st, off);
        pf += (st * ch + c) * src.stride + off;
      } else {
        pf += (size_t)r * N;
      }
      g = reinterpret_cast<const char *>(pf);
      mode = 1;
    }
    if (reinterpret_cast<uintptr_t>(g) & 15) mode = 0;
    if (mode) {
      const unsigned d = smem_u32(sraw);
      for (int v = tid; v < (N >> 2); v += nt) cp_async16(d + 16u * v, g + 16 * (size_t)v);
    }
    cp_async_commit();
    return mode;
  };
  int mode = blockIdx.x < nrows ? stage(blockIdx.x) : 0;
  for (int row = blockIdx.x; row < nrows; row += gridDim.x) {
    const int blk = row / ch;
    const int lW = desc[blk].lW, nW = desc[blk].nW;
    cp_async_wait_all();
    __syncthreads();
    if (mode == 1) {
      for (int v = tid; v < (N >> 2); v += nt)
        *reinterpret_cast<float4 *>(sx + 4 * v) = dev_window4(Wd, W, lW, nW, 4 * v, *reinterpret_cast<const float4 *>(sraw + 4 * v));
    } else if (mode == 2) {
      // stereo: four frames = one 128-bit word, this row keeps its channel's four samples
      const int sh = 16 * (row - blk * ch);
      for (int v = tid; v < (N >> 2); v += nt) {
        const int4 u = *reinterpret_cast<const int4 *>(sraw + 4 * v);
        const float4 x = make_float4((float)(short)((unsigned)u.x >> sh) / 32768.f, (float)(short)((unsigned)u.y >> sh) / 32768.f,
                                     (float)(short)((unsigned)u.z >> sh) / 32768.f, (float)(short)((unsigned)u.w >> sh) / 32768.f);
        *reinterpret_cast<float4 *>(sx + 4 * v) = dev_window4(Wd, W, lW, nW, 4 * v, x);
      }
    } else if (src.fmt == VB200_PCM_S16_INTERLEAVED) {
      const int c = row - blk * ch;
      long long st, off; blk_origin(src, blk, st, off);
      const short *p16 = reinterpret_cast<const short *>(src.base) + (st * src.stride + off) * ch + c;
      for (int i = tid; i < N; i += nt) {
        bool z;
        const float g = dev_window_gain(Wd, W, lW, nW, i, z);
        const float v = (float)__ldg(p16 + (long long)i * ch) / 32768.f;
        sx[i] = z ? 0.f : v * g;
      }
    } else {
      const float *pf = reinterpret_cast<const float *>(src.base);
      if (src.fmt == VB200_PCM_F32_PLANAR) {
        const int c = row - blk * ch;
        long long st, off; blk_origin(src, blk, st, off);
        pf += (st * ch + c) * src.stride + off;
      } else {
        pf += (size_t)row * N;
      }
      for (int i = tid; i < N; i += nt) {          // unaligned source: scalar loads
        bool z;
        const float g = dev_window_gain(Wd, W, lW, nW, i, z);
        sx[i] = z ? 0.f : __ldg(pf + i) * g;
      }
    }
    __syncthreads();
    mode = row + gridDim.x < nrows ? stage(row + gridDim.x) : 0;
    dev_mdct_forward<NC, (NC > 0)>(X, sx, sw, mdct + (size_t)row * n, tid, nt, mdct_pad_buffer(sf));
    const float *f = dev_drft_forward<NC>(X, sx, sf, tid, nt);
    // log spectrum + local maximum (lib/mapping0.c:310-345)
    float mx = -1e30f;
    float *lf = logfft + (size_t)row * n;
    for (int k = tid; k < n; k += nt) {
      float v;
      if (k == 0) {
        v = add345(scale_dB + todB_dev(f[fft_idx(0)]));
      } else {
        const float2 c = *reinterpret_cast<const float2 *>(f + fft_idx(2 * k - 1));   // aligned: shifted by one, padded
        const float re = c.x, im = c.y;
        const float t = re * re + im * im;
        v = add345(scale_dB + .5f * todB_dev(t));
      }
      lf[k] = v;
      mx = fmaxf(mx, v);
    }
    mx = warp_max(mx);
    if ((tid & 31) == 0) s_red[tid >> 5] = mx;
    __syncthreads();
    if (tid == 0) {
      float m = s_red[0];
      for (int w = 1; w < (nt >> 5); w++) m = fmaxf(m, s_red[w]);
      if (m > 0.f) m = 0.f;
      lmax[row] = m;
    }
    __syncthreads();
  }
}

// ---- ampmax: per-block global_ampmax.
// mode 0 (independent blocks): g[blk] = max(desc[blk].ampmax, locals)   (lib/mapping0.c:244,346)
// mode 1 (streams): the decay chain of vorbis_analysis_blockout (lib/block.c:626-628,
//   lib/psy.c:837-848), sequential per stream: one thread per stream.
__global__ void k_ampmax(int mode, int nstreams, int bps, int ch, const vb200_block_desc *__restrict__ desc,
                         const float *__restrict__ lmax, const float *__restrict__ amp0,
                         float secs_att, float *__restrict__ gmax) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nstreams) return;
  if (mode == 0) {
    float g = desc[s].ampmax;
    for (int c = 0; c < ch; c++) g = fmaxf(g, lmax[(size_t)s * ch + c]);
    gmax[s] = g;
    return;
  }
  float g = amp0 ? amp0[s] : -9999.f;
  float prev = g;
  for (int k = 0; k < bps; k++) {
    const size_t blk = (size_t)s * bps + k;
    if (prev > g) g = prev;
    g = g + secs_att;                      // amp += secs*ampmax_att_per_sec
    if (g < -9999.f) g = -9999.f;
    float o = g;
    for (int c = 0; c < ch; c++) o = fmaxf(o, lmax[blk * ch + c]);
    gmax[blk] = o;
    prev = o;
  }
}

// ---- Phase A, kernel 2: per (block, channel) logmdct, noise mask, tone mask, mix.
// (second per-channel loop of mapping0_forward, lib/mapping0.c:366-470)

// shared-memory carve-up for the psy kernels (floats)
struct PsySmem {
  float *logmdct, *noise, *scan, *fft;
  ToneSmem T;
};
__host__ __device__ inline size_t psy_smem_floats(int n, int total, int nruns) {
  const int tp = (total + 7) & ~7, rp = (nruns + 3) & ~3;
  size_t runs = 4 * (size_t)rp;                      // run_rec (int4), also hosts rec (tp shorts)
  if (runs < (size_t)tp / 2) runs = tp / 2;
  return (size_t)3 * n + 5 * (size_t)(n + 4) + 2 * (size_t)tp + tp / 2 + runs;
}
__device__ __forceinline__ PsySmem psy_carve(float *sm, int n, int total, int nruns) {
  const int tp = (total + 7) & ~7, rp = (nruns + 3) & ~3;
  PsySmem s;
  s.logmdct = sm; s.noise = s.logmdct + n; s.scan = s.noise + n;
  s.fft = s.scan + 5 * (n + 4);
  s.T.seed = s.fft + n;
  s.T.astk = s.T.seed + tp;
  s.T.pstk = reinterpret_cast<short *>(s.T.astk + tp);
  s.T.run_rec = reinterpret_cast<int4 *>(s.T.astk + tp + tp / 2);
  s.T.rec = reinterpret_cast<short *>(s.T.run_rec);
  (void)rp;
  return s;
}

#define PSY_THREADS 128
__global__ void __launch_bounds__(PSY_THREADS)
k_phaseA_psy(PsyDev P0, PsyDev P1, int ch, int nrows, PsyArgs A) {
  extern __shared__ __align__(16) float sm[];
  const int n = P0.n, ns = n + 4, tid = threadIdx.x, nt = PSY_THREADS;
  const int total = P0.total > P1.total ? P0.total : P1.total;
  const int nruns = P0.nruns > P1.nruns ? P0.nruns : P1.nruns;
  const PsySmem S = psy_carve(sm, n, total, nruns);
  const int warp = tid >> 5, lane = tid & 31;
  for (int row = blockIdx.x; row < nrows; row += gridDim.x) {
    const int blk = row / ch;
    const PsyDev &P = A.desc[blk].blocktype ? P1 : P0;
    const float *gm = A.mdct_in + (size_t)row * n;
    const float *lf = A.logfft + (size_t)row * n;
    const float g = A.gmax[blk], lmax = A.lmax[row];
    for (int i = tid; i < n; i += nt) {
      const float l = add345(todB_dev(gm[i]));          // lib/mapping0.c:384-385
      S.logmdct[i] = l;
      A.logmdct[(size_t)row * n + i] = l;
      S.fft[i] = lf[i];
    }
    __syncthreads();
    // all warps: run peaks / curve choice, and the first pass' per-bin sum terms
    dev_tone_runs(P, S.fft, g, lmax, S.T, tid, nt);
    dev_noise_terms(n, S.logmdct, nullptr, 140.f, S.scan, ns, tid, nt);
    __syncthreads();
    dev_tone_slots(P, S.T, tid, nt);
    __syncthreads();
    // warp 0: the sequential seed_chase + gather; warps 1-3: the noise mask (two sequential
    // prefix-sum passes on five lanes + regressions).  The two chains are independent.
    if (warp == 0) dev_tone_chase_gather(P, S.fft, lmax, S.T, lane);
    else dev_noisemask(P, S.logmdct, S.noise, S.scan, ns, tid - 32, nt - 32, 1, true);
    __syncthreads();
    const float *noff = P.noiseoffset + n;               // offset_select 1
    for (int i = tid; i < n; i += nt) {
      float m = gm[i];
      const float nz = S.noise[i], tn = S.fft[i];
      const float lm = dev_mix_bin(P, 1, nz, tn, __ldg(noff + i), S.logmdct[i], m);
      A.logmask[(size_t)row * n + i] = lm;
      A.mdct_out[(size_t)row * n + i] = m;
      if (A.tap_noise) A.tap_noise[(size_t)row * n + i] = nz;
      if (A.tap_tone) A.tap_tone[(size_t)row * n + i] = tn;
    }
    if (tid == 0 && (row % ch) == 0) A.ampmax_out[blk] = g;   // lib/mapping0.c:576
    __syncthreads();
  }
}

// ---- stage-isolated psy kernels (parity tests feed them the oracle's upstream vectors)
__global__ void __launch_bounds__(PSY_THREADS)
k_noisemask(PsyDev P, int nvec, const float *__restrict__ logmdct, float *__restrict__ noise) {
  extern __shared__ __align__(16) float sm[];
  const int n = P.n, ns = n + 4, tid = threadIdx.x, nt = PSY_THREADS;
  const PsySmem S = psy_carve(sm, n, P.total, P.nruns);
  for (int v = blockIdx.x; v < nvec; v += gridDim.x) {
    for (int i = tid; i < n; i += nt) S.logmdct[i] = logmdct[(size_t)v * n + i];
    __syncthreads();
    dev_noisemask(P, S.logmdct, S.noise, S.scan, ns, tid, nt, 0, false);
    for (int i = tid; i < n; i += nt) noise[(size_t)v * n + i] = S.noise[i];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(PSY_THREADS)
k_tonemask(PsyDev P, int nvec, const float *__restrict__ logfft, const float *__restrict__ gmax,
           const float *__restrict__ lmax, float *__restrict__ tone) {
  extern __shared__ __align__(16) float sm[];
  const int n = P.n, tid = threadIdx.x, nt = PSY_THREADS;
  const PsySmem S = psy_carve(sm, n, P.total, P.nruns);
  for (int v = blockIdx.x; v < nvec; v += gridDim.x) {
    for (int i = tid; i < n; i += nt) S.fft[i] = logfft[(size_t)v * n + i];
    __syncthreads();
    dev_tone_runs(P, S.fft, gmax[v], lmax[v], S.T, tid, nt);
    __syncthreads();
    dev_tone_slots(P, S.T, tid, nt);
    __syncthreads();
    if (tid < 32) dev_tone_chase_gather(P, S.fft, lmax[v], S.T, tid);
    __syncthreads();
    for (int i = tid; i < n; i += nt) tone[(size_t)v * n + i] = S.fft[i];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
k_offset_and_mix(PsyDev P, int nvec, int sel, const float *__restrict__ noise,
                 const float *__restrict__ tone, float *__restrict__ mdct,
                 const float *__restrict__ logmdct, float *__restrict__ logmask) {
  const int n = P.n;
  const size_t tot = (size_t)nvec * n;
  const float *noff = P.noiseoffset + (size_t)sel * n;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(e % n);
    float m = mdct[e];
    logmask[e] = dev_mix_bin(P, sel, noise[e], tone[e], __ldg(noff + i), logmdct[e], m);
    if (sel == 1) mdct[e] = m;
  }
}

// ---- decode: mdct_backward (lib/mapping0.c:792-795) + the windowed overlap-add of
// vorbis_synthesis_blockin (lib/block.c:767-823).  One CTA walks one (stream, channel)
// block by block; the previous block's second half stays in shared memory, so the only
// HBM traffic is the spectra in (2N) and the finished samples out (2N per channel-block).
// HS: half-rate decode (lib/block.c:182,197-198,735-842).  X0/X1/Wd are then the tables of the halved block
// sizes; the spectra keep the full-rate layout, so channel c of a block starts N_W/2 = X.N floats after
// channel c-1 and only its first X.N/2 lines are read.
// finished-sample sinks: planar float, or interleaved int16 as examples/decoder_example.c:250-262
struct SinkF32 {
  float *p;
  __device__ __forceinline__ void put(int i, float v) const { p[i] = v; }
};
struct SinkS16 {
  short *p; int ch;
  __device__ __forceinline__ void put(int i, float v) const {
    int val = (int)floorf(v * 32767.f + .5f);
    if (val > 32767) val = 32767;
    if (val < -32768) val = -32768;
    p[(long long)i * ch] = (short)val;
  }
};

// The four forms of the synthesis, one instance each per sink and rate:
// PLAIN (vb200_synthesis[_s16], vb200_decode_dsp): every stream decodes nblk blocks from a fresh state; block 0 primes.
// CARRY (vb200_decode_dsp_resume, vb200_decode_packets_resume): stream st decodes count[st] <= nblk blocks, and the
// overlap of every (stream, channel) = task comes from / goes back to carry_W[task] and
// carry_tail[task * tail_stride]: the block flag and the right half of the last IMDCT (what v->pcm holds after
// lib/block.c:817-823).  With a carried W >= 0, block 0 overlap-adds onto that tail and finishes samples like any
// later block; with -1 it only primes.  A stream with count 0 is not touched.  W is kept per (stream, channel)
// because the CTA of one channel must not read what the CTA of another channel of the same stream writes.
// TRIM (vb200_decode_streams_packets): as CARRY, with the carry of stream st in its slot of T.carry and the carried
// flag from T.W_in (what k_ds_plan read before anything wrote the heads); block k writes only [lo, hi) = T.win of
// its finished samples, from pcm_off (relative to the stream's pcm_base) on, into the packed layout of the call.
// Nothing is written, carries included, when the call's output does not fit T.cap.  Channel 0 commits the head.
// RANGE (vb200_decode_ranges): as TRIM, but every "stream" is a request that starts from a fresh state, so block 0
// primes; request r's row of the output is at T.base[r] = r * out_stride.  T.cap, T.W_in, T.head and the carries
// are neither read nor written.
// Arguments a form does not name are not read: carry_* in all but CARRY, pcm_stride in TRIM and RANGE, T in PLAIN
// and CARRY.
enum SynthMode { SYN_PLAIN, SYN_CARRY, SYN_TRIM, SYN_RANGE };

template <bool S16, bool HS, SynthMode MODE>
__global__ void __launch_bounds__(256)
k_synthesis(XformDev X0, XformDev X1, WinDev Wd, int ch, int nstreams, int nblk,
            const int *__restrict__ Wseq, const long long *__restrict__ coef_off,
            const float *__restrict__ coef, const long long *__restrict__ pcm_off,
            void *__restrict__ pcm_out, long long pcm_stride, const int *__restrict__ count,
            float *__restrict__ carry_tail, int *__restrict__ carry_W, int tail_stride, DsTrim T) {
  constexpr bool CARRY = MODE == SYN_CARRY, TRIM = MODE == SYN_TRIM || MODE == SYN_RANGE, FRESH = MODE == SYN_RANGE;
  extern __shared__ __align__(16) float sm[];
  const int tid = threadIdx.x, nt = blockDim.x;
  const int n0 = X0.N >> 1, n1 = X1.N >> 1;
  float *s_in = sm, *s_out = sm + n1, *s_prev = s_out + 2 * n1;
  const float *w0 = Wd.win[0], *w1 = Wd.win[1];
  const int off = n1 / 2 - n0 / 2;
  if constexpr (TRIM && !FRESH)
    if (T.base[nstreams] * ch > T.cap) return;
  for (int task = blockIdx.x; task < nstreams * ch; task += gridDim.x) {
    const int st = task / ch, c = task - st * ch;
    int lW = 0;
    int cnt = nblk, first_out = 1;
    if constexpr (CARRY || TRIM) {
      if (count) cnt = min(max(count[st], 0), nblk);
      if (cnt == 0) continue;
      int cw;
      if constexpr (FRESH) cw = -1;
      else if constexpr (TRIM) cw = T.W_in[st];
      else cw = carry_W[task];
      if (cw >= 0) {
        // the loads finish before block 0's first __syncthreads; s_prev is read only after it
        lW = cw ? 1 : 0;
        first_out = 0;
        const float *t;
        if constexpr (TRIM) t = T.tail(st, c);
        else t = carry_tail + (size_t)task * tail_stride;
        for (int i = tid; i < ((lW ? X1.N : X0.N) >> 1); i += nt) s_prev[i] = t[i];
      }
    }
    for (int k = 0; k < cnt; k++) {
      const int W = Wseq[(size_t)st * nblk + k];
      const XformDev &X = W ? X1 : X0;
      const int N = X.N, n2 = N >> 1;
      const size_t cstride = HS ? (size_t)N : (size_t)n2;
      const float4 *src = reinterpret_cast<const float4 *>(coef + coef_off[(size_t)st * nblk + k] + c * cstride);
      for (int i = tid; i < (n2 >> 2); i += nt) reinterpret_cast<float4 *>(s_in)[i] = __ldg(src + i);
      __syncthreads();
      dev_mdct_backward<0>(X, s_in, s_out, tid, nt);
      if (k >= first_out) {
        const long long o = pcm_off[(size_t)st * nblk + k];
        using Base = typename std::conditional<S16, SinkS16, SinkF32>::type;
        typename std::conditional<TRIM, SinkTrim<Base>, Base>::type dst;
        if constexpr (TRIM) {
          const int2 w = T.win[(size_t)st * nblk + k];
          const long long b = T.base[st];
          dst.lo = w.x; dst.hi = w.y;
          if constexpr (S16) {
            dst.b.p = reinterpret_cast<short *>(pcm_out) + (b + o) * ch + c;
            dst.b.ch = ch;
          } else {
            dst.b.p = reinterpret_cast<float *>(pcm_out) + b * ch + (T.base[st + 1] - b) * c + o;
          }
        } else if constexpr (S16) {
          dst.p = reinterpret_cast<short *>(pcm_out) + ((long long)st * pcm_stride + o) * ch + c;
          dst.ch = ch;
        } else {
          dst.p = reinterpret_cast<float *>(pcm_out) + ((size_t)st * ch + c) * pcm_stride + o;
        }
        const float *R = s_prev, *Lh = s_out;
        if (lW && W) {
          for (int i = tid; i < n1; i += nt) dst.put(i, R[i] * __ldg(w1 + n1 - i - 1) + Lh[i] * __ldg(w1 + i));
        } else if (lW && !W) {
          for (int i = tid; i < off; i += nt) dst.put(i, R[i]);
          for (int i = tid; i < n0; i += nt) dst.put(off + i, R[off + i] * __ldg(w0 + n0 - i - 1) + Lh[i] * __ldg(w0 + i));
        } else if (!lW && W) {
          for (int i = tid; i < n1 / 2 + n0 / 2; i += nt)
            dst.put(i, i < n0 ? R[i] * __ldg(w0 + n0 - i - 1) + Lh[off + i] * __ldg(w0 + i) : Lh[off + i]);
        } else {
          for (int i = tid; i < n0; i += nt) dst.put(i, R[i] * __ldg(w0 + n0 - i - 1) + Lh[i] * __ldg(w0 + i));
        }
      }
      __syncthreads();
      for (int i = tid; i < n2; i += nt) s_prev[i] = s_out[n2 + i];
      lW = W;
      __syncthreads();
    }
    if constexpr ((CARRY || TRIM) && !FRESH) {
      float *t;
      if constexpr (TRIM) t = T.tail(st, c);
      else t = carry_tail + (size_t)task * tail_stride;
      for (int i = tid; i < ((lW ? X1.N : X0.N) >> 1); i += nt) t[i] = s_prev[i];
      if constexpr (TRIM) {
        if (tid == 0 && c == 0) *T.carried(st) = T.head[st];
      } else {
        if (tid == 0) carry_W[task] = lW;
      }
      __syncthreads();                 // the next task's carry-in overwrites s_prev
    }
  }
}

// ---- decode: undo channel coupling, lib/mapping0.c:754-779 (square polar -> L/R), in place
__global__ void __launch_bounds__(256)
k_decouple(int n, int ch, int steps, const int *__restrict__ mag, const int *__restrict__ ang,
           long long total, float *__restrict__ res) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long blk = e / n;
    const int j = (int)(e - blk * n);
    float *base = res + blk * (long long)ch * n + j;
    for (int s = steps - 1; s >= 0; s--) dev_decouple(base + (long long)mag[s] * n, base + (long long)ang[s] * n);
  }
}

// ======================================================================== //
// launch helpers
static int threads_for(int N) {
  int t = N / 8;
  if (t < 64) t = 64;
  if (t > 256) t = 256;
  return t;
}

static int grid_for(vb200_ctx *c, int items, int ctas_per_sm) {
  // grid_div > 1: this launch shares the SMs with the kernels of a concurrent half-batch (encode split)
  int per_sm = ctas_per_sm / c->grid_div;
  if (per_sm < 1) per_sm = 1;
  long g = (long)c->sm_count * per_sm;
  if (g > items) g = items;
  if (g < 1) g = 1;
  return (int)g;
}

template <class K>
static int set_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024)
    CU(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

#define CHECK_CTX(c) do { if (!(c)) return fail(VB200_EINVAL, "null context"); CU(cudaSetDevice((c)->device)); } while (0)
#define CHECK_W(W)   do { if ((W) < 0 || (W) > 1) return fail(VB200_EINVAL, "W must be 0 or 1"); } while (0)

static int post_launch(vb200_ctx *c, int n = 1) {
  c->launches += n;
  CU(cudaGetLastError());
  return 0;
}

// ======================================================================== //
// transforms
extern "C" int vb200_mdct_forward_dev(vb200_ctx *c, int W, int nvec, const float *d_in, float *d_out, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nvec <= 0) return 0;
  const XformDev &X = c->dx[W];
  const size_t smem = sizeof(float) * (3 * (size_t)X.N + (X.N / 2 + X.N / 32 + X.N / 512 + 8));   // 2 x in, work, padded hand-over
  const int nt = threads_for(X.N);
  const int grid = grid_for(c, nvec, 8);
  int rc;
#define LAUNCH_MF(NN)                                                                   \
  do {                                                                                  \
    if ((rc = set_smem(k_mdct_forward<NN>, smem))) return rc;                           \
    k_mdct_forward<NN><<<grid, nt, smem, (cudaStream_t)stream>>>(X, nvec, d_in, d_out); \
  } while (0)
  switch (X.N) {
    case 256: LAUNCH_MF(256); break;
    case 512: LAUNCH_MF(512); break;
    case 1024: LAUNCH_MF(1024); break;
    case 2048: LAUNCH_MF(2048); break;
    default: LAUNCH_MF(0); break;
  }
#undef LAUNCH_MF
  return post_launch(c);
}

extern "C" int vb200_mdct_backward_dev(vb200_ctx *c, int W, int nvec, const float *d_in, float *d_out, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nvec <= 0) return 0;
  const XformDev &X = c->halfrate ? c->dx_hs[W] : c->dx[W];
  const size_t smem = sizeof(float) * (X.N + X.N / 2);
  const int nt = threads_for(X.N), grid = grid_for(c, nvec, 8);
  int rc;
#define LAUNCH_MB(NN)                                                                    \
  do {                                                                                   \
    if ((rc = set_smem(k_mdct_backward<NN>, smem))) return rc;                           \
    k_mdct_backward<NN><<<grid, nt, smem, (cudaStream_t)stream>>>(X, nvec, d_in, d_out); \
  } while (0)
  switch (X.N) {
    case 256: LAUNCH_MB(256); break;
    case 512: LAUNCH_MB(512); break;
    case 1024: LAUNCH_MB(1024); break;
    case 2048: LAUNCH_MB(2048); break;
    default: LAUNCH_MB(0); break;
  }
#undef LAUNCH_MB
  return post_launch(c);
}

// bytes of n elements of T, or n bytes for T = void
template <class T> static size_t elem_bytes(size_t n) {
  if constexpr (std::is_void_v<T>) return n; else return sizeof(T) * n;
}

// "Copy in, run, copy out" for the host-buffer variants.  Every device buffer a host form stages, input or output,
// takes the next buffer of the context's staging pool.  Sizes count elements of T, or bytes for T = void, where the
// C ABI passes void * (the PCM, vb200_encode_io's iwork).  The first failure is kept in rc, and every later call does
// nothing and returns nullptr, so a form stages everything, checks rc once, runs, queues its copies back and returns
// sync().  The copies on s_main read and write the caller's memory, which may be pinned: a form that returns before
// sync(), on any path, waits for them in the destructor, while its lock guard (declared first) still holds the context.
struct HostIO {
  vb200_ctx *c;
  int slot = 0, rc = 0;
  bool queued = false;               // copies queued on s_main since the last sync()
  ~HostIO() { if (queued) cudaStreamSynchronize(c->s_main); }   // the error being returned holds the reason
  // n elements, src copied in unless it is null
  template <class T> T *in(const T *src, size_t n) {
    if (!rc && slot == STAGE_SLOTS) rc = fail(VB200_EFAULT, "host call stages more buffers than the staging pool holds");
    if (rc) return nullptr;
    void *d;
    if ((rc = ensure_buf(c->stage[slot++], elem_bytes<T>(n), &d))) return nullptr;
    if (src && (rc = copy(d, src, elem_bytes<T>(n), cudaMemcpyHostToDevice))) return nullptr;
    return (T *)d;
  }
  template <class T> T *out(size_t n) { return in<T>(nullptr, n); }
  // packet bytes: the buffer is one byte longer, so that it exists when there are none
  uint8_t *packets(const uint8_t *src, int64_t n) {
    uint8_t *d = out<uint8_t>((size_t)n + 1);
    if (rc || (n && (rc = copy(d, src, (size_t)n, cudaMemcpyHostToDevice)))) return nullptr;
    return d;
  }
  template <class T> void back(T *dst, const T *d, size_t n) {
    if (!rc) rc = copy(dst, d, elem_bytes<T>(n), cudaMemcpyDeviceToHost);
  }
  int sync() {
    if (!rc) { queued = false; rc = wait(); }
    return rc;
  }

 private:
  int copy(void *dst, const void *src, size_t n, cudaMemcpyKind kind) {
    CU(cudaMemcpyAsync(dst, src, n, kind, c->s_main));
    queued = true;
    return 0;
  }
  int wait() { CU(cudaStreamSynchronize(c->s_main)); return 0; }
};

// "Copy in, run, copy out" chunk by chunk, for the host forms that stream a batch through the device.  The batch of
// `units` (streams of unit_blocks blocks, or blocks) is cut into chunks that rotate over the ENC_SETS buffer sets
// c->set[]: all host->device copies on one stream, all device->host copies on another (one DMA engine per direction
// anyway), the kernels of consecutive chunks alternately on two compute streams (a chunk's kernel tails overlap the
// next chunk's).  Events carry the order H2D(k) -> kernels(k) -> D2H(k) -> H2D(k + ENC_SETS) and nothing else, so the
// copy engines run ahead of / behind the kernels.  Per chunk a form calls in(), run() and back(), and after the last
// chunk returns sync().  Sizes count elements of the device pointer's type; the first failure is kept and the
// destructor waits, as in HostIO.
struct HostPipe {
  vb200_ctx *c;
  int full;                          // units of a full chunk: every set holds this many
  std::vector<int> sched;            // units of each chunk
  int rc = 0;
  bool queued = false;               // copies queued since the last sync()
  // chunk_blocks: blocks per full chunk unless VB200_CHUNK_BLOCKS sets it; one_chunk: the whole batch in one chunk
  HostPipe(vb200_ctx *c, int units, int unit_blocks, int chunk_blocks, bool one_chunk = false) : c(c) {
    { const char *e = getenv("VB200_CHUNK_BLOCKS"); if (e && atoi(e) > 0) chunk_blocks = atoi(e); }
    full = one_chunk ? units : std::clamp(chunk_blocks / unit_blocks, 1, units);
    // The pipeline's fill (first H2D + first kernels before anything overlaps) and drain (last kernels + last D2H)
    // are exposed, so from 6 full chunks up the first and the last two are small (full/4, full/2), the rest full size.
    const int q = std::max(full / 4, 1), hlf = std::max(full / 2, 1);
    const bool ramp = units >= 6 * full;
    if (ramp) sched = {q, hlf};
    for (int left = units - (ramp ? 2 * (q + hlf) : 0); left > 0; left -= sched.back())
      sched.push_back(std::min(left, full));
    if (ramp) sched.insert(sched.end(), {hlf, q});
  }
  ~HostPipe() {
    if (queued) for (cudaStream_t st : {c->s_enc[0], c->s_enc[1], c->s_enc[2], c->s_d2h}) cudaStreamSynchronize(st);
  }
  template <class T> void in(const T *d, const std::remove_cv_t<T> *src, size_t n) {
    if (!rc) rc = copy((void *)d, src, elem_bytes<T>(n), cudaMemcpyHostToDevice, c->s_enc[2]);
  }
  template <class T> void back(std::remove_cv_t<T> *dst, const T *d, size_t n) {
    if (!rc) rc = copy(dst, d, elem_bytes<T>(n), cudaMemcpyDeviceToHost, c->s_d2h);
  }
  // chunk k's kernels: launch(st) on its compute stream, after its copies in and before its copies back
  template <class F> int run(int k, F &&launch) { return rc ? rc : (rc = chunk(k, launch)); }
  int sync() {
    if (!rc) { queued = false; rc = wait(); }
    return rc;
  }

 private:
  int copy(void *dst, const void *src, size_t n, cudaMemcpyKind kind, cudaStream_t st) {
    CU(cudaMemcpyAsync(dst, src, n, kind, st));
    queued = true;
    return 0;
  }
  template <class F> int chunk(int k, F &launch) {
    const int L = k % ENC_SETS;
    cudaStream_t st = c->s_enc[k & 1];
    if (k > 0) CU(cudaEventRecord(c->ev_d2h[(k - 1) % ENC_SETS], c->s_d2h));   // chunk k-1's copies back end here
    CU(cudaEventRecord(c->ev_h2d[L], c->s_enc[2]));
    CU(cudaStreamWaitEvent(st, c->ev_h2d[L], 0));
    if (int r = launch(st)) return r;
    CU(cudaEventRecord(c->ev_cmp[L], st));
    CU(cudaStreamWaitEvent(c->s_d2h, c->ev_cmp[L], 0));
    if (k + 1 >= ENC_SETS && k + 1 < (int)sched.size())   // the next chunk's copies in: its set's previous chunk is back
      CU(cudaStreamWaitEvent(c->s_enc[2], c->ev_d2h[(k + 1) % ENC_SETS], 0));
    return 0;
  }
  int wait() {
    for (cudaStream_t st : {c->s_enc[0], c->s_enc[1], c->s_enc[2], c->s_d2h}) CU(cudaStreamSynchronize(st));
    return 0;
  }
};

extern "C" int vb200_mdct_forward(vb200_ctx *c, int W, int nvec, const float *in, float *out) {
  CHECK_CTX(c); CHECK_W(W);
  if (nvec <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const int N = c->dx[W].N;
  HostIO io{c};
  const float *di = io.in(in, (size_t)nvec * N);
  float *dout = io.out<float>((size_t)nvec * N / 2);
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_mdct_forward_dev(c, W, nvec, di, dout, c->s_main))) return rc;
  io.back(out, dout, (size_t)nvec * N / 2);
  return io.sync();
}

extern "C" int vb200_mdct_backward(vb200_ctx *c, int W, int nvec, const float *in, float *out) {
  CHECK_CTX(c); CHECK_W(W);
  if (nvec <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const int N = (c->halfrate ? c->dx_hs[W] : c->dx[W]).N;
  HostIO io{c};
  const float *di = io.in(in, (size_t)nvec * N / 2);
  float *dout = io.out<float>((size_t)nvec * N);
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_mdct_backward_dev(c, W, nvec, di, dout, c->s_main))) return rc;
  io.back(out, dout, (size_t)nvec * N);
  return io.sync();
}

extern "C" int vb200_apply_window(vb200_ctx *c, int W, int nvec, const int32_t *lW, const int32_t *nW, float *data) {
  CHECK_CTX(c); CHECK_W(W);
  if (nvec <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const int N = c->dx[W].N;
  HostIO io{c};
  float *dd = io.in(data, (size_t)nvec * N);
  const int32_t *dl = lW ? io.in(lW, nvec) : nullptr, *dn = nW ? io.in(nW, nvec) : nullptr;
  if (io.rc) return io.rc;
  k_apply_window<<<grid_for(c, nvec, 8), 256, 0, c->s_main>>>(c->dwin, W, nvec, dl, dn, dd);
  int rc;
  if ((rc = post_launch(c))) return rc;
  io.back(data, dd, (size_t)nvec * N);
  return io.sync();
}

extern "C" int vb200_drft_forward(vb200_ctx *c, int W, int nvec, float *data) {
  CHECK_CTX(c); CHECK_W(W);
  if (nvec <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const XformDev &X = c->dx[W];
  HostIO io{c};
  float *dd = io.in(data, (size_t)nvec * X.N);
  if (io.rc) return io.rc;
  const size_t smem = sizeof(float) * 2 * fft_buf_floats(X.N);
  int rc;
  if ((rc = set_smem(k_drft_forward, smem))) return rc;
  k_drft_forward<<<grid_for(c, nvec, 8), threads_for(X.N), smem, c->s_main>>>(X, nvec, dd);
  if ((rc = post_launch(c))) return rc;
  io.back(data, dd, (size_t)nvec * X.N);
  return io.sync();
}

// ======================================================================== //
// stage-isolated psy entry points
static size_t psy_smem_bytes(const PsyDev &a, const PsyDev &b) {
  const int total = a.total > b.total ? a.total : b.total;
  const int nruns = a.nruns > b.nruns ? a.nruns : b.nruns;
  return sizeof(float) * psy_smem_floats(a.n, total, nruns);
}

#define CHECK_LOOK(c, look) do { if ((look) < 0 || (look) >= (c)->n_psy) return fail(VB200_EINVAL, "no such psy look"); } while (0)

extern "C" int vb200_noisemask(vb200_ctx *c, int look, int nvec, const float *logmdct, float *noise) {
  CHECK_CTX(c); CHECK_LOOK(c, look);
  if (nvec <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const PsyDev &P = c->dpsy[look];
  HostIO io{c};
  const size_t len = (size_t)nvec * P.n;
  const float *di = io.in(logmdct, len);
  float *dout = io.out<float>(len);
  if (io.rc) return io.rc;
  const size_t smem = psy_smem_bytes(P, P);
  int rc;
  if ((rc = set_smem(k_noisemask, smem))) return rc;
  k_noisemask<<<grid_for(c, nvec, 4), PSY_THREADS, smem, c->s_main>>>(P, nvec, di, dout);
  if ((rc = post_launch(c))) return rc;
  io.back(noise, dout, len);
  return io.sync();
}

extern "C" int vb200_tonemask(vb200_ctx *c, int look, int nvec, const float *logfft,
                              const float *gmax, const float *lmax, float *tone) {
  CHECK_CTX(c); CHECK_LOOK(c, look);
  if (nvec <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const PsyDev &P = c->dpsy[look];
  HostIO io{c};
  const size_t len = (size_t)nvec * P.n;
  const float *di = io.in(logfft, len), *dg = io.in(gmax, nvec), *dl = io.in(lmax, nvec);
  float *dout = io.out<float>(len);
  if (io.rc) return io.rc;
  const size_t smem = psy_smem_bytes(P, P);
  int rc;
  if ((rc = set_smem(k_tonemask, smem))) return rc;
  k_tonemask<<<grid_for(c, nvec, 4), PSY_THREADS, smem, c->s_main>>>(P, nvec, di, dg, dl, dout);
  if ((rc = post_launch(c))) return rc;
  io.back(tone, dout, len);
  return io.sync();
}

extern "C" int vb200_offset_and_mix(vb200_ctx *c, int look, int nvec, int sel, const float *noise,
                                    const float *tone, float *mdct, const float *logmdct, float *logmask) {
  CHECK_CTX(c); CHECK_LOOK(c, look);
  if (sel < 0 || sel > 2) return fail(VB200_EINVAL, "offset_select");
  if (nvec <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const PsyDev &P = c->dpsy[look];
  HostIO io{c};
  const size_t len = (size_t)nvec * P.n;
  const float *dn = io.in(noise, len), *dt = io.in(tone, len);
  float *dm = io.in(mdct, len);
  const float *dl = io.in(logmdct, len);
  float *dk = io.out<float>(len);
  if (io.rc) return io.rc;
  k_offset_and_mix<<<grid_for(c, (int)((len + 255) / 256), 8), 256, 0, c->s_main>>>(P, nvec, sel, dn, dt, dm, dl, dk);
  int rc;
  if ((rc = post_launch(c))) return rc;
  io.back(logmask, dk, len);
  io.back(mdct, dm, len);
  return io.sync();
}

// ======================================================================== //
// Phase A
// stage 1: window + MDCT + FFT + log spectrum of `nblocks` blocks of size W
static int phaseA_transform_launch(vb200_ctx *c, int W, int nblocks, const vb200_phaseA_io *io, const PcmSrc &psrc,
                                   cudaStream_t st, float *d_logfft, float *d_lmax) {
  const XformDev &X = c->dx[W];
  const int ch = c->setup.channels, N = X.N;
  const int rows = nblocks * ch;
  {
    const size_t smem = sizeof(float) * (2 * N + 2 * fft_buf_floats(N));   // sx, sw, sf + the cp.async staging row
    int rc;
    float *mdct_raw = io->tap_mdct_raw ? io->tap_mdct_raw : io->mdct;
    const int grid = grid_for(c, rows, 8), nt = threads_for(N);
#define LAUNCH_XF(NN)                                                                        \
    do {                                                                                     \
      if ((rc = set_smem(k_phaseA_transform<NN>, smem))) return rc;                          \
      k_phaseA_transform<NN><<<grid, nt, smem, st>>>(X, c->dwin, W, ch, rows, psrc, io->desc,    \
                                                     mdct_raw, d_logfft, d_lmax);            \
    } while (0)
    switch (N) {
      case 256: LAUNCH_XF(256); break;
      case 512: LAUNCH_XF(512); break;
      case 1024: LAUNCH_XF(1024); break;
      case 2048: LAUNCH_XF(2048); break;
      default: LAUNCH_XF(0); break;
    }
#undef LAUNCH_XF
    rc = post_launch(c); if (rc) return rc;
  }
  return 0;
}

constexpr int PSY_CTAS_PER_SM = 5;   // the generic psy kernel's grid, and the CTAs its carve-out leaves room for

// stage 3: noise / tone masks + mix of `nblocks` blocks of size W, given every block's global ampmax
static int phaseA_psy_launch(vb200_ctx *c, int W, int nblocks, const vb200_phaseA_io *io, cudaStream_t st,
                             float *d_logfft, float *d_lmax, float *d_gmax) {
  const int ch = c->setup.channels, n = c->dx[W].N / 2;
  const int rows = nblocks * ch;
  const PsyDev &P0 = c->dpsy[2 * W], &P1 = c->dpsy[2 * W + 1];
  const int total = P0.total > P1.total ? P0.total : P1.total;
  const int nruns = P0.nruns > P1.nruns ? P0.nruns : P1.nruns;
  const int ngrp = P0.ngrp > P1.ngrp ? P0.ngrp : P1.ngrp;
  const size_t smem = psy_smem_bytes(P0, P1);
  int rc = set_smem(k_phaseA_psy, smem); if (rc) return rc;
  if (!c->psy_carveout_set) {
    // leave the rest of the 256 KB unified array to L1: the static psy tables (~60 KB per look)
    // are read through it on every row
    int pct = (int)((PSY_CTAS_PER_SM * (smem + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024));
    if (pct > 100) pct = 100;
    CU(cudaFuncSetAttribute(k_phaseA_psy, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
    c->psy_carveout_set = true;
  }
  PsyArgs A;
  A.mdct_in = io->tap_mdct_raw ? io->tap_mdct_raw : io->mdct;
  A.logfft = d_logfft; A.lmax = d_lmax; A.gmax = d_gmax; A.desc = io->desc;
  A.mdct_out = io->mdct; A.logmdct = io->logmdct; A.logmask = io->logmask; A.ampmax_out = io->ampmax_out;
  A.tap_noise = io->tap_noise; A.tap_tone = io->tap_tone;
  A.dbg_cycles = nullptr;
  if (getenv("VB200_PHASE_TIMING")) {
    void *p; if ((rc = ensure_buf(c->cycles, 16 * sizeof(unsigned long long), &p))) return rc;
    A.dbg_cycles = (unsigned long long *)p;
  }
  // VB200_PSY_V1=1 forces the generic kernel, so that the tests can check it on the setups the fast one takes
  const char *ev1 = getenv("VB200_PSY_V1");
  if (!(ev1 && atoi(ev1)) && P0.linesper == P1.linesper && psy3_supported(n, total, P0.linesper)) {
    constexpr int R = 2;                             // rows per CTA sharing one scan warp (DESIGN.md §4)
    const size_t row_bytes = sizeof(float) * ((psy3_floats(n, total, nruns, ngrp) + 3) & ~(size_t)3);
    const size_t smem3 = row_bytes * R;
    int ctas = (int)((227 * 1024) / (smem3 + 1024));
    if (ctas > PSY3_MINB / R) ctas = PSY3_MINB / R;
    if (ctas < 1) ctas = 1;
    const bool dbg3 = A.dbg_cycles || A.tap_noise || A.tap_tone;   // clock marks / taps: the debug instance
#define LAUNCH_PSY3D(KK, DD)                                                                       \
    do {                                                                                           \
      if ((rc = set_smem(k_phaseA_psy3<KK, R, DD>, smem3))) return rc;                             \
      k_phaseA_psy3<KK, R, DD><<<grid_for(c, (rows + R - 1) / R, ctas), PSY3_THREADS * R, smem3, st>>>(P0, P1, ch, rows, A); \
    } while (0)
#define LAUNCH_PSY3(KK) do { if (dbg3) LAUNCH_PSY3D(KK, true); else LAUNCH_PSY3D(KK, false); } while (0)
    switch (n / 128) {
      case 1: LAUNCH_PSY3(1); break;
      case 2: LAUNCH_PSY3(2); break;
      case 4: LAUNCH_PSY3(4); break;
      case 8: LAUNCH_PSY3(8); break;
      default: LAUNCH_PSY3(16); break;
    }
#undef LAUNCH_PSY3D
#undef LAUNCH_PSY3
  } else {
    k_phaseA_psy<<<grid_for(c, rows, PSY_CTAS_PER_SM), PSY_THREADS, smem, st>>>(P0, P1, ch, rows, A);
  }
  return post_launch(c);
}

static int phaseA_launch(vb200_ctx *c, int W, int nblocks, const vb200_phaseA_io *io,
                         int nstreams, int bps, const float *d_amp0, cudaStream_t st,
                         float *d_logfft, float *d_lmax, float *d_gmax, const PcmSrc *pcmsrc = nullptr) {
  PcmSrc psrc;
  if (pcmsrc) psrc = *pcmsrc;
  else { psrc.base = io->pcm; psrc.fmt = 0; psrc.bps = 1; psrc.hop = 0; psrc.stride = 0; psrc.blk_src = nullptr; }
  const XformDev &X = c->dx[W];
  const int ch = c->setup.channels, N = X.N;
  int rc;
  if (c->profiling) CU(cudaEventRecord(c->ev[0], st));
  if ((rc = phaseA_transform_launch(c, W, nblocks, io, psrc, st, d_logfft, d_lmax))) return rc;
  if (c->profiling) CU(cudaEventRecord(c->ev[1], st));
  {
    const int n = N / 2;
    const float secs = (float)n / (float)c->setup.rate;           // lib/psy.c:843
    const float secs_att = secs * c->setup.ampmax_att_per_sec;
    if (nstreams > 0)
      k_ampmax<<<(nstreams + 127) / 128, 128, 0, st>>>(1, nstreams, bps, ch, io->desc, d_lmax, d_amp0, secs_att, d_gmax);
    else
      k_ampmax<<<(nblocks + 127) / 128, 128, 0, st>>>(0, nblocks, 0, ch, io->desc, d_lmax, nullptr, secs_att, d_gmax);
    int rc = post_launch(c); if (rc) return rc;
  }
  if (c->profiling) CU(cudaEventRecord(c->ev[2], st));
  if ((rc = phaseA_psy_launch(c, W, nblocks, io, st, d_logfft, d_lmax, d_gmax))) return rc;
  if (c->profiling) CU(cudaEventRecord(c->ev[3], st));
  return 0;
}

static int phaseA_dev_common(vb200_ctx *c, int W, int nblocks, const vb200_phaseA_io *io,
                             int nstreams, int bps, const float *d_amp0, void *stream,
                             const PcmSrc *pcmsrc = nullptr) {
  CHECK_CTX(c); CHECK_W(W);
  if (c->n_psy != 4) return fail(VB200_EIMPL, "context has no psy lookups");
  if (!io || (!io->pcm && !pcmsrc) || !io->desc || !io->mdct || !io->logmdct || !io->logmask || !io->ampmax_out)
    return fail(VB200_EINVAL, "phase A io pointers");
  if (nblocks <= 0) return 0;
  const size_t rows = (size_t)nblocks * c->setup.channels, n = c->dx[W].N / 2;
  float *d_logfft, *d_lmax, *d_gmax; int rc;
  if ((rc = carve(c->phaseA, [&](Carve &k) {
         d_logfft = io->tap_logfft ? io->tap_logfft : k.take<float>(rows * n);
         d_lmax = k.take<float>(rows);
         d_gmax = k.take<float>(nblocks);
       }))) return rc;
  if ((rc = scratch_begin(c, (cudaStream_t)stream))) return rc;
  if ((rc = phaseA_launch(c, W, nblocks, io, nstreams, bps, d_amp0, (cudaStream_t)stream, d_logfft, d_lmax, d_gmax,
                          pcmsrc))) return rc;
  return scratch_end(c, (cudaStream_t)stream);
}

extern "C" int vb200_analysis_phaseA_pcmstream_dev(vb200_ctx *c, int W, int nstreams, int bps,
                                                   const void *d_pcm, int fmt, int64_t stream_stride, int hop,
                                                   const vb200_phaseA_io *io, const float *d_amp0, void *stream) {
  if (nstreams <= 0 || bps <= 0) return fail(VB200_EINVAL, "nstreams/blocks_per_stream");
  if (!d_pcm) return fail(VB200_EINVAL, "null pcm");
  if (fmt != VB200_PCM_F32_PLANAR && fmt != VB200_PCM_S16_INTERLEAVED) return fail(VB200_EINVAL, "pcm format");
  if (hop <= 0 || stream_stride <= 0) return fail(VB200_EINVAL, "hop/stream_stride");
  if (fmt == VB200_PCM_F32_PLANAR && ((hop & 3) || (stream_stride & 3)))
    return fail(VB200_EINVAL, "hop and stream_stride must be multiples of 4 for float PCM");
  if (!c || W < 0 || W > 1) return fail(VB200_EINVAL, "ctx/W");
  if ((int64_t)(bps - 1) * hop + c->dx[W].N > stream_stride) return fail(VB200_EINVAL, "blocks exceed the stream buffer");
  PcmSrc ps; ps.base = d_pcm; ps.fmt = fmt; ps.bps = bps; ps.hop = hop; ps.stride = stream_stride; ps.blk_src = nullptr;
  return phaseA_dev_common(c, W, nstreams * bps, io, nstreams, bps, d_amp0, stream, &ps);
}

extern "C" int vb200_analysis_phaseA_dev(vb200_ctx *c, int W, int nblocks, const vb200_phaseA_io *io, void *stream) {
  return phaseA_dev_common(c, W, nblocks, io, 0, 0, nullptr, stream);
}

extern "C" int vb200_analysis_phaseA_streams_dev(vb200_ctx *c, int W, int nstreams, int bps,
                                                 const vb200_phaseA_io *io, const float *d_amp0, void *stream) {
  if (nstreams <= 0 || bps <= 0) return fail(VB200_EINVAL, "nstreams/blocks_per_stream");
  return phaseA_dev_common(c, W, nstreams * bps, io, nstreams, bps, d_amp0, stream);
}

// Host-buffer Phase A: the blocks go through HostPipe in chunks of 4096; they are independent (desc[].ampmax is each
// block's ampmax on entry), so any chunking gives the same outputs.  Pinned host memory is needed for the copies to be
// truly asynchronous (pageable memory still works, staged by the driver).  With profiling on, the whole batch is one
// chunk, so that vb200_phaseA_kernel_ms brackets the whole call.
extern "C" int vb200_analysis_phaseA(vb200_ctx *c, int W, int nblocks, const vb200_phaseA_io *h) {
  CHECK_CTX(c); CHECK_W(W);
  if (!h) return fail(VB200_EINVAL, "null io");
  if (c->n_psy != 4) return fail(VB200_EIMPL, "context has no psy lookups");
  if (!h->pcm || !h->desc || !h->mdct || !h->logmdct || !h->logmask || !h->ampmax_out)
    return fail(VB200_EINVAL, "phase A io pointers");
  if (nblocks <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels, N = c->dx[W].N, n = N / 2;
  HostPipe pipe(c, nblocks, 1, 4096, c->profiling);
  const size_t cb = pipe.full, crow = cb * ch;
  int rc;
  vb200_phaseA_io dset[ENC_SETS];
  float *logfft[ENC_SETS], *lmax[ENC_SETS], *gmax[ENC_SETS];
  for (int b0 = 0, it = 0; it < (int)pipe.sched.size(); b0 += pipe.sched[it], it++) {
    const int L = it % ENC_SETS, nb = pipe.sched[it];
    const size_t rows = (size_t)nb * ch, r0 = (size_t)b0 * ch;
    vb200_phaseA_io &d = dset[L];
    if (it < ENC_SETS) {                             // the set's first chunk: every chunk fits cb blocks
      memset(&d, 0, sizeof(d));
      if ((rc = carve(c->set[L], [&](Carve &k) {
             d.pcm = k.take<float>(crow * N); d.desc = k.take<vb200_block_desc>(cb);
             d.mdct = k.take<float>(crow * n); d.logmdct = k.take<float>(crow * n); d.logmask = k.take<float>(crow * n);
             d.ampmax_out = k.take<float>(cb);
             logfft[L] = k.take<float>(crow * n); lmax[L] = k.take<float>(crow); gmax[L] = k.take<float>(cb);
             d.tap_noise = h->tap_noise ? k.take<float>(crow * n) : nullptr;
             d.tap_tone = h->tap_tone ? k.take<float>(crow * n) : nullptr;
             d.tap_mdct_raw = h->tap_mdct_raw ? k.take<float>(crow * n) : nullptr;
           }))) return rc;
    }
    pipe.in(d.pcm, h->pcm + r0 * N, rows * N);
    pipe.in(d.desc, h->desc + b0, nb);
    if ((rc = pipe.run(it, [&](cudaStream_t st) {
           return phaseA_launch(c, W, nb, &d, 0, 0, nullptr, st, logfft[L], lmax[L], gmax[L]);
         }))) return rc;
    // the spectra and the taps asked for; the set's logfft is the logfft tap
    const std::pair<float *, const float *> spectra[] = {
        {h->mdct, d.mdct}, {h->logmdct, d.logmdct}, {h->logmask, d.logmask}, {h->tap_noise, d.tap_noise},
        {h->tap_tone, d.tap_tone}, {h->tap_logfft, logfft[L]}, {h->tap_mdct_raw, d.tap_mdct_raw}};
    for (const auto &s : spectra)
      if (s.first) pipe.back(s.first + r0 * n, s.second, rows * n);
    pipe.back(h->ampmax_out + b0, d.ampmax_out, nb);
  }
  return pipe.sync();
}

// ======================================================================== //
// Phase B
static int cqn_setup(vb200_ctx *c, int W, int blocktype, int blobno, CqnDev *Q) {
  if (c->n_psy != 4) return fail(VB200_EIMPL, "context has no psy lookups");
  if (blocktype < 0 || blocktype > 1) return fail(VB200_EINVAL, "blocktype");
  if (blobno < 0 || blobno >= VB200_PACKETBLOBS) return fail(VB200_EINVAL, "blobno");
  const vb200_psy_setup &p = c->setup.psy[blocktype + 2 * W];
  static const double thr[] = {0.0, .5, 1.0, 1.5, 2.5, 4.5, 8.5, 16.5, 9e10};       // lib/psy.c:32
  static const double thr_limited[] = {0.0, .5, 1.0, 1.5, 2.0, 2.5, 4.5, 8.5, 9e10}; // lib/psy.c:33
  const int pre = c->setup.coupling_prepointamp[blobno], post = c->setup.coupling_postpointamp[blobno];
  if (pre < 0 || pre > 8 || post < 0 || post > 8) return fail(VB200_EINVAL, "pointamp index");
  Q->n = p.n; Q->ch = c->setup.channels;
  Q->partition = p.normal_p ? p.normal_partition : 16;
  if (Q->partition != 8 && Q->partition != 16 && Q->partition != 32)
    return fail(VB200_EIMPL, "normal_partition must be 8, 16 or 32");
  Q->limit = c->setup.coupling_pointlimit[p.blockflag][blobno];
  Q->sliding_lowpass = c->setup.sliding_lowpass[W][blobno];
  Q->steps = c->setup.coupling_steps[W];
  Q->normal_p = p.normal_p; Q->normal_start = p.normal_start; Q->normal_thresh = p.normal_thresh;
  Q->prepoint = (float)thr[pre];
  Q->postpoint = (float)(p.n > 1000 ? thr_limited[post] : thr[post]);
  Q->mag = c->d_mag[W]; Q->ang = c->d_ang[W]; Q->fromdB = c->d_fromdB;
  return 0;
}

// k_cqn keeps CQN_COLS x 32 lines of every channel per warp in shared memory, so it takes at most 79 channels.  The
// encode chains check this before their first launch, so that a refused call leaves its device outputs untouched.
constexpr int CQN_WPB = 4;
static size_t cqn_smem(int ch) { return (size_t)CQN_WPB * (CQN_COLS * ch * 32 * sizeof(float) + ch * sizeof(int)); }
static int cqn_channels_check(const vb200_ctx *c) {
  if (cqn_smem(c->setup.channels) > 200 * 1024) return fail(VB200_EIMPL, "too many channels for the coupling kernel");
  return 0;
}

// one launcher for both entry points: desc == NULL -> every block uses Q0
static int cqn_launch(vb200_ctx *c, const CqnDev &Q0, const CqnDev &Q1, const vb200_block_desc *d_desc, int nblocks,
                      const float *d_mdct, int32_t *d_iwork, int32_t *d_nonzero, cudaStream_t st) {
  int rc;
  const int wpb = CQN_WPB;
  const long tasks = (long)nblocks * (Q0.n / 32);
  if (tasks < (1L << 30) && (Q0.n & (Q0.n - 1)) == 0 && (Q0.ch == 1 || (Q0.ch == 2 && Q0.steps <= 1))) {
    const int grid = grid_for(c, (int)((tasks + wpb - 1) / wpb), 16);
    if (Q0.ch == 1) k_cqn_fast<1><<<grid, wpb * 32, 0, st>>>(Q0, Q1, d_desc, nblocks, d_mdct, d_iwork, d_nonzero);
    else k_cqn_fast<2><<<grid, wpb * 32, 0, st>>>(Q0, Q1, d_desc, nblocks, d_mdct, d_iwork, d_nonzero);
  } else {
    const size_t smem = cqn_smem(Q0.ch);
    if ((rc = cqn_channels_check(c))) return rc;
    if ((rc = set_smem(k_cqn, smem))) return rc;
    k_cqn<<<grid_for(c, (int)((tasks + wpb - 1) / wpb), 8), wpb * 32, smem, st>>>(Q0, Q1, d_desc, nblocks, d_mdct,
                                                                              d_iwork, d_nonzero);
  }
  if ((rc = post_launch(c))) return rc;
  if (Q0.steps > 0) {
    k_cqn_nonzero<<<(nblocks + 127) / 128, 128, 0, st>>>(nblocks, Q0.ch, Q0.steps, Q0.mag, Q0.ang, d_nonzero, 0);
    if ((rc = post_launch(c))) return rc;
  }
  return 0;
}

// bitrate-managed mode: couple/quantise/normalise of all VB200_PACKETBLOBS curves, curve k with blob k's
// parameters; curve k's iwork / nonzero rows start k * blob_blocks blocks in.  Mono and stereo with at most one
// coupling step take every curve in one k_cqn_fast_curves launch; other setups run k_cqn once per curve.
static int cqn_curves_launch(vb200_ctx *c, int W, const vb200_block_desc *d_desc, int nblocks, long long blob_blocks,
                             const float *d_mdct, int32_t *d_iwork, int32_t *d_nonzero, cudaStream_t st) {
  constexpr int NB = VB200_PACKETBLOBS;
  const int ch = c->setup.channels, n = c->dx[W].N / 2;
  CqnDev Q[2];                       // the kernel takes only the fields that do not depend on the blob from these
  CqnCurveTab T;
  int rc;
  for (int k = 0; k < NB; k++)
    for (int bt = 0; bt < 2; bt++) {
      if ((rc = cqn_setup(c, W, bt, k, &Q[bt]))) return rc;
      T.c[bt][k] = {Q[bt].limit, Q[bt].sliding_lowpass, Q[bt].prepoint, Q[bt].postpoint};
    }
  const long tasks = (long)nblocks * (n / 32);
  if (!(tasks < (1L << 30) && (n & (n - 1)) == 0 && (ch == 1 || (ch == 2 && Q[0].steps <= 1)))) {
    for (int k = 0; k < NB; k++) {
      CqnDev Q0, Q1;
      if ((rc = cqn_setup(c, W, 0, k, &Q0))) return rc;
      if ((rc = cqn_setup(c, W, 1, k, &Q1))) return rc;
      const size_t r0 = (size_t)k * blob_blocks * ch;
      if ((rc = cqn_launch(c, Q0, Q1, d_desc, nblocks, d_mdct, d_iwork + r0 * n, d_nonzero + r0, st))) return rc;
    }
    return 0;
  }
  const int wpb = 4, grid = grid_for(c, (int)((tasks + wpb - 1) / wpb), 16);
  if (ch == 1) k_cqn_fast_curves<1><<<grid, wpb * 32, 0, st>>>(Q[0], Q[1], T, d_desc, nblocks, blob_blocks, d_mdct, d_iwork, d_nonzero);
  else k_cqn_fast_curves<2><<<grid, wpb * 32, 0, st>>>(Q[0], Q[1], T, d_desc, nblocks, blob_blocks, d_mdct, d_iwork, d_nonzero);
  if ((rc = post_launch(c))) return rc;
  if (Q[0].steps > 0) {
    k_cqn_nonzero<<<dim3((nblocks + 127) / 128, NB), 128, 0, st>>>(nblocks, ch, Q[0].steps, Q[0].mag, Q[0].ang, d_nonzero,
                                                                   blob_blocks);
    if ((rc = post_launch(c))) return rc;
  }
  return 0;
}

extern "C" int vb200_couple_quantize_normalize_dev(vb200_ctx *c, int W, int blocktype, int blobno, int nblocks,
                                                   const float *d_mdct, int32_t *d_iwork, int32_t *d_nonzero,
                                                   void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nblocks <= 0) return 0;
  CqnDev Q; int rc;
  if ((rc = cqn_setup(c, W, blocktype, blobno, &Q))) return rc;
  return cqn_launch(c, Q, Q, nullptr, nblocks, d_mdct, d_iwork, d_nonzero, (cudaStream_t)stream);
}

extern "C" int vb200_couple_quantize_normalize(vb200_ctx *c, int W, int blocktype, int blobno, int nblocks,
                                               const float *mdct, int32_t *iwork, int32_t *nonzero) {
  CHECK_CTX(c); CHECK_W(W);
  if (nblocks <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels, n = c->dx[W].N / 2;
  const size_t rows = (size_t)nblocks * ch;
  HostIO io{c};
  const float *dm = io.in(mdct, rows * n);
  int32_t *di = io.in(iwork, rows * n), *dz = io.in(nonzero, rows);
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_couple_quantize_normalize_dev(c, W, blocktype, blobno, nblocks, dm, di, dz, c->s_main))) return rc;
  io.back(iwork, di, rows * n);
  io.back(nonzero, dz, rows);
  return io.sync();
}

// ======================================================================== //
// decode
// vorbis_synthesis_halfrate, lib/synthesis.c:166-174
extern "C" int vb200_synthesis_halfrate(vb200_ctx *c, int flag, const float *const window[2]) {
  CHECK_CTX(c);
  if (!flag) { c->halfrate = false; return 0; }
  if (c->setup.blocksizes[0] <= 64) return fail(VB200_EINVAL, "half-rate decode needs blocksizes[0] > 64 (lib/synthesis.c:170)");
  if (!c->hs_built) {
    std::lock_guard<std::mutex> lk(c->mu);
    for (int w = 0; w < 2; w++) {
      int rc;
      if ((rc = xform_upload(c, c->setup.blocksizes[w] / 2, window ? window[w] : nullptr, c->hx_hs[w], c->dx_hs[w])))
        return rc;
      c->dwin_hs.N[w] = c->hx_hs[w].N;
      c->dwin_hs.win[w] = c->dx_hs[w].win;
    }
    c->hs_built = true;
  }
  c->halfrate = true;
  return 0;
}

// every synthesis launch: smem, threads and grid from the context's transforms (half-rate or full), then the
// S16 x half-rate instance of MODE.  k: the carry of CARRY; T: the tables of TRIM and RANGE.
template <SynthMode MODE>
static int synthesis_launch(vb200_ctx *c, bool s16, int nstreams, int nblk, const int32_t *d_count,
                            const int32_t *d_Wseq, const int64_t *d_coef_off, const float *d_coef,
                            const int64_t *d_pcm_off, void *d_pcm, int64_t pcm_stride, const vb200_decode_carry *k,
                            const DsTrim &T, cudaStream_t st) {
  const bool hs = c->halfrate;
  const XformDev *X = hs ? c->dx_hs : c->dx;
  const int ch = c->setup.channels, N1 = X[1].N;
  const size_t smem = sizeof(float) * ((size_t)N1 / 2 + N1 + N1 / 2);
  auto *kern = s16 ? (hs ? k_synthesis<true, true, MODE> : k_synthesis<true, false, MODE>)
                   : (hs ? k_synthesis<false, true, MODE> : k_synthesis<false, false, MODE>);
  int rc = set_smem(kern, smem); if (rc) return rc;
  kern<<<grid_for(c, nstreams * ch, 8), threads_for(N1), smem, st>>>(
      X[0], X[1], hs ? c->dwin_hs : c->dwin, ch, nstreams, nblk, d_Wseq, (const long long *)d_coef_off, d_coef,
      (const long long *)d_pcm_off, d_pcm, (long long)pcm_stride, d_count, k ? k->tail : nullptr,
      k ? k->W : nullptr, c->setup.blocksizes[1] / 2, T);
  return post_launch(c);
}

extern "C" int vb200_synthesis_dev(vb200_ctx *c, int nstreams, int nblk, const int32_t *d_Wseq,
                                   const int64_t *d_coef_off, const float *d_coef,
                                   const int64_t *d_pcm_off, float *d_pcm, int64_t pcm_stride, void *stream) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  return synthesis_launch<SYN_PLAIN>(c, false, nstreams, nblk, nullptr, d_Wseq, d_coef_off, d_coef, d_pcm_off, d_pcm,
                                     pcm_stride, nullptr, DsTrim{}, (cudaStream_t)stream);
}

extern "C" int vb200_synthesis_s16_dev(vb200_ctx *c, int nstreams, int nblk, const int32_t *d_Wseq,
                                       const int64_t *d_coef_off, const float *d_coef,
                                       const int64_t *d_pcm_off, int16_t *d_pcm16, int64_t pcm_stride, void *stream) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  return synthesis_launch<SYN_PLAIN>(c, true, nstreams, nblk, nullptr, d_Wseq, d_coef_off, d_coef, d_pcm_off, d_pcm16,
                                     pcm_stride, nullptr, DsTrim{}, (cudaStream_t)stream);
}

extern "C" int vb200_synthesis(vb200_ctx *c, int nstreams, int nblk, const int32_t *Wseq,
                               const int64_t *coef_off, const float *coef, int64_t coef_len,
                               const int64_t *pcm_off, float *pcm, int64_t pcm_stride) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels;
  const size_t nb = (size_t)nstreams * nblk;
  for (size_t i = 0; i < nb; i++) if (Wseq[i] < 0 || Wseq[i] > 1) return fail(VB200_EINVAL, "Wseq values must be 0/1");
  HostIO io{c};
  const int32_t *dW = io.in(Wseq, nb);
  const int64_t *dco = io.in(coef_off, nb);
  const float *dc = io.in(coef, (size_t)coef_len);
  const int64_t *dpo = io.in(pcm_off, nb);
  const size_t plen = (size_t)nstreams * ch * (size_t)pcm_stride;
  float *dp = io.out<float>(plen);
  if (io.rc) return io.rc;
  CU(cudaMemsetAsync(dp, 0, sizeof(float) * plen, c->s_main));
  int rc;
  if ((rc = vb200_synthesis_dev(c, nstreams, nblk, dW, dco, dc, dpo, dp, pcm_stride, c->s_main))) return rc;
  io.back(pcm, dp, plen);
  return io.sync();
}

extern "C" int vb200_decouple_dev(vb200_ctx *c, int W, int nblocks, float *d_res, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nblocks <= 0 || c->setup.coupling_steps[W] <= 0) return 0;
  const int n = c->dx[W].N / 2;
  const long long total = (long long)nblocks * n;
  k_decouple<<<grid_for(c, (int)((total + 255) / 256), 16), 256, 0, (cudaStream_t)stream>>>(
      n, c->setup.channels, c->setup.coupling_steps[W], c->d_mag[W], c->d_ang[W], total, d_res);
  return post_launch(c);
}

extern "C" int vb200_decouple(vb200_ctx *c, int W, int nblocks, float *res) {
  CHECK_CTX(c); CHECK_W(W);
  if (nblocks <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t len = (size_t)nblocks * c->setup.channels * (c->dx[W].N / 2);
  HostIO io{c};
  float *d = io.in(res, len);
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_decouple_dev(c, W, nblocks, d, c->s_main))) return rc;
  io.back(res, d, len);
  return io.sync();
}

// ======================================================================== //
// floor 1
static int floor1_args(vb200_ctx *c, int W, int floor_sel, int nrows, Floor1Args *a) {
  if (floor_sel >= VB200_MAX_SUBMAPS) return fail(VB200_EINVAL, "floor_sel");
  const int ch = c->setup.channels;
  if (floor_sel >= 0) {
    if (c->setup.floor1[W][floor_sel].posts <= 0) return fail(VB200_EINVAL, "no floor1 setup for this floor_sel");
  } else {
    for (int k = 0; k < ch; k++)
      if (c->setup.floor1[W][c->setup.chmux[W][k]].posts <= 0)
        return fail(VB200_EINVAL, "no floor1 setup for a channel's submap");
  }
  a->floors = c->d_floor[W]; a->chmux = c->d_chmux[W];
  a->channels = ch; a->floor_sel = floor_sel; a->nrows = nrows; a->n = c->dx[W].N / 2;
  return 0;
}

extern "C" int vb200_floor1_fit_dev(vb200_ctx *c, int W, int floor_sel, int nrows, const float *d_logmdct,
                                    const float *d_logmask, int32_t *d_posts, int32_t *d_fit_nonzero, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nrows <= 0) return 0;
  Floor1Args a; int rc;
  if ((rc = floor1_args(c, W, floor_sel, nrows, &a))) return rc;
  // the per-warp area holds floors of the largest post count this block size has, not VB200_VIF_POSIT
  int pcap = 2;
  for (int k = 0; k < VB200_MAX_SUBMAPS; k++) pcap = std::max(pcap, c->setup.floor1[W][k].posts);
  const size_t smem = sizeof(Floor1Dev) * VB200_MAX_SUBMAPS + floor1_fit_smem_per_warp(a.n, pcap) * F1_WARPS;
  const int ctas = (nrows + F1_WARPS - 1) / F1_WARPS;
  const bool dbg = getenv("VB200_FLOOR1_TIMING") != nullptr;   // the instance with clock marks (tools/floor1_phase_timing.py)
  void (*kern)(Floor1Args, int, const float *, const float *, int32_t *, int32_t *, unsigned long long *) =
      dbg ? k_floor1_fit<true> : k_floor1_fit<false>;
  void *p = nullptr;
  if (dbg && (rc = ensure_buf(c->cycles, 16 * sizeof(unsigned long long), &p))) return rc;
  if ((rc = set_smem(kern, smem))) return rc;
  // one wave: as many CTAs per SM as registers and this shared-memory size let be resident
  CU(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  int per_sm = 0;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 32 * F1_WARPS, smem));
  kern<<<grid_for(c, ctas, std::max(per_sm, 1)), 32 * F1_WARPS, smem, (cudaStream_t)stream>>>(
      a, pcap, d_logmdct, d_logmask, d_posts, d_fit_nonzero, (unsigned long long *)p);
  return post_launch(c);
}

// `curves` curves of nrows rows each in one launch; curve k's rows start k * blob_rows rows in
static int floor1_render_launch(vb200_ctx *c, int W, int floor_sel, int nrows, int curves, long long blob_rows,
                                int32_t *d_posts, const int32_t *d_fit_nonzero, int32_t *d_ilogmask,
                                int32_t *d_nonzero, cudaStream_t st) {
  Floor1Args a; int rc;
  if ((rc = floor1_args(c, W, floor_sel, nrows, &a))) return rc;
  const int ctas = (nrows + F1_WARPS - 1) / F1_WARPS;
  k_floor1_render<<<dim3(grid_for(c, ctas, 8), curves), 32 * F1_WARPS, 0, st>>>(a, d_posts, d_fit_nonzero, d_ilogmask,
                                                                             d_nonzero, blob_rows);
  return post_launch(c);
}

extern "C" int vb200_floor1_render_dev(vb200_ctx *c, int W, int floor_sel, int nrows, int32_t *d_posts,
                                       const int32_t *d_fit_nonzero, int32_t *d_ilogmask, int32_t *d_nonzero,
                                       void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nrows <= 0) return 0;
  return floor1_render_launch(c, W, floor_sel, nrows, 1, 0, d_posts, d_fit_nonzero, d_ilogmask, d_nonzero,
                              (cudaStream_t)stream);
}

extern "C" int vb200_floor1_fit(vb200_ctx *c, int W, int floor_sel, int nrows, const float *logmdct,
                                const float *logmask, int32_t *posts, int32_t *fit_nonzero) {
  CHECK_CTX(c); CHECK_W(W);
  if (nrows <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = c->dx[W].N / 2;
  HostIO io{c};
  const float *da = io.in(logmdct, nrows * n), *db = io.in(logmask, nrows * n);
  int32_t *dp = io.out<int32_t>((size_t)nrows * VB200_FLOOR1_STRIDE), *dz = io.out<int32_t>(nrows);
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_floor1_fit_dev(c, W, floor_sel, nrows, da, db, dp, dz, c->s_main))) return rc;
  io.back(posts, dp, (size_t)nrows * VB200_FLOOR1_STRIDE);
  io.back(fit_nonzero, dz, nrows);
  return io.sync();
}

extern "C" int vb200_floor1_render(vb200_ctx *c, int W, int floor_sel, int nrows, int32_t *posts,
                                   const int32_t *fit_nonzero, int32_t *ilogmask, int32_t *nonzero) {
  CHECK_CTX(c); CHECK_W(W);
  if (nrows <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = c->dx[W].N / 2;
  HostIO io{c};
  int32_t *dp = io.in(posts, (size_t)nrows * VB200_FLOOR1_STRIDE);
  const int32_t *dz = io.in(fit_nonzero, nrows);
  int32_t *di = io.out<int32_t>(nrows * n), *dn = io.out<int32_t>(nrows);
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_floor1_render_dev(c, W, floor_sel, nrows, dp, dz, di, dn, c->s_main))) return rc;
  io.back(posts, dp, (size_t)nrows * VB200_FLOOR1_STRIDE);
  io.back(ilogmask, di, nrows * n);
  io.back(nonzero, dn, nrows);
  return io.sync();
}

// ======================================================================== //
// the whole per-block encode DSP (Phase A -> floor1 fit -> floor render -> Phase B)
static_assert(sizeof(vb200_encode_io) == 128, "vb200_encode_io layout (mirrored by vorbis_b200/abi.py)");
struct EncScratch {
  float *mdct, *logmdct, *logmask, *logfft, *lmax, *gmax;
  int32_t *fitnz;
  int32_t *iw32;                     // residue as int32 when the caller wants int16 out
};

// int32 residue -> saturated int16, counting per block what did not fit (VB200_IWORK_S16)
__global__ void __launch_bounds__(256)
k_pack_s16(const int4 *__restrict__ src, short4 *__restrict__ dst, long nvec, int vec_per_block_log2,
           int vec_per_block, int32_t *__restrict__ overflow) {
  for (long v = (long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (long)gridDim.x * blockDim.x) {
    const int4 a = __ldcs(src + v);
    int bad = 0;
    auto sat = [&](int x) { if (x > 32767) { bad++; return (short)32767; } if (x < -32768) { bad++; return (short)-32768; } return (short)x; };
    short4 o;
    o.x = sat(a.x); o.y = sat(a.y); o.z = sat(a.z); o.w = sat(a.w);
    __stcs(dst + v, o);
    // clipping is the rare case: the division for channel counts that are not a power of two only runs there
    if (bad) atomicAdd(overflow + (vec_per_block_log2 >= 0 ? (v >> vec_per_block_log2) : (v / vec_per_block)), bad);
  }
}

static size_t enc_pcm_bytes(const vb200_encode_io *io, int ch, int N, int nstreams, int bps) {
  switch (io->pcm_fmt) {
    case VB200_PCM_F32_BLOCKS: return sizeof(float) * (size_t)nstreams * bps * ch * N;
    case VB200_PCM_F32_PLANAR: return sizeof(float) * (size_t)nstreams * ch * (size_t)io->stream_stride;
    default: return sizeof(int16_t) * (size_t)nstreams * ch * (size_t)io->stream_stride;
  }
}

// host forms of the chain: the inputs copied in, and int32 outputs of `curves` curves staged, in d
static void enc_stage(HostIO &io, const vb200_encode_io *h, vb200_encode_io *d, int ch, int N, int nstreams, int bps,
                      int curves) {
  const size_t nb = (size_t)nstreams * bps, rows = curves * nb * ch;
  d->pcm = io.in(h->pcm, enc_pcm_bytes(h, ch, N, nstreams, bps));
  d->desc = io.in(h->desc, nb);
  const float *a0 = io.in(h->ampmax0, nstreams);     // staged even when there is none
  d->ampmax0 = h->ampmax0 ? a0 : nullptr;
  d->posts = io.out<int32_t>(rows * VB200_FLOOR1_STRIDE);
  d->nonzero = io.out<int32_t>(rows);
  d->iwork = io.out<int32_t>(rows * (N / 2));
  d->ampmax_out = io.out<float>(nb);
}

// own_outputs: the call stages posts / nonzero / iwork itself, so the io need not give them
static int enc_check(vb200_ctx *c, int W, int nstreams, int bps, int blobno, const vb200_encode_io *io,
                     bool own_outputs = false) {
  if (!io || !io->pcm || !io->desc || !io->ampmax_out || (!own_outputs && (!io->posts || !io->nonzero || !io->iwork)))
    return fail(VB200_EINVAL, "encode io pointers");
  if (io->iwork_fmt != VB200_IWORK_S32 && io->iwork_fmt != VB200_IWORK_S16) return fail(VB200_EINVAL, "iwork format");
  if (io->iwork_fmt == VB200_IWORK_S16 && !io->overflow) return fail(VB200_EINVAL, "int16 residue needs the overflow array");
  if (nstreams <= 0 || bps <= 0) return fail(VB200_EINVAL, "nstreams/blocks_per_stream");
  if (c->n_psy != 4) return fail(VB200_EIMPL, "context has no psy lookups");
  if (blobno < 0 || blobno >= VB200_PACKETBLOBS) return fail(VB200_EINVAL, "blobno");
  int rc;
  if ((rc = cqn_channels_check(c))) return rc;
  const int fmt = io->pcm_fmt;
  if (fmt != VB200_PCM_F32_BLOCKS && fmt != VB200_PCM_F32_PLANAR && fmt != VB200_PCM_S16_INTERLEAVED)
    return fail(VB200_EINVAL, "pcm format");
  if (fmt != VB200_PCM_F32_BLOCKS) {
    if (io->hop <= 0 || io->stream_stride <= 0) return fail(VB200_EINVAL, "hop/stream_stride");
    if (fmt == VB200_PCM_F32_PLANAR && ((io->hop & 3) || (io->stream_stride & 3)))
      return fail(VB200_EINVAL, "hop and stream_stride must be multiples of 4 for float PCM");
    if ((int64_t)(bps - 1) * io->hop + c->dx[W].N > io->stream_stride)
      return fail(VB200_EINVAL, "blocks exceed the stream buffer");
  }
  return 0;
}

// ---- bitrate-managed mode (lib/mapping0.c:507-573, 596-646): the chain with three masks, three fits, the twelve
// interpolated curves, and the floor render + couple/quantise/normalise of every one of the 15 curves

// scratch of the managed tail: the psy stage's noise and tone taps, the low- / high-noise mask, the flags of the
// three fits and the present flag of every curve
struct MgdScratch {
  float *noise, *tone, *alt;
  int32_t *fz3, *present;
};

static void mgd_layout(Carve &k, size_t rows, size_t blob_rows, size_t n, MgdScratch *M) {
  M->noise = k.take<float>(rows * n);
  M->tone = k.take<float>(rows * n);
  M->alt = k.take<float>(rows * n);
  M->fz3 = k.take<int32_t>(rows * 3);
  M->present = k.take<int32_t>(blob_rows * VB200_PACKETBLOBS);
}

// Bitrate-managed mode after the psy stage (run with the noise and tone taps into M): the middle fit, the
// low-noise (2) and high-noise (0) masks and their fits, the twelve interpolated curves, then the floor render,
// couple/quantise/normalise and nonzero propagation of all 15 curves.  posts / nonzero / iwork are blob-major
// with blob_blocks blocks (>= nblocks) from one curve to the next.
static int managed_tail(vb200_ctx *c, int W, int nblocks, long long blob_blocks, const vb200_block_desc *d_desc,
                        const float *mdct, const float *logmdct, const float *logmask, const MgdScratch &M,
                        int32_t *posts, int32_t *nonzero, int32_t *iwork, cudaStream_t st) {
  constexpr int NB = VB200_PACKETBLOBS, MID = VB200_PACKETBLOBS / 2;
  const int ch = c->setup.channels, n = c->dx[W].N / 2;
  const size_t rows = (size_t)nblocks * ch, brows = (size_t)blob_blocks * ch, pblob = brows * VB200_FLOOR1_STRIDE;
  int32_t *fz_lo = M.fz3, *fz_mid = M.fz3 + rows, *fz_hi = M.fz3 + 2 * rows;
  int rc;
  // the middle curve (select 1, what un-managed mode codes), then the low-noise (2) and high-noise (0) masks
  if ((rc = vb200_floor1_fit_dev(c, W, -1, (int)rows, logmdct, logmask, posts + MID * pblob, fz_mid, st))) return rc;
  const PsyDev &P0 = c->dpsy[(W ? 2 : 0)], &P1 = c->dpsy[(W ? 2 : 0) + 1];
  const long long total = (long long)rows * n;
  for (int pass = 0; pass < 2; pass++) {
    const int sel = pass ? 0 : 2;
    k_mix_select<<<grid_for(c, (int)((total + 255) / 256), 8), 256, 0, st>>>(P0, P1, d_desc, ch, total, sel, M.noise,
                                                                            M.tone, logmdct, M.alt);
    if ((rc = post_launch(c))) return rc;
    if ((rc = vb200_floor1_fit_dev(c, W, -1, (int)rows, logmdct, M.alt, posts + (sel ? NB - 1 : 0) * pblob,
                                   sel ? fz_hi : fz_lo, st))) return rc;
  }
  k_floor1_interpolate<<<grid_for(c, (int)((rows * VB200_FLOOR1_STRIDE + 255) / 256), 8), 256, 0, st>>>(
      (long long)rows, (long long)brows, posts, fz_lo, fz_mid, fz_hi, M.present);
  if ((rc = post_launch(c))) return rc;
  if ((rc = floor1_render_launch(c, W, -1, (int)rows, NB, (long long)brows, posts, M.present, iwork, nonzero, st)))
    return rc;
  return cqn_curves_launch(c, W, d_desc, nblocks, blob_blocks, mdct, iwork, nonzero, st);
}

// all pointers device; S holds the float intermediates.  M: bitrate-managed, the psy stage taps into M and
// managed_tail codes every curve (blobno unused); null: the curve of blob blobno
static int encode_launch(vb200_ctx *c, int W, int nstreams, int bps, int blobno, const vb200_encode_io *d,
                         const EncScratch &S, cudaStream_t st, const MgdScratch *M = nullptr) {
  const int ch = c->setup.channels, nblocks = nstreams * bps, rows = nblocks * ch;
  vb200_phaseA_io a;
  memset(&a, 0, sizeof(a));
  a.desc = d->desc; a.mdct = S.mdct; a.logmdct = S.logmdct; a.logmask = S.logmask; a.ampmax_out = d->ampmax_out;
  if (M) { a.tap_noise = M->noise; a.tap_tone = M->tone; }
  PcmSrc ps; const PcmSrc *pp = nullptr;
  if (d->pcm_fmt == VB200_PCM_F32_BLOCKS) a.pcm = (const float *)d->pcm;
  else { ps.base = d->pcm; ps.fmt = d->pcm_fmt; ps.bps = bps; ps.hop = d->hop; ps.stride = d->stream_stride; ps.blk_src = nullptr; pp = &ps; }
  int rc;
  if ((rc = phaseA_launch(c, W, nblocks, &a, d->independent ? 0 : nstreams, bps, d->ampmax0, st,
                          S.logfft, S.lmax, S.gmax, pp))) return rc;
  if (M)
    return managed_tail(c, W, nblocks, nblocks, d->desc, S.mdct, S.logmdct, S.logmask, *M, d->posts, d->nonzero,
                        (int32_t *)d->iwork, st);
  if ((rc = vb200_floor1_fit_dev(c, W, -1, rows, S.logmdct, S.logmask, d->posts, S.fitnz, st))) return rc;
  if (c->profiling) CU(cudaEventRecord(c->ev[4], st));
  const bool s16 = d->iwork_fmt == VB200_IWORK_S16;
  int32_t *iw = s16 ? S.iw32 : (int32_t *)d->iwork;
  if ((rc = vb200_floor1_render_dev(c, W, -1, rows, d->posts, S.fitnz, iw, d->nonzero, st))) return rc;
  if (c->profiling) CU(cudaEventRecord(c->ev[5], st));
  CqnDev Q0, Q1;
  if ((rc = cqn_setup(c, W, 0, blobno, &Q0))) return rc;
  if ((rc = cqn_setup(c, W, 1, blobno, &Q1))) return rc;
  if ((rc = cqn_launch(c, Q0, Q1, d->desc, nblocks, S.mdct, iw, d->nonzero, st))) return rc;
  if (d->classes &&
      (rc = vb200_residue_classify_dev(c, W, nblocks, iw, d->nonzero, d->classes, (int)d->class_stride, st))) return rc;
  if (s16) {
    const int n = c->dx[W].N / 2;
    const long nvec = (long)rows * n / 4;
    int lg = 0;
    while ((1L << lg) < (long)ch * n / 4) lg++;
    if ((1L << lg) != (long)ch * n / 4) lg = -1;      // channels not a power of two (5.1): per-block counts by division
    CU(cudaMemsetAsync(d->overflow, 0, sizeof(int32_t) * (size_t)nblocks, st));
    k_pack_s16<<<grid_for(c, (int)((nvec + 255) / 256), 8), 256, 0, st>>>((const int4 *)iw, (short4 *)d->iwork, nvec, lg, (int)((long)ch * n / 4), d->overflow);
    if ((rc = post_launch(c))) return rc;
  }
  if (c->profiling) CU(cudaEventRecord(c->ev[6], st));
  return 0;
}

// the chain's regions of an arena; d: the caller's spectra where it gives them
static void enc_layout(Carve &k, size_t rows, size_t nblocks, size_t n, const vb200_encode_io *d, bool s16,
                       EncScratch *S) {
  S->mdct = d && d->mdct ? d->mdct : k.take<float>(rows * n);
  S->logmdct = d && d->logmdct ? d->logmdct : k.take<float>(rows * n);
  S->logmask = d && d->logmask ? d->logmask : k.take<float>(rows * n);
  S->logfft = k.take<float>(rows * n);
  S->lmax = k.take<float>(rows);
  S->gmax = k.take<float>(nblocks);
  S->fitnz = k.take<int32_t>(rows);
  S->iw32 = s16 ? k.take<int32_t>(rows * n) : nullptr;
}

extern "C" int vb200_encode_dsp_dev(vb200_ctx *c, int W, int nstreams, int bps, int blobno,
                                    const vb200_encode_io *d, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  int rc;
  if ((rc = enc_check(c, W, nstreams, bps, blobno, d))) return rc;
  const size_t ch = c->setup.channels, n = c->dx[W].N / 2, nblocks = (size_t)nstreams * bps;
  EncScratch S;
  if ((rc = carve(c->enc, [&](Carve &k) { enc_layout(k, nblocks * ch, nblocks, n, d, d->iwork_fmt == VB200_IWORK_S16, &S); })))
    return rc;
  // Two half-batches (whole streams each) on two internal streams, every kernel launched with half its
  // grid: the halves drift apart, so CTAs of different kernels (shared-memory bound transform, issue bound
  // psy, latency bound floor fit) share the SMs instead of one kernel type owning the machine at a time.
  // H100 80GB HBM3 at a 700 W limit, 100 000 blocks: 6.27-6.28 M blocks/s split, 6.17-6.18 M in one piece.
  if ((rc = scratch_begin(c, (cudaStream_t)stream))) return rc;
  if (nstreams < 2 || c->profiling || nblocks < 2048) {
    if ((rc = encode_launch(c, W, nstreams, bps, blobno, d, S, (cudaStream_t)stream))) return rc;
    return scratch_end(c, (cudaStream_t)stream);
  }
  cudaStream_t user = (cudaStream_t)stream;
  CU(cudaEventRecord(c->ev_fork, user));
  c->grid_div = 2;
  for (int k = 0, s0 = 0; k < 2; k++) {
    const int ns = k ? nstreams - s0 : nstreams / 2;
    const size_t b0 = (size_t)s0 * bps, r0 = b0 * ch;
    vb200_encode_io h = *d;
    EncScratch T = S;
    h.pcm = (const char *)d->pcm + enc_pcm_bytes(d, (int)ch, c->dx[W].N, 1, bps) * s0;
    h.desc = d->desc + b0;
    if (d->ampmax0) h.ampmax0 = d->ampmax0 + s0;
    h.posts = d->posts + r0 * VB200_FLOOR1_STRIDE; h.nonzero = d->nonzero + r0; h.ampmax_out = d->ampmax_out + b0;
    h.iwork = (char *)d->iwork + (d->iwork_fmt == VB200_IWORK_S16 ? sizeof(int16_t) : sizeof(int32_t)) * r0 * n;
    if (d->overflow) h.overflow = d->overflow + b0;
    if (d->classes) h.classes = d->classes + r0 * (size_t)d->class_stride;
    T.mdct += r0 * n; T.logmdct += r0 * n; T.logmask += r0 * n; T.logfft += r0 * n;
    T.lmax += r0; T.gmax += b0; T.fitnz += r0;
    if (T.iw32) T.iw32 += r0 * n;
    cudaError_t e = cudaStreamWaitEvent(c->s_split[k], c->ev_fork, 0);
    if (e == cudaSuccess) rc = encode_launch(c, W, ns, bps, blobno, &h, T, c->s_split[k]);
    if (rc || e != cudaSuccess) { c->grid_div = 1; return rc ? rc : fail(VB200_EFAULT, "encode split", e); }
    s0 += ns;
  }
  for (int k = 0; k < 2; k++) {
    cudaError_t e = cudaEventRecord(c->ev_join[k], c->s_split[k]);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(user, c->ev_join[k], 0);
    if (e != cudaSuccess) { c->grid_div = 1; return fail(VB200_EFAULT, "encode split join", e); }
  }
  c->grid_div = 1;
  return scratch_end(c, user);
}

static int managed_check(vb200_ctx *c, int W, int nstreams, int bps, const vb200_encode_io *io,
                         bool own_outputs = false) {
  int rc;
  if ((rc = enc_check(c, W, nstreams, bps, VB200_PACKETBLOBS / 2, io, own_outputs))) return rc;
  if (io->iwork_fmt != VB200_IWORK_S32) return fail(VB200_EINVAL, "managed mode writes int32 residue");
  if (io->classes) return fail(VB200_EINVAL, "managed mode does not classify");
  return 0;
}

extern "C" int vb200_encode_dsp_managed_dev(vb200_ctx *c, int W, int nstreams, int bps, const vb200_encode_io *d,
                                            void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  int rc;
  if ((rc = managed_check(c, W, nstreams, bps, d))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t ch = c->setup.channels, n = c->dx[W].N / 2, nblocks = (size_t)nstreams * bps, rows = nblocks * ch;
  EncScratch S;
  MgdScratch M;
  if ((rc = carve(c->mgd, [&](Carve &k) {
         enc_layout(k, rows, nblocks, n, nullptr, false, &S);        // the caller's spectra are not used
         mgd_layout(k, rows, rows, n, &M);
       }))) return rc;
  if ((rc = scratch_begin(c, st))) return rc;
  if ((rc = encode_launch(c, W, nstreams, bps, VB200_PACKETBLOBS / 2, d, S, st, &M))) return rc;
  return scratch_end(c, st);
}

// host buffers: one synchronous H2D - compute - D2H round trip (managed mode is not the throughput path)
extern "C" int vb200_encode_dsp_managed(vb200_ctx *c, int W, int nstreams, int bps, const vb200_encode_io *h) {
  CHECK_CTX(c); CHECK_W(W);
  int rc;
  if ((rc = managed_check(c, W, nstreams, bps, h))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels, N = c->dx[W].N, n = N / 2;
  const size_t nb = (size_t)nstreams * bps, rows = nb * ch;
  constexpr int NB = VB200_PACKETBLOBS;
  HostIO io{c};
  vb200_encode_io d = *h;
  d.mdct = d.logmdct = d.logmask = nullptr;
  enc_stage(io, h, &d, ch, N, nstreams, bps, NB);
  if (io.rc) return io.rc;
  if ((rc = vb200_encode_dsp_managed_dev(c, W, nstreams, bps, &d, c->s_main))) return rc;
  io.back(h->posts, d.posts, NB * rows * VB200_FLOOR1_STRIDE);
  io.back(h->nonzero, d.nonzero, NB * rows);
  io.back(h->iwork, d.iwork, sizeof(int32_t) * NB * rows * n);
  io.back(h->ampmax_out, d.ampmax_out, nb);
  return io.sync();
}

extern "C" int vb200_encode_dsp(vb200_ctx *c, int W, int nstreams, int bps, int blobno, const vb200_encode_io *h) {
  CHECK_CTX(c); CHECK_W(W);
  int rc;
  if ((rc = enc_check(c, W, nstreams, bps, blobno, h))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels, N = c->dx[W].N, n = N / 2;
  HostPipe pipe(c, nstreams, bps, 8192);             // H100 80GB HBM3 at a 400 W limit (ramped schedule): 4096 -> 5.34, 8192 -> 5.36, 16384 -> 5.21 M blocks/s end to end
  const int cs = pipe.full;                          // whole streams per chunk
  const size_t pcm_per_stream = enc_pcm_bytes(h, ch, N, 1, bps);
  const bool s16 = h->iwork_fmt == VB200_IWORK_S16;
  const size_t isz = s16 ? sizeof(int16_t) : sizeof(int32_t), cb = (size_t)cs * bps, crow = cb * ch;
  vb200_encode_io dset[ENC_SETS];
  EncScratch sset[ENC_SETS];
  for (int s0 = 0, it = 0; it < (int)pipe.sched.size(); s0 += pipe.sched[it], it++) {
    const int L = it % ENC_SETS, ns = pipe.sched[it];
    const size_t nb = (size_t)ns * bps, b0 = (size_t)s0 * bps, rows = nb * ch, r0 = b0 * ch;
    vb200_encode_io &d = dset[L];
    EncScratch &S = sset[L];
    if (it < ENC_SETS) {                             // the set's first chunk: every chunk fits cs streams
      d = *h;
      d.mdct = d.logmdct = d.logmask = nullptr;
      if ((rc = carve(c->set[L], [&](Carve &k) {
             d.pcm = k.take<char>(pcm_per_stream * cs); d.desc = k.take<vb200_block_desc>(cb);
             d.ampmax0 = h->ampmax0 ? k.take<float>(cs) : nullptr;
             d.posts = k.take<int32_t>(crow * VB200_FLOOR1_STRIDE); d.nonzero = k.take<int32_t>(crow);
             d.iwork = k.take<char>(isz * crow * n);
             d.overflow = s16 ? k.take<int32_t>(cb) : nullptr;
             d.classes = h->classes ? k.take<int32_t>(crow * (size_t)h->class_stride) : nullptr;
             d.ampmax_out = k.take<float>(cb);
             enc_layout(k, crow, cb, n, nullptr, s16, &S);
           }))) return rc;
    }
    pipe.in(d.pcm, (const char *)h->pcm + pcm_per_stream * s0, pcm_per_stream * ns);
    pipe.in(d.desc, h->desc + b0, nb);
    if (h->ampmax0) pipe.in(d.ampmax0, h->ampmax0 + s0, ns);
    if ((rc = pipe.run(it, [&](cudaStream_t st) { return encode_launch(c, W, ns, bps, blobno, &d, S, st); })))
      return rc;
    pipe.back(h->posts + r0 * VB200_FLOOR1_STRIDE, d.posts, rows * VB200_FLOOR1_STRIDE);
    pipe.back(h->nonzero + r0, d.nonzero, rows);
    pipe.back((char *)h->iwork + isz * r0 * n, d.iwork, isz * rows * n);
    if (s16) pipe.back(h->overflow + b0, d.overflow, nb);
    if (h->classes) pipe.back(h->classes + r0 * (size_t)h->class_stride, d.classes, rows * (size_t)h->class_stride);
    pipe.back(h->ampmax_out + b0, d.ampmax_out, nb);
    if (h->mdct) pipe.back(h->mdct + r0 * n, S.mdct, rows * n);
    if (h->logmdct) pipe.back(h->logmdct + r0 * n, S.logmdct, rows * n);
    if (h->logmask) pipe.back(h->logmask + r0 * n, S.logmask, rows * n);
  }
  return pipe.sync();
}

// ======================================================================== //
// whole streams: block planning and the two size batches
static int envelope_search_launch(vb200_ctx *c, int nstreams, const void *d_pcm, int fmt, int64_t stride,
                                  int first_step, int nsteps, int32_t *d_state, uint8_t *d_ret, void *stream,
                                  const int32_t *d_steps_per_stream, const int32_t *d_first_per_stream);

static int plan_check(vb200_ctx *c) {
  if (c->n_psy != 4) return fail(VB200_EINVAL, "context has no psy setup");
  if ((c->setup.blocksizes[0] / 4) % PLAN_STEP) return fail(VB200_EIMPL, "blocksizes[0]/4 must be a multiple of the 64-sample envelope step");
  return 0;
}

// device: marks -> plan (slots final), gather tables and descriptors of both sizes; d_totals[2] on the device.
// d_work: 4 * nstreams ints of scratch.
static int plan_launch(vb200_ctx *c, int nstreams, const int32_t *d_mark, int64_t mark_stride, int nsteps,
                       const int64_t *d_len, const int64_t *d_eof, int max_blocks, vb200_stream_block *d_plan,
                       int32_t *d_nblocks, const int cap[2], int2 *d_src[2], vb200_block_desc *d_desc[2],
                       int32_t *d_totals, int32_t *d_work, cudaStream_t st, const CarryDev *K = nullptr) {
  int32_t *d_counts = d_work, *d_offs = d_work + 2 * (size_t)nstreams;
  const int g = (nstreams + 127) / 128;
  if (K)
    k_plan_blocks_carry<<<g, 128, 0, st>>>(nstreams, c->setup.blocksizes[0], c->setup.blocksizes[1], d_mark, mark_stride,
                                           nsteps, d_len, d_eof, max_blocks, d_plan, d_nblocks, d_counts, *K);
  else
    k_plan_blocks<<<g, 128, 0, st>>>(nstreams, c->setup.blocksizes[0], c->setup.blocksizes[1], d_mark, mark_stride, nsteps,
                                     d_len, d_eof, max_blocks, d_plan, d_nblocks, d_counts);
  k_plan_offsets<<<1, 32, 0, st>>>(nstreams, d_counts, d_offs, d_totals);
  k_plan_fill<<<g, 128, 0, st>>>(nstreams, max_blocks, d_plan, d_nblocks, d_offs, cap[0], cap[1],
                                 d_src[0], d_src[1], d_desc[0], d_desc[1]);
  return post_launch(c, 3);
}

extern "C" int vb200_plan_blocks(vb200_ctx *c, int nstreams, const int32_t *mark, int64_t mark_stride, int nsteps,
                                 const int64_t *pcm_len, const int64_t *eof, int max_blocks,
                                 vb200_stream_block *plan, int32_t *nblocks) {
  CHECK_CTX(c);
  int rc;
  if ((rc = plan_check(c))) return rc;
  if (nstreams <= 0) return 0;
  if (!mark || !pcm_len || !plan || !nblocks || max_blocks < 1 || nsteps < 0 || mark_stride < nsteps + 3)
    return fail(VB200_EINVAL, "plan_blocks arguments");
  std::lock_guard<std::mutex> lk(c->mu);
  cudaStream_t st = c->s_main;
  const size_t cap = (size_t)nstreams * max_blocks;
  HostIO io{c};
  const int32_t *dm = io.in(mark, (size_t)nstreams * mark_stride);
  const int64_t *dl = io.in(pcm_len, nstreams), *de = eof ? io.in(eof, nstreams) : nullptr;
  vb200_stream_block *dp = io.out<vb200_stream_block>(cap);
  int32_t *dn = io.out<int32_t>(nstreams);
  if (io.rc) return io.rc;
  int32_t *d_tot, *d_work; int2 *d_src[2]; vb200_block_desc *d_desc[2];
  if ((rc = carve(c->plan, [&](Carve &k) {
         d_tot = k.take<int32_t>(2); d_work = k.take<int32_t>(4 * (size_t)nstreams);
         for (int w = 0; w < 2; w++) { d_src[w] = k.take<int2>(cap); d_desc[w] = k.take<vb200_block_desc>(cap); }
       }))) return rc;
  const int caps[2] = {(int)cap, (int)cap};
  if ((rc = scratch_begin(c, st))) return rc;
  if ((rc = plan_launch(c, nstreams, dm, mark_stride, nsteps, dl, de, max_blocks, dp, dn, caps, d_src, d_desc, d_tot,
                        d_work, st)))
    return rc;
  if ((rc = scratch_end(c, st))) return rc;
  io.back(plan, dp, cap);
  io.back(nblocks, dn, nstreams);
  return io.sync();
}

// The start of every streams call: the context's plan setup and the io, whose count[] is zeroed.  A call that has
// checks of its own runs them next, then returns for nstreams <= 0, then checks streams_inputs.
static int streams_open(vb200_ctx *c, vb200_streams_io *h) {
  int rc;
  if ((rc = plan_check(c))) return rc;
  if (!h) return fail(VB200_EINVAL, "null io");
  h->count[0] = h->count[1] = 0;
  return 0;
}

// the inputs every streams call reads; name: the call, for the message
static int streams_inputs(const vb200_streams_io *h, const char *name) {
  if (!h->pcm || !h->pcm_len || !h->plan || !h->nblocks || h->max_blocks < 1)
    return fail(VB200_EINVAL, (std::string(name) + ": pcm, pcm_len, plan, nblocks").c_str());
  return 0;
}

// arguments of the device streams calls; zeroes count[] (nstreams <= 0: nothing to do)
static int streams_check(vb200_ctx *c, int nstreams, vb200_streams_io *d) {
  int rc;
  if ((rc = streams_open(c, d)) || nstreams <= 0) return rc;
  if ((rc = streams_inputs(d, "encode_streams"))) return rc;
  if (d->pcm_fmt != VB200_PCM_F32_PLANAR && d->pcm_fmt != VB200_PCM_S16_INTERLEAVED) return fail(VB200_EINVAL, "pcm_fmt");
  for (int w = 0; w < 2; w++)
    if (d->cap[w] < 0 || (d->cap[w] > 0 && (!d->posts[w] || !d->nonzero[w] || !d->iwork[w] || !d->ampmax_out[w])))
      return fail(VB200_EINVAL, "encode_streams: outputs of a size with capacity > 0");
  if (d->stream_stride < c->setup.blocksizes[1]) return fail(VB200_EINVAL, "stream_stride");
  return cqn_channels_check(c);
}

// The front half of both streams calls, up to the psy stage: envelope search, marks, plan, the transforms of
// both sizes and the ampmax chain along every stream.  Sets count[]; for each size with blocks, S[w] holds the
// transforms, a[w] the psy stage's io, d_desc[w] the batch's block descriptors and, given M, M[w] the scratch of
// the managed tail, which a[w] taps the noise and tone masks into.  Begins the call's use of the context scratch.
// K: carried streams (the envelope state, marks, planner and ampmax chain start from the carries and go back to
// them); K->count's largest entry is nsteps_env.
// async_tot (the _dev raw-PCM calls): nothing waits for the plan.  The launches and carves after it are sized by
// cap[] (count[] = cap[]), k_plan_pad fills the slots the plan leaves empty with a valid block, and *async_tot gets
// the plan's device totals; a plan past cap[] or a mark window overflow is for the caller to report on the device.
static int streams_front(vb200_ctx *c, int nstreams, vb200_streams_io *d, cudaStream_t st, EncScratch S[2],
                         vb200_phaseA_io a[2], vb200_block_desc *d_desc[2], MgdScratch *M = nullptr,
                         const CarryDev *K = nullptr, int nsteps_env = 0, const int32_t **async_tot = nullptr) {
  int rc;
  const int ch = c->setup.channels;
  // 1. envelope search over the whole timeline (fresh detector state), 2. marks, 3. plan
  const int nsteps = (int)(d->stream_stride / PLAN_STEP) - PLAN_VE_WIN;
  if (nsteps < 1) return fail(VB200_EINVAL, "stream too short");
  const int64_t mark_stride = nsteps + 4;
  const size_t sw = VB200_VE_STATE_WORDS(ch);
  const int nret = K ? nsteps_env : nsteps;
  int32_t *d_state, *d_mark, *d_tot, *d_work; uint8_t *d_ret; int2 *d_src[2];
  if ((rc = carve(c->plan, [&](Carve &k) {
         d_state = K ? nullptr : k.take<int32_t>(sw * nstreams);      // carried streams use the carries' state
         d_ret = k.take<uint8_t>((size_t)nstreams * (nret > 0 ? nret : 1));
         d_mark = k.take<int32_t>((size_t)nstreams * mark_stride); d_tot = k.take<int32_t>(2);
         d_work = k.take<int32_t>(4 * (size_t)nstreams);
         for (int w = 0; w < 2; w++) {
           const size_t cw = d->cap[w] > 0 ? d->cap[w] : 1;
           d_src[w] = k.take<int2>(cw); d_desc[w] = k.take<vb200_block_desc>(cw);
         }
       }))) return rc;
  if ((rc = scratch_begin(c, st))) return rc;
  if (K) {
    if (nret > 0 && (rc = envelope_search_launch(c, nstreams, d->pcm, d->pcm_fmt, d->stream_stride, 0, nret, K->env, d_ret,
                                                 st, K->count, K->first))) return rc;
  } else {
    CU(cudaMemsetAsync(d_state, 0, sizeof(int32_t) * sw * nstreams, st));
    if ((rc = vb200_envelope_search_dev(c, nstreams, d->pcm, d->pcm_fmt, d->stream_stride, 0, nsteps, d_state, d_ret, st))) return rc;
  }
  {
    const long long total = (long long)nstreams * mark_stride;
    if (K)
      k_env_marks_carry<<<grid_for(c, (int)((total + 255) / 256), 8), 256, 0, st>>>(nstreams, nret, d_ret, d_mark,
                                                                                    mark_stride, *K);
    else
      k_env_marks<<<grid_for(c, (int)((total + 255) / 256), 8), 256, 0, st>>>(nstreams, nsteps, d_ret, d->pcm_len, d_mark, mark_stride);
    if ((rc = post_launch(c))) return rc;
  }
  if ((rc = plan_launch(c, nstreams, d_mark, mark_stride, nsteps, d->pcm_len, d->eof, d->max_blocks, d->plan, d->nblocks,
                        d->cap, d_src, d_desc, d_tot, d_work, st, K))) return rc;
  int tot[2], overflow = 0;
  if (async_tot) {
    tot[0] = d->cap[0]; tot[1] = d->cap[1];
    *async_tot = d_tot;
    if (tot[0] > 0 || tot[1] > 0) {
      k_plan_pad<<<dim3(grid_for(c, (std::max(tot[0], tot[1]) + 255) / 256, 8), 2), 256, 0, st>>>(
          d_tot, tot[0], tot[1], d_src[0], d_src[1], d_desc[0], d_desc[1]);
      if ((rc = post_launch(c))) return rc;
    }
  } else {
    CU(cudaMemcpyAsync(tot, d_tot, sizeof(tot), cudaMemcpyDeviceToHost, st));
    if (K) CU(cudaMemcpyAsync(&overflow, K->overflow, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));                     // the launches below are sized by the plan
  }
  d->count[0] = tot[0]; d->count[1] = tot[1];
  if (overflow) return fail(VB200_EINVAL, "encode carry: the mark window does not fit the carry's mark capacity");
  if (tot[0] > d->cap[0] || tot[1] > d->cap[1]) return fail(VB200_EINVAL, "encode_streams: more blocks than cap[] (count[] holds the need)");
  // 4. transforms of both sizes, 5. the ampmax chain along every stream
  if ((rc = carve(c->chain, [&](Carve &k) {
         for (int w = 0; w < 2; w++) {
           const size_t n = c->dx[w].N / 2, nb = tot[w];
           if (!nb) continue;
           enc_layout(k, nb * ch, nb, n, nullptr, false, &S[w]);
           if (M) mgd_layout(k, nb * ch, (size_t)d->cap[w] * ch, n, &M[w]);
         }
       }))) return rc;
  for (int w = 0; w < 2; w++) {
    memset(&a[w], 0, sizeof(a[w]));
    if (!tot[w]) continue;
    const size_t nb = tot[w];
    a[w].desc = d_desc[w]; a[w].mdct = S[w].mdct; a[w].logmdct = S[w].logmdct; a[w].logmask = S[w].logmask;
    a[w].ampmax_out = d->ampmax_out[w];
    if (M) { a[w].tap_noise = M[w].noise; a[w].tap_tone = M[w].tone; }
    PcmSrc ps; ps.base = d->pcm; ps.fmt = d->pcm_fmt; ps.bps = 1; ps.hop = 0; ps.stride = d->stream_stride; ps.blk_src = d_src[w];
    if ((rc = phaseA_transform_launch(c, w, (int)nb, &a[w], ps, st, S[w].logfft, S[w].lmax))) return rc;
  }
  {
    float sa[2];
    for (int w = 0; w < 2; w++) sa[w] = ((float)(c->dx[w].N / 2) / (float)c->setup.rate) * c->setup.ampmax_att_per_sec;   // lib/psy.c:843
    for (int w = 0; w < 2; w++)                        // the padded slots' ampmax, which nothing reads
      if (async_tot && tot[w]) CU(cudaMemsetAsync(S[w].gmax, 0, sizeof(float) * tot[w], st));
    if (K)
      k_ampmax_plan_carry<<<(nstreams + 127) / 128, 128, 0, st>>>(nstreams, d->max_blocks, ch, d->plan, d->nblocks,
                                                                  tot[0] ? S[0].lmax : nullptr, tot[1] ? S[1].lmax : nullptr,
                                                                  sa[0], sa[1], tot[0] ? S[0].gmax : nullptr,
                                                                  tot[1] ? S[1].gmax : nullptr, tot[0], tot[1], K->pc);
    else
      k_ampmax_plan<<<(nstreams + 127) / 128, 128, 0, st>>>(nstreams, d->max_blocks, ch, d->plan, d->nblocks,
                                                            tot[0] ? S[0].lmax : nullptr, tot[1] ? S[1].lmax : nullptr,
                                                            sa[0], sa[1], tot[0] ? S[0].gmax : nullptr, tot[1] ? S[1].gmax : nullptr,
                                                            tot[0], tot[1]);
    if ((rc = post_launch(c))) return rc;
  }
  return 0;
}

// managed: the bitrate-managed chain, every curve cap[w] blocks after the one before (blobno unused).  desc_out
// (optional): the two batches' block descriptors, which stay in the plan arena until its next carve
static int encode_streams_launch(vb200_ctx *c, int nstreams, int blobno, bool managed, vb200_streams_io *d,
                                 cudaStream_t st, vb200_block_desc **desc_out, const CarryDev *K = nullptr,
                                 int nsteps_env = 0, const int32_t **async_tot = nullptr) {
  int rc;
  if ((rc = streams_check(c, nstreams, d)) || nstreams <= 0) return rc;
  if (!managed && (blobno < 0 || blobno >= VB200_PACKETBLOBS)) return fail(VB200_EINVAL, "blobno");
  const int ch = c->setup.channels;
  EncScratch S[2];
  vb200_phaseA_io a[2];
  vb200_block_desc *d_desc[2];
  MgdScratch M[2];
  if ((rc = streams_front(c, nstreams, d, st, S, a, d_desc, managed ? M : nullptr, K, nsteps_env, async_tot))) return rc;
  // 6. the rest of the chain per size
  for (int w = 0; w < 2; w++) {
    if (!d->count[w]) continue;
    const int nb = d->count[w], rows = nb * ch;
    if ((rc = phaseA_psy_launch(c, w, nb, &a[w], st, S[w].logfft, S[w].lmax, S[w].gmax))) return rc;
    if (managed) {
      if ((rc = managed_tail(c, w, nb, d->cap[w], d_desc[w], S[w].mdct, S[w].logmdct, S[w].logmask, M[w], d->posts[w],
                             d->nonzero[w], d->iwork[w], st))) return rc;
      continue;
    }
    if ((rc = vb200_floor1_fit_dev(c, w, -1, rows, S[w].logmdct, S[w].logmask, d->posts[w], S[w].fitnz, st))) return rc;
    if ((rc = vb200_floor1_render_dev(c, w, -1, rows, d->posts[w], S[w].fitnz, d->iwork[w], d->nonzero[w], st))) return rc;
    CqnDev Q0, Q1;
    if ((rc = cqn_setup(c, w, 0, blobno, &Q0))) return rc;
    if ((rc = cqn_setup(c, w, 1, blobno, &Q1))) return rc;
    if ((rc = cqn_launch(c, Q0, Q1, d_desc[w], nb, S[w].mdct, d->iwork[w], d->nonzero[w], st))) return rc;
  }
  if (desc_out) { desc_out[0] = d_desc[0]; desc_out[1] = d_desc[1]; }
  return scratch_end(c, st);
}

extern "C" int vb200_encode_streams_dev(vb200_ctx *c, int nstreams, int blobno, vb200_streams_io *d, void *stream) {
  CHECK_CTX(c);
  return encode_streams_launch(c, nstreams, blobno, false, d, (cudaStream_t)stream, nullptr);
}

extern "C" int vb200_encode_streams_managed_dev(vb200_ctx *c, int nstreams, vb200_streams_io *d, void *stream) {
  CHECK_CTX(c);
  return encode_streams_launch(c, nstreams, 0, true, d, (cudaStream_t)stream, nullptr);
}

// A host vb200_streams_io staged through io into the device copy d: the inputs copied in (the pcm only when
// stage_pcm, else h->pcm is already on the device), the plan and nblocks, and for each size with cap[w] > 0 the
// outputs of cap[w] blocks, of every curve for managed.
static void streams_stage(vb200_ctx *c, HostIO &io, int nstreams, bool managed, bool stage_pcm,
                          const vb200_streams_io *h, vb200_streams_io *d) {
  const size_t ch = c->setup.channels, curves = managed ? VB200_PACKETBLOBS : 1;
  const size_t pcm_bytes = (size_t)nstreams * ch * (size_t)h->stream_stride * (h->pcm_fmt == VB200_PCM_S16_INTERLEAVED ? 2 : 4);
  *d = *h;
  if (stage_pcm) d->pcm = io.in(h->pcm, pcm_bytes);
  d->pcm_len = io.in(h->pcm_len, nstreams);
  if (h->eof) d->eof = io.in(h->eof, nstreams);
  d->plan = io.out<vb200_stream_block>((size_t)nstreams * h->max_blocks);
  d->nblocks = io.out<int32_t>(nstreams);
  for (int w = 0; w < 2; w++) {
    if (h->cap[w] <= 0) continue;
    const size_t rows = curves * h->cap[w] * ch, n = c->dx[w].N / 2;
    d->posts[w] = io.out<int32_t>(rows * VB200_FLOOR1_STRIDE);
    d->nonzero[w] = io.out<int32_t>(rows);
    d->iwork[w] = io.out<int32_t>(rows * n);
    d->ampmax_out[w] = io.out<float>(h->cap[w]);
  }
}

// host buffers of both streams calls: one synchronous H2D - compute - D2H round trip.  managed: every output but
// ampmax_out holds the VB200_PACKETBLOBS curves one after the other, cap[W] blocks apart, and count[W] blocks of each
// come back.
static int streams_host(vb200_ctx *c, int nstreams, int blobno, bool managed, vb200_streams_io *h) {
  int rc;
  if ((rc = streams_open(c, h)) || nstreams <= 0) return rc;
  if ((rc = streams_inputs(h, "encode_streams"))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t ch = c->setup.channels, pcap = (size_t)nstreams * h->max_blocks;
  const int curves = managed ? VB200_PACKETBLOBS : 1;
  HostIO io{c};
  vb200_streams_io d;
  streams_stage(c, io, nstreams, managed, true, h, &d);
  if (io.rc) return io.rc;
  rc = encode_streams_launch(c, nstreams, blobno, managed, &d, c->s_main, nullptr);
  h->count[0] = d.count[0]; h->count[1] = d.count[1];
  if (rc) return rc;
  io.back(h->plan, d.plan, pcap);
  io.back(h->nblocks, d.nblocks, nstreams);
  for (int w = 0; w < 2; w++) {
    const size_t nb = d.count[w], n = c->dx[w].N / 2, cw = h->cap[w];
    if (!nb) continue;
    for (int k = 0; k < curves; k++) {
      const size_t r0 = k * cw * ch, p0 = r0 * VB200_FLOOR1_STRIDE;
      io.back(h->posts[w] + p0, d.posts[w] + p0, nb * ch * VB200_FLOOR1_STRIDE);
      io.back(h->nonzero[w] + r0, d.nonzero[w] + r0, nb * ch);
      io.back(h->iwork[w] + r0 * n, d.iwork[w] + r0 * n, nb * ch * n);
    }
    io.back(h->ampmax_out[w], d.ampmax_out[w], nb);
  }
  return io.sync();
}

extern "C" int vb200_encode_streams(vb200_ctx *c, int nstreams, int blobno, vb200_streams_io *h) {
  CHECK_CTX(c);
  return streams_host(c, nstreams, blobno, false, h);
}

extern "C" int vb200_encode_streams_managed(vb200_ctx *c, int nstreams, vb200_streams_io *h) {
  CHECK_CTX(c);
  return streams_host(c, nstreams, 0, true, h);
}

// ======================================================================== //
// residue partition classification
extern "C" int vb200_residue_partvals(vb200_ctx *c, int W) {
  if (!c || W < 0 || W > 1) return VB200_EINVAL;
  return c->res_partvals[W];
}

// curves == 1: nblocks blocks; curves == VB200_PACKETBLOBS: every curve of nblocks blocks, iwork / nonzero rows
// curve_rows apart (k_residue_classify_curves), classes [curves][nblocks][ch][class_stride]
static int residue_classify_launch(vb200_ctx *c, int W, int nblocks, int curves, long long curve_rows,
                                   const int32_t *d_iwork, const int32_t *d_nonzero, int32_t *d_classes,
                                   int class_stride, cudaStream_t st) {
  if (c->res_partvals[W] <= 0) return fail(VB200_EINVAL, "no residue setup for this block size");
  if (class_stride < c->res_partvals[W]) return fail(VB200_EINVAL, "class_stride < partvals");
  const int ch = c->setup.channels, n = c->dx[W].N / 2, submaps = c->setup.submaps[W] > 0 ? c->setup.submaps[W] : 1;
  for (int sm = 0; sm < submaps; sm++) {                   // the reads must stay inside the rows
    const vb200_residue_setup &r = c->setup.residue[W][sm];
    if (r.type < 0 || r.grouping <= 0) continue;
    int cib = 0;
    for (int k = 0; k < ch; k++) if (c->setup.chmux[W][k] == sm) cib++;
    const long reach = r.type == 2 ? (cib ? r.begin / cib + (long)((r.end - r.begin) / r.grouping) * ((r.grouping + cib - 1) / cib) : 0)
                                   : (long)r.begin + (long)((r.end - r.begin) / r.grouping) * r.grouping;
    if (reach > n) return fail(VB200_EINVAL, "residue range exceeds the block");
  }
  CU(cudaMemsetAsync(d_classes, 0, sizeof(int32_t) * curves * (size_t)nblocks * ch * class_stride, st));
  ResArgs A;
  A.res = c->d_res[W]; A.chmux = c->d_chmux[W]; A.ch = ch; A.n = n; A.submaps = submaps; A.nblocks = nblocks;
  A.stride = class_stride;
  const long tasks = (long)curves * nblocks * submaps;
  const int grid = grid_for(c, (int)((tasks + RES_WARPS - 1) / RES_WARPS), 16);
  if (curves == 1) k_residue_classify<<<grid, 32 * RES_WARPS, 0, st>>>(A, d_iwork, d_nonzero, d_classes);
  else k_residue_classify_curves<<<grid, 32 * RES_WARPS, 0, st>>>(A, curve_rows, d_iwork, d_nonzero, d_classes);
  return post_launch(c);
}

extern "C" int vb200_residue_classify_dev(vb200_ctx *c, int W, int nblocks, const int32_t *d_iwork,
                                          const int32_t *d_nonzero, int32_t *d_classes, int class_stride, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nblocks <= 0) return 0;
  if (!d_iwork || !d_nonzero || !d_classes) return fail(VB200_EINVAL, "residue_classify pointers");
  return residue_classify_launch(c, W, nblocks, 1, 0, d_iwork, d_nonzero, d_classes, class_stride, (cudaStream_t)stream);
}

extern "C" int vb200_residue_classify(vb200_ctx *c, int W, int nblocks, const int32_t *iwork, const int32_t *nonzero,
                                      int32_t *classes, int class_stride) {
  CHECK_CTX(c); CHECK_W(W);
  if (nblocks <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t ch = c->setup.channels, n = c->dx[W].N / 2;
  const size_t rows = nblocks * ch;
  HostIO io{c};
  const int32_t *di = io.in(iwork, rows * n), *dz = io.in(nonzero, rows);
  int32_t *dc = io.out<int32_t>(rows * (size_t)(class_stride > 0 ? class_stride : 1));
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_residue_classify_dev(c, W, nblocks, di, dz, dc, class_stride, c->s_main))) return rc;
  io.back(classes, dc, rows * (size_t)class_stride);
  return io.sync();
}

// ======================================================================== //
// decode: floor multiply and the fused decode chain
extern "C" int vb200_floor1_inverse2_dev(vb200_ctx *c, int W, int floor_sel, int nrows, const int32_t *d_posts,
                                         const int32_t *d_present, float *d_data, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  if (nrows <= 0) return 0;
  if (!d_posts || !d_present || !d_data) return fail(VB200_EINVAL, "floor1_inverse2 pointers");
  Floor1Args a; int rc;
  if ((rc = floor1_args(c, W, floor_sel, nrows, &a))) return rc;
  const int ctas = (nrows + F1_WARPS - 1) / F1_WARPS;
  k_floor1_inverse2<<<grid_for(c, ctas, 8), 32 * F1_WARPS, 0, (cudaStream_t)stream>>>(a, d_posts, d_present, d_data, c->d_fromdB);
  return post_launch(c);
}

extern "C" int vb200_floor1_inverse2(vb200_ctx *c, int W, int floor_sel, int nrows, const int32_t *posts,
                                     const int32_t *present, float *data) {
  CHECK_CTX(c); CHECK_W(W);
  if (nrows <= 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = c->dx[W].N / 2;
  HostIO io{c};
  const int32_t *dp = io.in(posts, (size_t)nrows * VB200_FLOOR1_STRIDE), *dz = io.in(present, nrows);
  float *dd = io.in(data, nrows * n);
  if (io.rc) return io.rc;
  int rc;
  if ((rc = vb200_floor1_inverse2_dev(c, W, floor_sel, nrows, dp, dz, dd, c->s_main))) return rc;
  io.back(data, dd, nrows * n);
  return io.sync();
}

static size_t entropy_smem(const EntDev &E, bool fused) {
  return (fused ? sizeof(int32_t) * (size_t)E.ch * (VB200_FLOOR1_STRIDE + 1) : 0) + 2 * (size_t)E.ch + E.cls_cap;
}

// CTAs per SM of k_decode_packets' grid.  One thread of each CTA decodes a packet serially while the others wait,
// but the kernel takes 80 registers (-Xptxas -v, sm_90a), so at most 6 CTAs of 128 threads are resident per SM;
// a grid of more than k_decode_prepare's 8 per SM would only queue
static const int DECODE_PACKETS_CTAS = 8;

static int ent_check(const vb200_ctx *c) {
  if (!c->ent.books) return fail(VB200_EINVAL, "no vb200_decode_entropy_setup registered");
  return 0;
}

// the front half of every decode chain on nstreams x nblk blocks: de-coupling and the floor-1 multiply of each
// block's rows in d_res, from the posts and presence of vb200_decode_entropy (k_decode_prepare) or, with packets P,
// from the entropy decode of each block's packet in front of them (k_decode_packets).  With d_count, the blocks of a
// stream past its count are skipped.
static int decode_front(vb200_ctx *c, int nstreams, int nblk, const int32_t *d_count, const int32_t *d_Wseq,
                        const int64_t *d_coef_off, float *d_res, const int32_t *d_posts, const int32_t *d_present,
                        const DecodePackets *P, cudaStream_t st) {
  const int ch = c->setup.channels;
  DecodePrepArgs A;
  for (int w = 0; w < 2; w++) {
    for (int k = 0; k < ch; k++)
      if (c->setup.floor1[w][c->setup.chmux[w][k]].posts <= 0)
        return fail(VB200_EINVAL, "no floor1 setup for a channel's submap");
    A.floors[w] = c->d_floor[w]; A.chmux[w] = c->d_chmux[w];
    A.mag[w] = c->d_mag[w]; A.ang[w] = c->d_ang[w];
    A.steps[w] = c->setup.coupling_steps[w]; A.n[w] = c->dx[w].N / 2;
  }
  A.ch = ch; A.nblk = nblk; A.nitems = (long)nstreams * nblk;
  const long long *coef_off = (const long long *)d_coef_off;
  if (P) {
    const size_t smem = entropy_smem(c->ent, true);
    auto *kern = d_count ? k_decode_packets<true> : k_decode_packets<false>;
    int rc = set_smem(kern, smem); if (rc) return rc;
    kern<<<grid_for(c, (int)A.nitems, DECODE_PACKETS_CTAS), 128, smem, st>>>(A, c->ent, *P, d_Wseq, coef_off, d_res,
                                                                            c->d_fromdB, d_count);
  } else {
    auto *kern = d_count ? k_decode_prepare<true> : k_decode_prepare<false>;
    kern<<<grid_for(c, (int)A.nitems, 8), 128, 0, st>>>(A, d_Wseq, coef_off, d_res, d_posts, d_present, c->d_fromdB,
                                                        d_count);
  }
  return post_launch(c);
}

extern "C" int vb200_decode_dsp_dev(vb200_ctx *c, int nstreams, int nblk, const int32_t *d_Wseq, const int64_t *d_coef_off,
                                    float *d_res, const int32_t *d_posts, const int32_t *d_present,
                                    const int64_t *d_pcm_off, void *d_pcm, int pcm_s16, int64_t pcm_stride, void *stream) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  if (!d_Wseq || !d_coef_off || !d_res || !d_posts || !d_present || !d_pcm_off || !d_pcm)
    return fail(VB200_EINVAL, "decode pointers");
  const cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = decode_front(c, nstreams, nblk, nullptr, d_Wseq, d_coef_off, d_res, d_posts, d_present, nullptr, st)))
    return rc;
  return synthesis_launch<SYN_PLAIN>(c, pcm_s16, nstreams, nblk, nullptr, d_Wseq, d_coef_off, d_res, d_pcm_off, d_pcm,
                                     pcm_stride, nullptr, DsTrim{}, st);
}

extern "C" int vb200_decode_dsp(vb200_ctx *c, int nstreams, int nblk, const int32_t *Wseq, const int64_t *coef_off,
                                float *res, int64_t res_len, const int32_t *posts, const int32_t *present,
                                const int64_t *pcm_off, void *pcm, int pcm_s16, int64_t pcm_stride) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  if (!Wseq || !coef_off || !res || !posts || !present || !pcm_off || !pcm) return fail(VB200_EINVAL, "decode pointers");
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels;
  const size_t nb = (size_t)nstreams * nblk;
  for (size_t i = 0; i < nb; i++) if (Wseq[i] < 0 || Wseq[i] > 1) return fail(VB200_EINVAL, "Wseq values must be 0/1");
  HostIO io{c};
  const int32_t *dW = io.in(Wseq, nb);
  const int64_t *dco = io.in(coef_off, nb);
  float *dc = io.in(res, (size_t)res_len);
  const int64_t *dpo = io.in(pcm_off, nb);
  const size_t pbytes = (pcm_s16 ? sizeof(int16_t) : sizeof(float)) * (size_t)nstreams * ch * (size_t)pcm_stride;
  void *dp = io.out<void>(pbytes);
  const int32_t *dps = io.in(posts, nb * ch * VB200_FLOOR1_STRIDE), *dpr = io.in(present, nb * ch);
  if (io.rc) return io.rc;
  CU(cudaMemsetAsync(dp, 0, pbytes, c->s_main));
  int rc;
  if ((rc = vb200_decode_dsp_dev(c, nstreams, nblk, dW, dco, dc, dps, dpr, dpo, dp, pcm_s16, pcm_stride, c->s_main)))
    return rc;
  io.back(pcm, dp, pbytes);
  return io.sync();
}

// ---- decode resumed across calls: the overlap of every (stream, channel) carried in vb200_decode_carry
// host-form checks of the blocks of nstreams x nblk: count[s] in [0, nblk] (all nblk without count), then of each
// counted block in order its flag and, for the packet forms (pkt_off given), its packet inside data and its rows
// inside res
static int blocks_check(const vb200_ctx *c, int nstreams, int nblk, const int32_t *count, const int32_t *Wseq,
                        const int64_t *pkt_off, const int32_t *pkt_bytes, int64_t data_bytes, const int64_t *coef_off,
                        int64_t res_len) {
  const int ch = c->setup.channels;
  for (int s = 0; s < nstreams; s++) {
    const int n = count ? count[s] : nblk;
    if (n < 0 || n > nblk) return fail(VB200_EINVAL, "count[s] must be in [0, nblk]");
    for (int k = 0; k < n; k++) {
      const size_t i = (size_t)s * nblk + k;
      if (Wseq[i] < 0 || Wseq[i] > 1) return fail(VB200_EINVAL, "Wseq values must be 0/1");
      if (!pkt_off) continue;
      if (pkt_bytes[i] < 0 || pkt_off[i] < 0 || pkt_off[i] > data_bytes || pkt_bytes[i] > data_bytes - pkt_off[i])
        return fail(VB200_EINVAL, "packet outside data");
      if (coef_off[i] < 0 || coef_off[i] + (int64_t)ch * (c->setup.blocksizes[Wseq[i]] / 2) > res_len)
        return fail(VB200_EINVAL, "block rows outside res");
    }
  }
  return 0;
}

// the vb200_decode_carry of a _resume host form: checked, staged after the call's other inputs, and written back
// after its PCM
struct HostCarry {
  vb200_decode_carry *h;
  size_t ntask, tlen;
  vb200_decode_carry d{};
  HostCarry(const vb200_ctx *c, int nstreams, vb200_decode_carry *carry)
      : h(carry), ntask((size_t)nstreams * c->setup.channels), tlen(ntask * (size_t)(c->setup.blocksizes[1] / 2)) {}
  int check() const {
    for (size_t i = 0; i < ntask; i++)
      if (h->W[i] < -1 || h->W[i] > 1) return fail(VB200_EINVAL, "carried W must be -1, 0 or 1");
    return 0;
  }
  void stage(HostIO &io) {
    d.tail = io.in(h->tail, tlen);
    d.W = io.in(h->W, ntask);
  }
  void write_back(HostIO &io) const {
    io.back(h->tail, d.tail, tlen);
    io.back(h->W, d.W, ntask);
  }
};

extern "C" int vb200_decode_dsp_resume_dev(vb200_ctx *c, int nstreams, int nblk, const int32_t *d_count,
                                           const int32_t *d_Wseq, const int64_t *d_coef_off, float *d_res,
                                           const int32_t *d_posts, const int32_t *d_present, const int64_t *d_pcm_off,
                                           void *d_pcm, int pcm_s16, int64_t pcm_stride,
                                           const vb200_decode_carry *d_carry, void *stream) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  if (!d_Wseq || !d_coef_off || !d_res || !d_posts || !d_present || !d_pcm_off || !d_pcm || !d_carry ||
      !d_carry->tail || !d_carry->W)
    return fail(VB200_EINVAL, "decode pointers");
  const cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = decode_front(c, nstreams, nblk, d_count, d_Wseq, d_coef_off, d_res, d_posts, d_present, nullptr, st)))
    return rc;
  return synthesis_launch<SYN_CARRY>(c, pcm_s16, nstreams, nblk, d_count, d_Wseq, d_coef_off, d_res, d_pcm_off, d_pcm,
                                     pcm_stride, d_carry, DsTrim{}, st);
}

extern "C" int vb200_decode_dsp_resume(vb200_ctx *c, int nstreams, int nblk, const int32_t *count, const int32_t *Wseq,
                                       const int64_t *coef_off, float *res, int64_t res_len, const int32_t *posts,
                                       const int32_t *present, const int64_t *pcm_off, void *pcm, int pcm_s16,
                                       int64_t pcm_stride, vb200_decode_carry *carry) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  if (!Wseq || !coef_off || !res || !posts || !present || !pcm_off || !pcm || !carry || !carry->tail || !carry->W)
    return fail(VB200_EINVAL, "decode pointers");
  const int ch = c->setup.channels;
  const size_t nb = (size_t)nstreams * nblk;
  HostCarry k(c, nstreams, carry);
  int rc;
  if ((rc = blocks_check(c, nstreams, nblk, count, Wseq, nullptr, nullptr, 0, nullptr, 0))) return rc;
  if ((rc = k.check())) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  HostIO io{c};
  const int32_t *dW = io.in(Wseq, nb);
  const int64_t *dco = io.in(coef_off, nb);
  float *dc = io.in(res, (size_t)res_len);
  const int64_t *dpo = io.in(pcm_off, nb);
  const size_t pbytes = (pcm_s16 ? sizeof(int16_t) : sizeof(float)) * (size_t)nstreams * ch * (size_t)pcm_stride;
  void *dp = io.out<void>(pbytes);
  const int32_t *dps = io.in(posts, nb * ch * VB200_FLOOR1_STRIDE), *dpr = io.in(present, nb * ch);
  const int32_t *dn = count ? io.in(count, nstreams) : nullptr;
  k.stage(io);
  if (io.rc) return io.rc;
  CU(cudaMemsetAsync(dp, 0, pbytes, c->s_main));
  if ((rc = vb200_decode_dsp_resume_dev(c, nstreams, nblk, dn, dW, dco, dc, dps, dpr, dpo, dp, pcm_s16, pcm_stride,
                                        &k.d, c->s_main))) return rc;
  io.back(pcm, dp, pbytes);
  k.write_back(io);
  return io.sync();
}

// ---- decode: the entropy half of mapping0_inverse on the device (vb200_entropy.cuh)
static const int ENT_FIRST_BITS = 10, ENT_SUB_BITS = 8;
static const size_t ENT_SMEM_MAX = 160 * 1024;

static int ilog_u(unsigned v) { int r = 0; while (v) { r++; v >>= 1; } return r; }

// the table of codewords cws (of book b) past their first `consumed` bits, k bits wide, appended to tab; base:
// where the book's tables start.  False where two codewords claim one index or an index stays empty.
static bool ent_fill(const vb200_codebook &b, const std::vector<int> &cws, int consumed, int k, size_t base,
                     std::vector<uint32_t> &tab) {
  const size_t at = tab.size();
  tab.resize(at + ((size_t)1 << k), 0u);
  std::vector<std::vector<int>> sub((size_t)1 << k);
  for (int i : cws) {
    const int len = b.length[i] - consumed;
    const uint32_t bits = b.bits[i] >> consumed;
    if (len <= k) {
      for (uint32_t j = 0; j < (1u << (k - len)); j++) {
        const size_t slot = at + ((bits & ((1u << len) - 1)) | (j << len));
        if (tab[slot]) return false;
        tab[slot] = ((uint32_t)i << 6) | (uint32_t)b.length[i];
      }
    } else {
      sub[bits & ((1u << k) - 1)].push_back(i);
    }
  }
  for (size_t v = 0; v < sub.size(); v++) {
    if (sub[v].empty()) continue;
    if (tab[at + v]) return false;
    int longest = 0;
    for (int i : sub[v]) longest = std::max(longest, b.length[i] - consumed - k);
    const int sk = std::min(longest, ENT_SUB_BITS);
    const size_t off = tab.size() - base;
    if (off >= ((size_t)1 << 26)) return false;
    tab[at + v] = 0x80000000u | ((uint32_t)off << 5) | (uint32_t)sk;
    if (!ent_fill(b, sub[v], consumed + k, sk, base, tab)) return false;
  }
  for (size_t v = 0; v < sub.size(); v++) if (!tab[at + v]) return false;
  return true;
}

static int ent_book(const vb200_codebook &b, EntBook &d, std::vector<uint32_t> &tab, std::vector<float> &vec,
                    std::vector<int> &ent) {
  memset(&d, 0, sizeof(d));
  if (b.dim < 1 || b.dim > 127 || b.used < 0 || b.used >= (1 << 24)) return fail(VB200_EINVAL, "codebook dim / used");
  d.dim = b.dim; d.used = b.used;
  if (b.used == 0) return 0;
  if (!b.length || !b.bits || !b.entry) return fail(VB200_EINVAL, "codebook arrays");
  unsigned long long kraft = 0;
  int longest = 0;
  for (int i = 0; i < b.used; i++) {
    const int len = b.length[i];
    if (len < 1 || len > 32 || (len < 32 && (b.bits[i] >> len)) || b.entry[i] < 0)
      return fail(VB200_EINVAL, "codeword length / bits / entry");
    kraft += 1ull << (32 - len);
    longest = std::max(longest, len);
  }
  d.tab_off = (int)tab.size(); d.ent_off = (int)ent.size(); d.vec_off = (int)vec.size();
  if (tab.size() > (1u << 30) || vec.size() + (size_t)b.used * b.dim > (1u << 30)) return fail(VB200_EINVAL, "codebooks too large");
  if (b.used == 1 && b.length[0] == 1) {          // the single-entry book reads one bit whatever its value
    d.k = 1;
    tab.push_back(1u); tab.push_back(1u);
  } else {
    if (kraft != (1ull << 32)) return fail(VB200_EINVAL, "codebook is not a complete prefix code");
    std::vector<int> all(b.used);
    for (int i = 0; i < b.used; i++) all[i] = i;
    d.k = std::min(longest, ENT_FIRST_BITS);
    if (!ent_fill(b, all, 0, d.k, tab.size(), tab)) return fail(VB200_EINVAL, "codebook is not a prefix code");
  }
  for (int i = 0; i < b.used; i++) ent.push_back(b.entry[i]);
  if (b.value) vec.insert(vec.end(), b.value, b.value + (size_t)b.used * b.dim);
  else d.vec_off = -1;
  return 0;
}

// the channels of submap sm in block size w (*bundle) and the samples its residue spans: n, or for type 2 the
// bundle's n lines interleaved
static long res_limit(const vb200_setup &S, int w, int sm, int type, int *bundle) {
  const long n = S.blocksizes[w] / 2;
  *bundle = 0;
  for (int k = 0; k < S.channels; k++) *bundle += S.chmux[w][k] == sm;
  return type == 2 ? *bundle * n : n;
}

// The floor and residue tables of both entropy coders: es->floor / es->residue of every submap of both block sizes
// checked against the context setup and the books' dims, into hf / hr (residue type -1 past a size's submaps).
// verb ("decode" / "encode") names the coder in the VB200_EIMPL messages.  EntRes::partvals is left to the caller.
template <class ES>
static int ent_tables(const vb200_setup &S, const ES *es, const char *verb, EntFloor (&hf)[2][VB200_MAX_SUBMAPS],
                      EntRes (&hr)[2][VB200_MAX_SUBMAPS]) {
  const int nb = es->nbooks;
  auto book_ok = [&](int b) { return b >= 0 && b < nb; };
  memset(hf, 0, sizeof(hf));
  memset(hr, 0, sizeof(hr));
  for (int w = 0; w < 2; w++) {
    const int subs = S.submaps[w];
    if (subs < 1) return fail(VB200_EINVAL, "no submaps in the context setup");
    for (int k = 0; k < S.channels; k++)
      if (S.chmux[w][k] >= subs) return fail(VB200_EINVAL, "chmux past submaps");
    for (int sm = 0; sm < VB200_MAX_SUBMAPS; sm++) hr[w][sm].type = -1;
    for (int sm = 0; sm < subs; sm++) {
      const vb200_floor_decode &f = es->floor[w][sm];
      const vb200_floor1_setup &f1 = S.floor1[w][sm];
      EntFloor &F = hf[w][sm];
      if (f.type != 1) return fail(VB200_EIMPL, (std::string("only floor type 1 ") + verb + "s on the device").c_str());
      if (f1.posts <= 0) return fail(VB200_EINVAL, "no floor1 setup for a submap");
      if (f.partitions < 0 || f.partitions > 31) return fail(VB200_EINVAL, "floor partitions");
      int posts = 2;
      for (int i = 0; i < f.partitions; i++) {
        const int cl = f.partitionclass[i];
        if (cl < 0 || cl > 15) return fail(VB200_EINVAL, "floor partition class");
        if (f.class_dim[cl] < 1 || f.class_dim[cl] > 8 || f.class_subs[cl] < 0 || f.class_subs[cl] > 3)
          return fail(VB200_EINVAL, "floor class dim / subs");
        posts += f.class_dim[cl];
      }
      if (posts != f1.posts) return fail(VB200_EINVAL, "floor partitions do not give the floor's posts");
      static const int quant_q[4] = {256, 128, 86, 64};
      F.partitions = f.partitions; F.posts = f1.posts;
      F.quant_q = quant_q[f1.mult - 1]; F.qbits = ilog_u((unsigned)F.quant_q - 1);
      for (int cl = 0; cl < 16; cl++) for (int j = 0; j < 8; j++) F.subbook[cl][j] = -1;
      for (int i = 0; i < f.partitions; i++) {
        const int cl = f.partitionclass[i];
        F.pclass[i] = (unsigned char)cl;
        F.cdim[cl] = (unsigned char)f.class_dim[cl]; F.csubs[cl] = (unsigned char)f.class_subs[cl];
        if (f.class_subs[cl] && !book_ok(f.class_book[cl])) return fail(VB200_EINVAL, "floor class book");
        F.cbook[cl] = (short)(f.class_subs[cl] ? f.class_book[cl] : 0);
        for (int j = 0; j < (1 << f.class_subs[cl]); j++) {
          const int b = f.class_subbook[cl][j];
          if (b != -1 && !book_ok(b)) return fail(VB200_EINVAL, "floor subclass book");
          F.subbook[cl][j] = (short)b;
        }
      }
      const vb200_residue_decode &r = es->residue[w][sm];
      EntRes &R = hr[w][sm];
      if (r.type == 0)
        return fail(VB200_EIMPL, (std::string("residue type 0 does not ") + verb + " on the device").c_str());
      if (r.type != 1 && r.type != 2) return fail(VB200_EINVAL, "residue type");
      int bundle;
      if (r.grouping < 1 || r.begin < 0 || r.end < r.begin || r.begin > res_limit(S, w, sm, r.type, &bundle))
        return fail(VB200_EINVAL, "residue begin / end / grouping do not fit the block");
      if (r.partitions < 1 || r.partitions > 64 || !book_ok(r.groupbook)) return fail(VB200_EINVAL, "residue partitions / groupbook");
      const int ppw = es->books[r.groupbook].dim;
      long long pv = 1;
      for (int j = 0; j < ppw && pv <= (1ll << 31); j++) pv *= r.partitions;
      if (pv != r.partvals) return fail(VB200_EINVAL, "residue partvals != partitions ^ dim(groupbook)");
      R.type = r.type; R.begin = r.begin; R.end = r.end; R.grouping = r.grouping;
      R.groupbook = r.groupbook; R.ppw = ppw; R.partitions = r.partitions; R.stages = 0;
      for (int cl = 0; cl < 64; cl++)
        for (int st = 0; st < 8; st++) {
          const int b = cl < r.partitions ? r.stagebook[cl][st] : -1;
          if (b != -1 && !book_ok(b)) return fail(VB200_EINVAL, "residue stage book");
          R.stagebook[cl][st] = (short)b;
          if (b >= 0) R.stages = std::max(R.stages, st + 1);
        }
    }
  }
  return 0;
}

// Frees the registered tables of `owned` once no kernel may still read them: the context's stream, then the device
// (the _dev forms run on the caller's streams).  With c->mu held.
static int release_tables(vb200_ctx *c, std::vector<void *> &owned) {
  CU(cudaStreamSynchronize(c->s_main));
  CU(cudaDeviceSynchronize());
  for (void *p : owned) cudaFree(p);
  owned.clear();
  return 0;
}

extern "C" int vb200_decode_entropy_setup(vb200_ctx *c, const vb200_entropy_setup *es) {
  CHECK_CTX(c);
  if (!es || es->nbooks < 0 || (es->nbooks > 0 && !es->books)) return fail(VB200_EINVAL, "entropy setup");
  if (es->modebits < 0 || es->modebits > 8) return fail(VB200_EINVAL, "modebits");
  const vb200_setup &S = c->setup;
  const int nb = es->nbooks, ch = S.channels;
  std::vector<EntBook> books(nb > 0 ? nb : 1);
  std::vector<uint32_t> tab;
  std::vector<float> vec;
  std::vector<int> ent;
  int rc;
  for (int i = 0; i < nb; i++)
    if ((rc = ent_book(es->books[i], books[i], tab, vec, ent))) return rc;
  EntFloor hf[2][VB200_MAX_SUBMAPS];
  EntRes hr[2][VB200_MAX_SUBMAPS];
  if ((rc = ent_tables(S, es, "decode", hf, hr))) return rc;
  size_t cls_cap = 1;
  for (int w = 0; w < 2; w++)
    for (int sm = 0; sm < S.submaps[w]; sm++) {
      EntRes &R = hr[w][sm];
      R.partvals = es->residue[w][sm].partvals;
      for (int cl = 0; cl < R.partitions; cl++)
        for (int st = 0; st < R.stages; st++) {
          const int b = R.stagebook[cl][st];
          if (b >= 0 && es->books[b].used > 0 && !es->books[b].value)
            return fail(VB200_EINVAL, "residue stage book without values");
        }
      int bundle;
      const long end = std::min((long)R.end, res_limit(S, w, sm, R.type, &bundle));
      cls_cap = std::max(cls_cap, (size_t)((end - R.begin) / R.grouping) * (R.type == 2 ? 1 : bundle));
    }
  const size_t smem = sizeof(int32_t) * (size_t)ch * (VB200_FLOOR1_STRIDE + 1) + 2 * (size_t)ch + cls_cap;
  if (smem > ENT_SMEM_MAX) return fail(VB200_EIMPL, "partition classes of a block exceed the shared memory");
  std::lock_guard<std::mutex> lk(c->mu);
  if ((rc = release_tables(c, c->ent_owned))) return rc;
  c->ent = EntDev{};
  EntDev E{};
  if ((rc = upload(c->ent_owned, books.data(), books.size(), &E.books))) return rc;
  if ((rc = upload(c->ent_owned, tab.data(), tab.size(), &E.tab))) return rc;
  if ((rc = upload(c->ent_owned, vec.data(), vec.size(), &E.vec))) return rc;
  if ((rc = upload(c->ent_owned, ent.data(), ent.size(), &E.ent))) return rc;
  for (int w = 0; w < 2; w++) {
    if ((rc = upload(c->ent_owned, hf[w], (size_t)VB200_MAX_SUBMAPS, &E.floor[w]))) return rc;
    if ((rc = upload(c->ent_owned, hr[w], (size_t)VB200_MAX_SUBMAPS, &E.res[w]))) return rc;
    E.chmux[w] = c->d_chmux[w]; E.mag[w] = c->d_mag[w]; E.ang[w] = c->d_ang[w];
    E.steps[w] = S.coupling_steps[w]; E.submaps[w] = S.submaps[w]; E.n[w] = S.blocksizes[w] / 2;
  }
  E.ch = ch; E.modebits = es->modebits; E.cls_cap = (int)cls_cap;
  c->ent = E;
  return 0;
}

extern "C" int vb200_decode_entropy_dev(vb200_ctx *c, int nblocks, const int32_t *d_Wseq, const int64_t *d_pkt_off,
                                        const int32_t *d_pkt_bytes, const uint8_t *d_data, const int64_t *d_coef_off,
                                        float *d_res, int32_t *d_posts, int32_t *d_present, void *stream) {
  CHECK_CTX(c);
  if (nblocks <= 0) return 0;
  if (!d_Wseq || !d_pkt_off || !d_pkt_bytes || !d_data || !d_coef_off || !d_res || !d_posts || !d_present)
    return fail(VB200_EINVAL, "decode_entropy pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  const size_t smem = entropy_smem(c->ent, false);
  if ((rc = set_smem(k_decode_entropy, smem))) return rc;
  const DecodePackets P{(const long long *)d_pkt_off, d_pkt_bytes, d_data};
  k_decode_entropy<<<grid_for(c, nblocks, 16), 32, smem, (cudaStream_t)stream>>>(
      c->ent, c->d_floor[0], c->d_floor[1], P, nblocks, d_Wseq, (const long long *)d_coef_off, d_res, d_posts,
      d_present);
  return post_launch(c);
}

extern "C" int vb200_decode_entropy(vb200_ctx *c, int nblocks, const int32_t *Wseq, const int64_t *pkt_off,
                                    const int32_t *pkt_bytes, const uint8_t *data, int64_t data_bytes,
                                    const int64_t *coef_off, float *res, int64_t res_len, int32_t *posts,
                                    int32_t *present) {
  CHECK_CTX(c);
  if (nblocks <= 0) return 0;
  if (!Wseq || !pkt_off || !pkt_bytes || !data || !coef_off || !res || !posts || !present || data_bytes < 0)
    return fail(VB200_EINVAL, "decode_entropy pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  if ((rc = blocks_check(c, 1, nblocks, nullptr, Wseq, pkt_off, pkt_bytes, data_bytes, coef_off, res_len))) return rc;
  const int ch = c->setup.channels;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t nb = (size_t)nblocks;
  HostIO io{c};
  const int32_t *dW = io.in(Wseq, nb);
  const int64_t *dpo = io.in(pkt_off, nb);
  const int32_t *dpb = io.in(pkt_bytes, nb);
  const uint8_t *dd = io.packets(data, data_bytes);
  const int64_t *dco = io.in(coef_off, nb);
  float *dr = io.in(res, (size_t)res_len);
  int32_t *dps = io.out<int32_t>(nb * ch * VB200_FLOOR1_STRIDE), *dpr = io.out<int32_t>(nb * ch);
  if (io.rc) return io.rc;
  if ((rc = vb200_decode_entropy_dev(c, nblocks, dW, dpo, dpb, dd, dco, dr, dps, dpr, c->s_main))) return rc;
  io.back(res, dr, (size_t)res_len);
  io.back(posts, dps, nb * ch * VB200_FLOOR1_STRIDE);
  io.back(present, dpr, nb * ch);
  return io.sync();
}

extern "C" int vb200_decode_packets_resume_dev(vb200_ctx *c, int nstreams, int nblk, const int32_t *d_count,
                                               const int32_t *d_Wseq, const int64_t *d_coef_off, float *d_res,
                                               const int64_t *d_pkt_off, const int32_t *d_pkt_bytes,
                                               const uint8_t *d_data, const int64_t *d_pcm_off, void *d_pcm,
                                               int pcm_s16, int64_t pcm_stride, const vb200_decode_carry *d_carry,
                                               void *stream) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  if (!d_Wseq || !d_coef_off || !d_res || !d_pkt_off || !d_pkt_bytes || !d_data || !d_pcm_off || !d_pcm || !d_carry ||
      !d_carry->tail || !d_carry->W)
    return fail(VB200_EINVAL, "decode pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  const DecodePackets P{(const long long *)d_pkt_off, d_pkt_bytes, d_data};
  if ((rc = decode_front(c, nstreams, nblk, d_count, d_Wseq, d_coef_off, d_res, nullptr, nullptr, &P, st))) return rc;
  return synthesis_launch<SYN_CARRY>(c, pcm_s16, nstreams, nblk, d_count, d_Wseq, d_coef_off, d_res, d_pcm_off, d_pcm,
                                     pcm_stride, d_carry, DsTrim{}, st);
}

extern "C" int vb200_decode_packets_resume(vb200_ctx *c, int nstreams, int nblk, const int32_t *count,
                                           const int32_t *Wseq, const int64_t *coef_off, int64_t res_len,
                                           const int64_t *pkt_off, const int32_t *pkt_bytes, const uint8_t *data,
                                           int64_t data_bytes, const int64_t *pcm_off, void *pcm, int pcm_s16,
                                           int64_t pcm_stride, vb200_decode_carry *carry) {
  CHECK_CTX(c);
  if (nstreams <= 0 || nblk <= 0) return 0;
  if (!Wseq || !coef_off || !pkt_off || !pkt_bytes || !data || !pcm_off || !pcm || !carry || !carry->tail ||
      !carry->W || data_bytes < 0 || res_len < 0)
    return fail(VB200_EINVAL, "decode pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  const int ch = c->setup.channels;
  const size_t nb = (size_t)nstreams * nblk;
  HostCarry k(c, nstreams, carry);
  if ((rc = blocks_check(c, nstreams, nblk, count, Wseq, pkt_off, pkt_bytes, data_bytes, coef_off, res_len))) return rc;
  if ((rc = k.check())) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  HostIO io{c};
  const int32_t *dW = io.in(Wseq, nb);
  const int64_t *dco = io.in(coef_off, nb);
  float *dc = io.out<float>((size_t)(res_len ? res_len : 1));
  const int64_t *dpo = io.in(pcm_off, nb);
  const size_t pbytes = (pcm_s16 ? sizeof(int16_t) : sizeof(float)) * (size_t)nstreams * ch * (size_t)pcm_stride;
  void *dp = io.out<void>(pbytes);
  const int64_t *dko = io.in(pkt_off, nb);
  const int32_t *dkb = io.in(pkt_bytes, nb);
  const uint8_t *dd = io.packets(data, data_bytes);
  const int32_t *dn = count ? io.in(count, nstreams) : nullptr;
  k.stage(io);
  if (io.rc) return io.rc;
  CU(cudaMemsetAsync(dp, 0, pbytes, c->s_main));
  if ((rc = vb200_decode_packets_resume_dev(c, nstreams, nblk, dn, dW, dco, dc, dko, dkb, dd, dpo, dp, pcm_s16,
                                            pcm_stride, &k.d, c->s_main))) return rc;
  io.back(pcm, dp, pbytes);
  k.write_back(io);
  return io.sync();
}

// ---- whole streams from packets (vb200_decode_streams.cuh): header parse, per-stream plan, prefix scan, then the
// fused entropy decode and the trimming synthesis on the plan's tables.  A stream's carry is a DsHead, then the
// overlap tail of each channel.
static size_t ds_carry_bytes(const vb200_ctx *c) {
  return DS_HEAD_BYTES + sizeof(float) * (size_t)c->setup.channels * (c->setup.blocksizes[1] / 2);
}

extern "C" int vb200_decode_streams_carry_bytes(vb200_ctx *c) {
  if (!c) return fail(VB200_EINVAL, "null context");
  return (int)ds_carry_bytes(c);
}

extern "C" int vb200_decode_streams_carry_init(vb200_ctx *c, int nstreams, void *d_carry) {
  CHECK_CTX(c);
  if (nstreams <= 0) return 0;
  if (!d_carry) return fail(VB200_EINVAL, "null carry");
  DsHead h{};
  h.granulepos = -1; h.sample_count = -1; h.sequence = -1; h.W = -1;
  h.rate = c->halfrate ? DS_RATE_HALF : DS_RATE_FULL;
  const size_t B = ds_carry_bytes(c);
  std::vector<DsHead> heads((size_t)nstreams, h);
  CU(cudaMemcpy2DAsync(d_carry, B, heads.data(), sizeof(DsHead), sizeof(DsHead), (size_t)nstreams,
                       cudaMemcpyHostToDevice, c->s_main));
  CU(cudaStreamSynchronize(c->s_main));
  return 0;
}

// the plan front of vb200_decode_streams_packets_dev and vb200_decode_streams_index_dev: the plan's tables carved
// from arena, then own(k) carves the caller's scratch (and P.pcm_base where the caller has none); then k_ds_header
// and k_ds_plan on st.  The heads are d_carry's, ds_carry_bytes apart, or without d_carry fresh ones carved here.
template <class Own>
static int ds_plan_front(vb200_ctx *c, DevBuf &arena, DsPlanArgs &P, int nstreams, int max_packets,
                         const int32_t *d_npkt, const vb200_packet_info *d_info, const uint8_t *d_data,
                         const void *d_carry, vb200_decoded_packet *d_out, cudaStream_t st, Own &&own) {
  const long long n = (long long)nstreams * max_packets;
  DsHead *fresh = nullptr;
  int rc;
  if ((rc = carve(arena, [&](Carve &k) {
         P.Wseq = k.take<int>(n); P.pkt_bytes = k.take<int>(n); P.pkt_off = k.take<long long>(n);
         P.coef_off = k.take<long long>(n); P.pcm_off = k.take<long long>(n); P.win = k.take<int2>(n);
         P.count = k.take<int>(nstreams); P.W_in = k.take<int>(nstreams); P.head = k.take<DsHead>(nstreams);
         own(k);
         if (!d_carry) fresh = k.take<DsHead>(nstreams);
       }))) return rc;
  int *hdr = P.Wseq;                     // k_ds_plan reads slot k's header before it writes block j <= k there
  P.nstreams = nstreams; P.max_packets = max_packets; P.ch = c->setup.channels; P.hs = c->halfrate ? 1 : 0;
  P.bs[0] = c->setup.blocksizes[0]; P.bs[1] = c->setup.blocksizes[1];
  P.npkt = d_npkt; P.info = d_info; P.hdr = hdr; P.out = d_out;
  // vorbis_synthesis_restart's head has every field k_ds_plan reads at -1 (granulepos, sample_count, sequence, W);
  // rate is not read there
  P.carry = d_carry ? (const unsigned char *)d_carry : (const unsigned char *)fresh;
  P.carry_bytes = d_carry ? (long long)ds_carry_bytes(c) : (long long)sizeof(DsHead);
  if ((rc = scratch_begin(c, st))) return rc;
  if (!d_carry) CU(cudaMemsetAsync(fresh, 0xff, sizeof(DsHead) * (size_t)nstreams, st));
  k_ds_header<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(nstreams, max_packets, c->ent.modebits, d_npkt, d_info,
                                                             d_data, hdr);
  if ((rc = post_launch(c))) return rc;
  k_ds_plan<<<(nstreams + 127) / 128, 128, 0, st>>>(P);
  return post_launch(c);
}

extern "C" int vb200_decode_streams_packets_dev(vb200_ctx *c, int nstreams, int max_packets, const int32_t *d_npkt,
                                                const vb200_packet_info *d_info, const uint8_t *d_data, void *d_carry,
                                                int pcm_s16, void *d_pcm, int64_t pcm_cap, int64_t *d_pcm_base,
                                                vb200_decoded_packet *d_out, void *stream) {
  CHECK_CTX(c);
  if (nstreams <= 0) return 0;
  if (max_packets < 1) return fail(VB200_EINVAL, "max_packets must be >= 1");
  if (!d_npkt || !d_info || !d_data || !d_carry || !d_pcm || !d_pcm_base || !d_out)
    return fail(VB200_EINVAL, "decode streams pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  const long long n = (long long)nstreams * max_packets;
  if (n > INT32_MAX) return fail(VB200_EINVAL, "nstreams * max_packets must fit an int");
  const int ch = c->setup.channels;
  const cudaStream_t st = (cudaStream_t)stream;
  DsPlanArgs P;
  float *res;
  P.pcm_base = (long long *)d_pcm_base;
  if ((rc = ds_plan_front(c, c->dsk, P, nstreams, max_packets, d_npkt, d_info, d_data, d_carry, d_out, st,
                          [&](Carve &k) { res = k.take<float>(n * ch * (c->setup.blocksizes[1] / 2)); })))
    return rc;
  k_ds_scan<<<1, 1024, 0, st>>>(nstreams, P.pcm_base);
  if ((rc = post_launch(c))) return rc;
  const DecodePackets DP{P.pkt_off, P.pkt_bytes, d_data};
  if ((rc = decode_front(c, nstreams, max_packets, P.count, P.Wseq, (const int64_t *)P.coef_off, res, nullptr, nullptr,
                         &DP, st))) return rc;
  DsTrim T;
  T.win = P.win; T.base = P.pcm_base; T.W_in = P.W_in; T.head = P.head; T.carry = (unsigned char *)d_carry;
  T.carry_bytes = P.carry_bytes; T.cap = pcm_cap; T.tail_stride = c->setup.blocksizes[1] / 2;
  if ((rc = synthesis_launch<SYN_TRIM>(c, pcm_s16, nstreams, max_packets, P.count, P.Wseq, (const int64_t *)P.coef_off,
                                       res, (const int64_t *)P.pcm_off, d_pcm, 0, nullptr, T, st))) return rc;
  return scratch_end(c, st);
}

// host-form checks of the packet-stream forms: npkt[s] in [0, max_packets], every counted packet inside data
static int ds_check_packets(int nstreams, int max_packets, const int32_t *npkt, const vb200_packet_info *info,
                            int64_t data_bytes) {
  for (int s = 0; s < nstreams; s++) {
    if (npkt[s] < 0 || npkt[s] > max_packets) return fail(VB200_EINVAL, "npkt[s] must be in [0, max_packets]");
    for (int k = 0; k < npkt[s]; k++) {
      const vb200_packet_info &p = info[(size_t)s * max_packets + k];
      if (p.offset < 0 || p.bytes < 0 || p.offset > data_bytes - p.bytes) return fail(VB200_EINVAL, "packet outside data");
    }
  }
  return 0;
}

extern "C" int vb200_decode_streams_packets(vb200_ctx *c, int nstreams, int max_packets, const int32_t *npkt,
                                            const vb200_packet_info *info, const uint8_t *data, int64_t data_bytes,
                                            void *d_carry, int pcm_s16, void *pcm, int64_t pcm_cap, int64_t *pcm_base,
                                            vb200_decoded_packet *out) {
  CHECK_CTX(c);
  if (nstreams <= 0) return 0;
  if (max_packets < 1) return fail(VB200_EINVAL, "max_packets must be >= 1");
  if (!npkt || !info || !data || !d_carry || !pcm || !pcm_base || !out || data_bytes < 0 || pcm_cap < 0)
    return fail(VB200_EINVAL, "decode streams pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  if ((rc = ds_check_packets(nstreams, max_packets, npkt, info, data_bytes))) return rc;
  const size_t n = (size_t)nstreams * max_packets;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t B = ds_carry_bytes(c);
  std::vector<DsHead> heads((size_t)nstreams);
  CU(cudaMemcpy2DAsync(heads.data(), sizeof(DsHead), d_carry, B, sizeof(DsHead), (size_t)nstreams,
                       cudaMemcpyDeviceToHost, c->s_main));
  CU(cudaStreamSynchronize(c->s_main));
  const int rate = c->halfrate ? DS_RATE_HALF : DS_RATE_FULL;
  for (const DsHead &h : heads)
    if (h.rate != rate || h.W < -1 || h.W > 1)
      return fail(VB200_EINVAL, "carry not initialised for this context's rate mode (vb200_decode_streams_carry_init)");
  const int ch = c->setup.channels;
  const size_t el = pcm_s16 ? sizeof(int16_t) : sizeof(float);
  HostIO io{c};
  const int32_t *dn = io.in(npkt, nstreams);
  const vb200_packet_info *di = io.in(info, n);
  const uint8_t *dd = io.packets(data, data_bytes);
  void *dp = io.out<void>(el * (size_t)std::max<int64_t>(pcm_cap, 1));
  int64_t *db = io.out<int64_t>(nstreams + 1);
  vb200_decoded_packet *dout = io.out<vb200_decoded_packet>(n);
  if (io.rc) return io.rc;
  if ((rc = vb200_decode_streams_packets_dev(c, nstreams, max_packets, dn, di, dd, d_carry, pcm_s16, dp, pcm_cap, db,
                                             dout, c->s_main)))
    return rc;
  io.back(pcm_base, db, nstreams + 1);
  io.back(out, dout, n);
  if ((rc = io.sync())) return rc;
  const int64_t total = pcm_base[nstreams] * ch;
  if (total > pcm_cap) return fail(VB200_EINVAL, "the PCM does not fit pcm_cap (pcm_base is filled)");
  if (total) io.back(pcm, dp, el * (size_t)total);
  return io.sync();
}

// ---- sample ranges from packets (vb200_decode_ranges.cuh).  The index is k_ds_header and k_ds_plan on fresh
// heads; the ranges are k_dr_plan, k_decode_packets<true> and k_synthesis<*, *, SYN_RANGE>.
extern "C" int vb200_decode_streams_index_dev(vb200_ctx *c, int nstreams, int max_packets, const int32_t *d_npkt,
                                              const vb200_packet_info *d_info, const uint8_t *d_data,
                                              int64_t *d_length, vb200_decoded_packet *d_out, void *stream) {
  CHECK_CTX(c);
  if (nstreams <= 0) return 0;
  if (max_packets < 1) return fail(VB200_EINVAL, "max_packets must be >= 1");
  if (!d_npkt || !d_info || !d_data || !d_length || !d_out) return fail(VB200_EINVAL, "decode streams index pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  if ((long long)nstreams * max_packets > INT32_MAX) return fail(VB200_EINVAL, "nstreams * max_packets must fit an int");
  const cudaStream_t st = (cudaStream_t)stream;
  DsPlanArgs P;
  if ((rc = ds_plan_front(c, c->drg, P, nstreams, max_packets, d_npkt, d_info, d_data, nullptr, d_out, st,
                          [&](Carve &k) { P.pcm_base = k.take<long long>(nstreams + 1); })))
    return rc;
  CU(cudaMemcpyAsync(d_length, P.pcm_base + 1, sizeof(int64_t) * (size_t)nstreams, cudaMemcpyDeviceToDevice, st));
  return scratch_end(c, st);
}

extern "C" int vb200_decode_streams_index(vb200_ctx *c, int nstreams, int max_packets, const int32_t *npkt,
                                          const vb200_packet_info *info, const uint8_t *data, int64_t data_bytes,
                                          int64_t *length, vb200_decoded_packet *out) {
  CHECK_CTX(c);
  if (nstreams <= 0) return 0;
  if (max_packets < 1) return fail(VB200_EINVAL, "max_packets must be >= 1");
  if (!npkt || !info || !data || !length || !out || data_bytes < 0) return fail(VB200_EINVAL, "decode streams index pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  if ((rc = ds_check_packets(nstreams, max_packets, npkt, info, data_bytes))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = (size_t)nstreams * max_packets;
  HostIO io{c};
  const int32_t *dn = io.in(npkt, nstreams);
  const vb200_packet_info *di = io.in(info, n);
  const uint8_t *dd = io.packets(data, data_bytes);
  int64_t *dl = io.out<int64_t>(nstreams);
  vb200_decoded_packet *dout = io.out<vb200_decoded_packet>(n);
  if (io.rc) return io.rc;
  if ((rc = vb200_decode_streams_index_dev(c, nstreams, max_packets, dn, di, dd, dl, dout, c->s_main))) return rc;
  io.back(length, dl, nstreams);
  io.back(out, dout, n);
  return io.sync();
}

// a request's block slots and residue floats (vb200_decode_ranges.cuh proves they hold every ordinary range); the
// residue is rounded up to 64 floats so that every request's region, and so every block in it, is 16-byte aligned
static long long dr_blocks(const vb200_ctx *c, int32_t out_stride) {
  return ((long long)out_stride << (c->halfrate ? 1 : 0)) / (c->setup.blocksizes[0] / 2) + 3;
}
static long long dr_residue(const vb200_ctx *c, int32_t out_stride) {
  const long long f = (long long)c->setup.channels *
                      (2 * ((long long)out_stride << (c->halfrate ? 1 : 0)) + 3ll * (c->setup.blocksizes[1] / 2));
  return (f + 63) & ~63ll;
}

extern "C" int vb200_decode_ranges_dev(vb200_ctx *c, int nstreams, int max_packets, const int32_t *d_npkt,
                                       const vb200_packet_info *d_info, const uint8_t *d_data,
                                       int nreq, const vb200_pcm_range *d_req, int pcm_s16, void *d_pcm,
                                       int32_t out_stride, int32_t *d_got, void *stream) {
  CHECK_CTX(c);
  if (nreq < 0) return fail(VB200_EINVAL, "nreq must be >= 0");
  if (nreq == 0) return 0;
  if (max_packets < 1) return fail(VB200_EINVAL, "max_packets must be >= 1");
  if (out_stride < 0) return fail(VB200_EINVAL, "out_stride must be >= 0");
  if (nstreams < 0 || (nstreams > 0 && (!d_npkt || !d_info || !d_data)) || !d_req || !d_pcm || !d_got)
    return fail(VB200_EINVAL, "decode ranges pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  const long long nblk = dr_blocks(c, out_stride), rescap = dr_residue(c, out_stride);
  if ((long long)nreq * nblk > INT32_MAX) return fail(VB200_EINVAL, "nreq * block slots must fit an int");
  const int ch = c->setup.channels;
  const bool hs = c->halfrate;
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t nb = (size_t)nreq * nblk;
  DrPlanArgs P;
  float *res;
  if ((rc = carve(c->drg, [&](Carve &k) {
         P.Wseq = k.take<int>(nb); P.pkt_bytes = k.take<int>(nb); P.pkt_off = k.take<long long>(nb);
         P.coef_off = k.take<long long>(nb); P.pcm_off = k.take<long long>(nb); P.win = k.take<int2>(nb);
         P.count = k.take<int>(nreq); P.base = k.take<long long>(nreq + 1);
         res = k.take<float>((size_t)nreq * rescap);
       }))) return rc;
  P.nstreams = nstreams; P.max_packets = max_packets; P.nreq = nreq; P.ch = ch; P.hs = hs ? 1 : 0;
  P.modebits = c->ent.modebits;
  P.bs[0] = c->setup.blocksizes[0]; P.bs[1] = c->setup.blocksizes[1];
  P.out_stride = out_stride; P.nblk = (int)nblk; P.res_cap = rescap;
  P.npkt = d_npkt; P.info = d_info; P.data = d_data; P.req = d_req; P.got = d_got;
  if ((rc = scratch_begin(c, st))) return rc;
  const size_t el = pcm_s16 ? sizeof(int16_t) : sizeof(float);
  CU(cudaMemsetAsync(d_pcm, 0, el * (size_t)nreq * ch * (size_t)out_stride, st));
  k_dr_plan<<<(unsigned)(((long long)nreq * 32 + 127) / 128), 128, 0, st>>>(P);
  if ((rc = post_launch(c))) return rc;
  const DecodePackets DP{P.pkt_off, P.pkt_bytes, d_data};
  if ((rc = decode_front(c, nreq, (int)nblk, P.count, P.Wseq, (const int64_t *)P.coef_off, res, nullptr, nullptr, &DP,
                         st))) return rc;
  DsTrim T{};
  T.win = P.win; T.base = P.base;
  if ((rc = synthesis_launch<SYN_RANGE>(c, pcm_s16, nreq, (int)nblk, P.count, P.Wseq, (const int64_t *)P.coef_off, res,
                                        (const int64_t *)P.pcm_off, d_pcm, 0, nullptr, T, st))) return rc;
  return scratch_end(c, st);
}

extern "C" int vb200_decode_ranges(vb200_ctx *c, int nstreams, int max_packets, const int32_t *npkt,
                                   const vb200_packet_info *info, const uint8_t *data, int64_t data_bytes,
                                   int nreq, const vb200_pcm_range *req, int pcm_s16, void *pcm, int32_t out_stride,
                                   int32_t *got) {
  CHECK_CTX(c);
  if (nreq < 0) return fail(VB200_EINVAL, "nreq must be >= 0");
  if (max_packets < 1) return fail(VB200_EINVAL, "max_packets must be >= 1");
  if (nstreams < 0 || !npkt || !info || !data || !req || !pcm || !got || data_bytes < 0 || out_stride < 0)
    return fail(VB200_EINVAL, "decode ranges pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  if ((rc = ds_check_packets(nstreams, max_packets, npkt, info, data_bytes))) return rc;
  for (int r = 0; r < nreq; r++)
    if (req[r].stream < 0 || req[r].stream >= nstreams || req[r].start < 0 || req[r].length < 0 ||
        req[r].length > out_stride)
      return fail(VB200_EINVAL, "a request's stream, start or length is out of range");
  if (nreq == 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = (size_t)nstreams * max_packets;      // nstreams >= 1: a request names a stream
  const size_t pbytes = (pcm_s16 ? sizeof(int16_t) : sizeof(float)) * (size_t)nreq * c->setup.channels * out_stride;
  HostIO io{c};
  const int32_t *dn = io.in(npkt, nstreams);
  const vb200_packet_info *di = io.in(info, n);
  const uint8_t *dd = io.packets(data, data_bytes);
  const vb200_pcm_range *dq = io.in(req, nreq);
  void *dp = io.out<void>(std::max<size_t>(pbytes, 1));
  int32_t *dg = io.out<int32_t>(nreq);
  if (io.rc) return io.rc;
  if ((rc = vb200_decode_ranges_dev(c, nstreams, max_packets, dn, di, dd, nreq, dq, pcm_s16, dp, out_stride, dg,
                                    c->s_main))) return rc;
  if (pbytes) io.back(pcm, dp, pbytes);
  io.back(got, dg, nreq);
  return io.sync();
}

// ---- sample ranges straight from Ogg files (vb200_ogg_ranges.cuh): k_or_plan in place of k_dr_plan, then the same
// k_decode_packets<true> and k_synthesis<*, *, SYN_RANGE> over the gathered packets
extern "C" int vb200_ogg_ranges_dev(vb200_ctx *c, int nrows, const uint8_t *d_bytes, const int64_t *d_row_off,
                                    int nreq, const vb200_pcm_range *d_req, int pcm_s16, void *d_pcm,
                                    int32_t out_stride, int64_t pkt_cap, int32_t *d_got, void *stream) {
  CHECK_CTX(c);
  if (nreq < 0) return fail(VB200_EINVAL, "nreq must be >= 0");
  if (nreq == 0) return 0;
  if (out_stride < 0) return fail(VB200_EINVAL, "out_stride must be >= 0");
  if (pkt_cap < 0) return fail(VB200_EINVAL, "pkt_cap must be >= 0");
  if (nrows < 0 || (nrows > 0 && (!d_bytes || !d_row_off)) || !d_req || !d_pcm || !d_got)
    return fail(VB200_EINVAL, "ogg ranges pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  const long long nblk = dr_blocks(c, out_stride), rescap = dr_residue(c, out_stride);
  if ((long long)nreq * nblk > INT32_MAX) return fail(VB200_EINVAL, "nreq * block slots must fit an int");
  const int ch = c->setup.channels;
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t nb = (size_t)nreq * nblk;
  OrPlanArgs P;
  float *res;
  if ((rc = carve(c->drg, [&](Carve &k) {
         P.Wseq = k.take<int>(nb); P.pkt_bytes = k.take<int>(nb); P.pkt_off = k.take<long long>(nb);
         P.coef_off = k.take<long long>(nb); P.pcm_off = k.take<long long>(nb); P.win = k.take<int2>(nb);
         P.count = k.take<int>(nreq); P.base = k.take<long long>(nreq + 1);
         res = k.take<float>((size_t)nreq * rescap);
         P.pkt = k.take<uint8_t>((size_t)nreq * pkt_cap + 1);
       }))) return rc;
  P.nrows = nrows; P.nreq = nreq; P.ch = ch; P.hs = c->halfrate ? 1 : 0;
  P.modebits = c->ent.modebits;
  P.bs[0] = c->setup.blocksizes[0]; P.bs[1] = c->setup.blocksizes[1];
  P.out_stride = out_stride; P.nblk = (int)nblk; P.res_cap = rescap; P.pkt_cap = pkt_cap;
  P.bytes = d_bytes; P.row_off = d_row_off; P.req = d_req; P.got = d_got;
  if ((rc = scratch_begin(c, st))) return rc;
  const size_t el = pcm_s16 ? sizeof(int16_t) : sizeof(float);
  CU(cudaMemsetAsync(d_pcm, 0, el * (size_t)nreq * ch * (size_t)out_stride, st));
  k_or_plan<<<(unsigned)((nreq + OR_WARPS - 1) / OR_WARPS), 32 * OR_WARPS, 0, st>>>(P);
  if ((rc = post_launch(c))) return rc;
  const DecodePackets DP{P.pkt_off, P.pkt_bytes, P.pkt};
  if ((rc = decode_front(c, nreq, (int)nblk, P.count, P.Wseq, (const int64_t *)P.coef_off, res, nullptr, nullptr, &DP,
                         st))) return rc;
  DsTrim T{};
  T.win = P.win; T.base = P.base;
  if ((rc = synthesis_launch<SYN_RANGE>(c, pcm_s16, nreq, (int)nblk, P.count, P.Wseq, (const int64_t *)P.coef_off, res,
                                        (const int64_t *)P.pcm_off, d_pcm, 0, nullptr, T, st))) return rc;
  return scratch_end(c, st);
}

extern "C" int vb200_ogg_ranges(vb200_ctx *c, int nrows, const uint8_t *bytes, const int64_t *row_off,
                                int nreq, const vb200_pcm_range *req, int pcm_s16, void *pcm, int32_t out_stride,
                                int64_t pkt_cap, int32_t *got) {
  CHECK_CTX(c);
  if (nreq < 0) return fail(VB200_EINVAL, "nreq must be >= 0");
  if (nrows < 0 || !row_off || !req || !pcm || !got || out_stride < 0 || pkt_cap < 0)
    return fail(VB200_EINVAL, "ogg ranges pointers");
  int rc;
  if ((rc = ent_check(c))) return rc;
  if (row_off[0] < 0) return fail(VB200_EINVAL, "ogg_ranges: row_off[0] < 0");
  for (int f = 0; f < nrows; f++)
    if (row_off[f + 1] < row_off[f]) return fail(VB200_EINVAL, "ogg_ranges: row_off decreases");
  const int64_t total = row_off[nrows];
  if (total && !bytes) return fail(VB200_EINVAL, "ogg ranges pointers");
  for (int r = 0; r < nreq; r++)
    if (req[r].stream < 0 || req[r].stream >= nrows || req[r].start < 0 || req[r].length < 0 ||
        req[r].length > out_stride)
      return fail(VB200_EINVAL, "a request's row, start or length is out of range");
  if (nreq == 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t pbytes = (pcm_s16 ? sizeof(int16_t) : sizeof(float)) * (size_t)nreq * c->setup.channels * out_stride;
  HostIO io{c};
  const uint8_t *db = io.packets(bytes, total);
  const int64_t *doff = io.in(row_off, (size_t)nrows + 1);
  const vb200_pcm_range *dq = io.in(req, nreq);
  void *dp = io.out<void>(std::max<size_t>(pbytes, 1));
  int32_t *dg = io.out<int32_t>(nreq);
  if (io.rc) return io.rc;
  if ((rc = vb200_ogg_ranges_dev(c, nrows, db, doff, nreq, dq, pcm_s16, dp, out_stride, pkt_cap, dg, c->s_main)))
    return rc;
  if (pbytes) io.back(pcm, dp, pbytes);
  io.back(got, dg, nreq);
  return io.sync();
}

// ======================================================================== //
// encode: the entropy coding of mapping0_forward on the device (vb200_entropy_enc.cuh)
static const size_t EENT_SMEM_MAX = 200 * 1024;

extern "C" int vb200_encode_entropy_setup(vb200_ctx *c, const struct vb200_encode_entropy_setup *es) {
  CHECK_CTX(c);
  if (!es || es->nbooks < 0 || (es->nbooks > 0 && !es->books)) return fail(VB200_EINVAL, "encode entropy setup");
  if (es->modebits < 0 || es->modebits > 8) return fail(VB200_EINVAL, "modebits");
  const vb200_setup &S = c->setup;
  const int nb = es->nbooks, ch = S.channels;
  std::vector<EncBook> books(nb > 0 ? nb : 1);
  std::vector<unsigned char> len;
  std::vector<uint32_t> cw;
  std::vector<int> longest(nb > 0 ? nb : 1, 0);
  for (int i = 0; i < nb; i++) {
    const vb200_enc_codebook &b = es->books[i];
    if (b.dim < 1 || b.entries < 0 || b.entries >= (1 << 24) || (b.entries > 0 && (!b.length || !b.codeword)))
      return fail(VB200_EINVAL, "codebook dim / entries / arrays");
    if (len.size() + (size_t)b.entries > (1u << 30)) return fail(VB200_EINVAL, "codebooks too large");
    books[i] = EncBook{b.dim, b.entries, b.minval, b.delta, b.quantvals, (int)len.size()};
    for (int e = 0; e < b.entries; e++) {
      if (b.length[e] > 32) return fail(VB200_EINVAL, "codeword longer than 32 bits");
      longest[i] = std::max(longest[i], (int)b.length[e]);
    }
    len.insert(len.end(), b.length, b.length + b.entries);
    cw.insert(cw.end(), b.codeword, b.codeword + b.entries);
  }
  EntFloor hf[2][VB200_MAX_SUBMAPS];
  EntRes hr[2][VB200_MAX_SUBMAPS];
  int rc;
  if ((rc = ent_tables(S, es, "encode", hf, hr))) return rc;
  int slots[2] = {0, 0}, bound[2] = {0, 0};
  for (int w = 0; w < 2; w++) {
    long long nslot = 1 + ch, bits = 1 + es->modebits + (w ? 2 : 0);
    for (int sm = 0; sm < S.submaps[w]; sm++) {
      const EntFloor &F = hf[w][sm];
      EntRes &R = hr[w][sm];
      const vb200_residue_setup &rs = S.residue[w][sm];
      int bundle;
      if (R.end > res_limit(S, w, sm, R.type, &bundle))
        return fail(VB200_EINVAL, "residue begin / end / grouping do not fit the block");
      if (rs.type != R.type || rs.begin != R.begin || rs.end != R.end || rs.grouping != R.grouping ||
          rs.partitions != R.partitions)
        return fail(VB200_EINVAL, "residue differs from the context's classification setup");
      R.partvals = (R.end - R.begin) / R.grouping;
      int stage_longest[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (int cl = 0; cl < R.partitions; cl++)
        for (int st = 0; st < R.stages; st++) {
          const int b = R.stagebook[cl][st];
          if (b < 0) continue;
          const vb200_enc_codebook &B = es->books[b];
          long long lattice = 1;
          for (int j = 0; j < B.dim && lattice <= B.entries; j++) lattice *= B.quantvals;
          if (B.dim > 8 || B.quantvals <= 0 || lattice > B.entries)
            return fail(VB200_EINVAL, "residue stage book: dim > 8 or a lattice that does not fit its entries");
          stage_longest[st] = std::max(stage_longest[st], (R.grouping / B.dim) * longest[b]);
        }
      long long fbits = 1 + 2 * F.qbits;
      for (int i = 0; i < F.partitions; i++) {
        const int cl = F.pclass[i];
        int sub_longest = 0;
        for (int j = 0; j < (1 << F.csubs[cl]); j++)
          if (F.subbook[cl][j] >= 0) sub_longest = std::max(sub_longest, longest[F.subbook[cl][j]]);
        fbits += (F.csubs[cl] ? longest[F.cbook[cl]] : 0) + (long long)F.cdim[cl] * sub_longest;
      }
      bits += bundle * fbits;
      const long long nvec = R.type == 2 ? 1 : bundle, groups = (R.partvals + R.ppw - 1) / R.ppw;
      nslot += groups * nvec + (long long)R.stages * R.partvals * nvec;
      bits += nvec * groups * longest[R.groupbook];
      for (int st = 0; st < R.stages; st++) bits += nvec * R.partvals * stage_longest[st];
    }
    if (sizeof(int) * (size_t)nslot > EENT_SMEM_MAX) return fail(VB200_EIMPL, "pieces of one packet exceed the shared memory");
    if (bits >= (1ll << 31) - 64) return fail(VB200_EIMPL, "packet bound exceeds 2^31 bits");
    slots[w] = (int)nslot;
    bound[w] = (int)(((bits + 7) / 8 + 3) & ~3ll);
  }
  std::lock_guard<std::mutex> lk(c->mu);
  if ((rc = release_tables(c, c->eent_owned))) return rc;
  c->eent = EncEntDev{};
  EncEntDev E{};
  if ((rc = upload(c->eent_owned, books.data(), books.size(), &E.books))) return rc;
  if ((rc = upload(c->eent_owned, len.data(), len.size(), &E.len))) return rc;
  if ((rc = upload(c->eent_owned, cw.data(), cw.size(), &E.cw))) return rc;
  for (int w = 0; w < 2; w++) {
    if ((rc = upload(c->eent_owned, hf[w], (size_t)VB200_MAX_SUBMAPS, &E.floor[w]))) return rc;
    if ((rc = upload(c->eent_owned, hr[w], (size_t)VB200_MAX_SUBMAPS, &E.res[w]))) return rc;
    E.submaps[w] = S.submaps[w]; E.slots[w] = slots[w]; E.bound[w] = bound[w];
  }
  E.ch = ch; E.modebits = es->modebits;
  c->eent = E;
  return 0;
}

extern "C" int vb200_encode_packet_bound(vb200_ctx *c, int W) {
  CHECK_CTX(c); CHECK_W(W);
  if (!c->eent.books) return fail(VB200_EINVAL, "no vb200_encode_entropy_setup registered");
  return c->eent.bound[W];
}

// classification into scratch (k_residue_classify), then k_encode_packets; all pointers device.  Managed
// (k_residue_classify_curves, k_encode_packets_curves): the VB200_PACKETBLOBS curves of every block, blob_blocks
// blocks from one curve of posts / nonzero / iwork to the next; packet k*nblocks + b.  The private residue copies
// stay one per CTA either way.
static int encode_entropy_launch(vb200_ctx *c, int W, int nblocks, const vb200_block_desc *d_desc,
                                 const int32_t *d_posts, const int32_t *d_nonzero, const int32_t *d_iwork,
                                 int64_t pkt_stride, int32_t *d_bits, uint8_t *d_data, cudaStream_t st,
                                 bool managed = false, long long blob_blocks = 0) {
  const int ch = c->setup.channels, n = c->dx[W].N / 2, stride = c->res_partvals[W] > 0 ? c->res_partvals[W] : 1;
  const int curves = managed ? VB200_PACKETBLOBS : 1;
  const int grid = grid_for(c, curves * nblocks, 8);
  int32_t *cls, *work;
  int rc;
  if ((rc = carve(c->coder, [&](Carve &k) {
         cls = k.take<int32_t>((size_t)curves * nblocks * ch * stride);
         work = k.take<int32_t>((size_t)grid * ch * n);
       }))) return rc;
  if ((rc = residue_classify_launch(c, W, nblocks, curves, blob_blocks * ch, d_iwork, d_nonzero, cls, stride, st)))
    return rc;
  EncArgs A;
  A.E = c->eent; A.f1 = c->d_floor[W]; A.chmux = c->d_chmux[W]; A.desc = d_desc;
  A.posts = d_posts; A.nonzero = d_nonzero; A.iwork = d_iwork; A.classes = cls;
  A.curve_rows = blob_blocks * ch; A.work = work; A.W = W; A.nblocks = nblocks; A.n = n; A.class_stride = stride;
  A.pkt_stride = pkt_stride; A.pkt_bits = d_bits; A.data = d_data;
  const size_t smem = sizeof(int) * (size_t)c->eent.slots[W];
  if (managed) {
    if ((rc = set_smem(k_encode_packets_curves, smem))) return rc;
    k_encode_packets_curves<<<grid, ENC_THREADS, smem, st>>>(A);
  } else {
    if ((rc = set_smem(k_encode_packets, smem))) return rc;
    k_encode_packets<<<dim3(grid, 1), ENC_THREADS, smem, st>>>(A);
  }
  return post_launch(c);
}

static int encode_entropy_check(vb200_ctx *c, int nblocks) {
  if (!c->eent.books) return fail(VB200_EINVAL, "no vb200_encode_entropy_setup registered");
  if (nblocks < 0) return fail(VB200_EINVAL, "nblocks");
  return 0;
}

// both device entropy calls: checks, then encode_entropy_launch in the context scratch
static int encode_entropy_dev(vb200_ctx *c, int W, int nblocks, bool managed, int64_t blob_blocks,
                              const vb200_block_desc *d_desc, const int32_t *d_posts, const int32_t *d_nonzero,
                              const int32_t *d_iwork, int64_t pkt_stride, int32_t *d_pkt_bits, uint8_t *d_data,
                              cudaStream_t st) {
  int rc;
  if ((rc = encode_entropy_check(c, nblocks))) return rc;
  if (managed) {
    if (blob_blocks < nblocks) return fail(VB200_EINVAL, "blob_blocks < nblocks");
    if ((int64_t)VB200_PACKETBLOBS * nblocks > INT32_MAX) return fail(VB200_EINVAL, "nblocks");
  }
  if (pkt_stride % 4 || pkt_stride < c->eent.bound[W]) return fail(VB200_EINVAL, "pkt_stride: a multiple of 4, >= the packet bound");
  if (nblocks == 0) return 0;
  if (!d_desc || !d_posts || !d_nonzero || !d_iwork || !d_pkt_bits || !d_data) return fail(VB200_EINVAL, "encode_entropy pointers");
  if ((rc = scratch_begin(c, st))) return rc;
  if ((rc = encode_entropy_launch(c, W, nblocks, d_desc, d_posts, d_nonzero, d_iwork, pkt_stride, d_pkt_bits, d_data, st,
                                  managed, blob_blocks))) return rc;
  return scratch_end(c, st);
}

extern "C" int vb200_encode_entropy_dev(vb200_ctx *c, int W, int nblocks, const vb200_block_desc *d_desc,
                                        const int32_t *d_posts, const int32_t *d_nonzero, const int32_t *d_iwork,
                                        int64_t pkt_stride, int32_t *d_pkt_bits, uint8_t *d_data, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  return encode_entropy_dev(c, W, nblocks, false, 0, d_desc, d_posts, d_nonzero, d_iwork, pkt_stride, d_pkt_bits,
                            d_data, (cudaStream_t)stream);
}

// host forms: packets of the strided device buffer packed back to back, then the counts, offsets and bytes copied
// back through io (the bytes only when they fit data_cap).  Synchronises.
static int packets_pack_d2h(HostIO &io, int nblocks, const uint8_t *d_strided, int64_t stride, const int32_t *d_bits,
                            int64_t *pkt_off, int32_t *pkt_bits, uint8_t *data, int64_t data_cap) {
  vb200_ctx *c = io.c;
  cudaStream_t st = c->s_main;
  long long *doff;
  uint8_t *dpk;
  int rc;
  if ((rc = carve(c->pack, [&](Carve &k) {
         doff = k.take<long long>((size_t)nblocks + 1);
         dpk = k.take<uint8_t>((size_t)std::max<int64_t>(data_cap, 1));
       }))) return rc;
  k_packet_offsets<<<1, 1024, 0, st>>>(d_bits, nblocks, doff);
  if ((rc = post_launch(c))) return rc;
  k_packet_gather<<<grid_for(c, nblocks, 8), 256, 0, st>>>(d_strided, stride, d_bits, doff, nblocks, data_cap, dpk);
  if ((rc = post_launch(c))) return rc;
  long long total = 0;
  io.back(pkt_bits, d_bits, nblocks);
  io.back(pkt_off, (const int64_t *)doff, nblocks);
  io.back(&total, doff + nblocks, 1);
  if ((rc = io.sync())) return rc;
  if (total > data_cap) return fail(VB200_EINVAL, "packets exceed data_cap (pkt_bits filled)");
  if (total) io.back(data, dpk, total);
  return io.sync();
}

extern "C" int vb200_encode_entropy(vb200_ctx *c, int W, int nblocks, const vb200_block_desc *desc, const int32_t *posts,
                                    const int32_t *nonzero, const int32_t *iwork, int64_t *pkt_off, int32_t *pkt_bits,
                                    uint8_t *data, int64_t data_cap) {
  CHECK_CTX(c); CHECK_W(W);
  int rc;
  if ((rc = encode_entropy_check(c, nblocks))) return rc;
  if (nblocks == 0) return 0;
  if (!desc || !posts || !nonzero || !iwork || !pkt_off || !pkt_bits || (!data && data_cap > 0) || data_cap < 0)
    return fail(VB200_EINVAL, "encode_entropy pointers");
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t nb = (size_t)nblocks, ch = c->setup.channels, n = c->dx[W].N / 2;
  const int64_t stride = c->eent.bound[W];
  HostIO io{c};
  const vb200_block_desc *dd = io.in(desc, nb);
  const int32_t *dp = io.in(posts, nb * ch * VB200_FLOOR1_STRIDE), *dz = io.in(nonzero, nb * ch),
                *di = io.in(iwork, nb * ch * n);
  int32_t *db = io.out<int32_t>(nb);
  uint8_t *ds = io.out<uint8_t>((size_t)stride * nb);
  if (io.rc) return io.rc;
  if ((rc = vb200_encode_entropy_dev(c, W, nblocks, dd, dp, dz, di, stride, db, ds, c->s_main))) return rc;
  return packets_pack_d2h(io, nblocks, ds, stride, db, pkt_off, pkt_bits, data, data_cap);
}

// Both block packet calls: the chain into staged outputs, the entropy coder, the packets packed back to back.
// managed: all VB200_PACKETBLOBS packets of every block.  name: the call, for the messages.
static int encode_packets(vb200_ctx *c, int W, int nstreams, int bps, int blobno, bool managed, const char *name,
                          const vb200_encode_io *h, int64_t *pkt_off, int32_t *pkt_bits, uint8_t *data,
                          int64_t data_cap) {
  int rc;
  if (!c->eent.books) return fail(VB200_EINVAL, "no vb200_encode_entropy_setup registered");
  if (!h || h->posts || h->nonzero || h->iwork || h->classes || h->overflow || h->mdct || h->logmdct || h->logmask ||
      h->iwork_fmt != VB200_IWORK_S32)
    return fail(VB200_EINVAL, (std::string(name) + ": posts / nonzero / iwork / classes / overflow / spectra must be NULL").c_str());
  if (!pkt_off || !pkt_bits || (!data && data_cap > 0) || data_cap < 0)
    return fail(VB200_EINVAL, (std::string(name) + " outputs").c_str());
  if (managed) {
    if ((rc = managed_check(c, W, nstreams, bps, h, true))) return rc;
    if ((int64_t)VB200_PACKETBLOBS * nstreams * bps > INT32_MAX) return fail(VB200_EINVAL, "nblocks");
  } else if ((rc = enc_check(c, W, nstreams, bps, blobno, h, true))) {
    return rc;
  }
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels, N = c->dx[W].N, curves = managed ? VB200_PACKETBLOBS : 1;
  const size_t n = N / 2, nb = (size_t)nstreams * bps, rows = nb * ch;
  const int64_t stride = c->eent.bound[W];
  cudaStream_t st = c->s_main;
  HostIO io{c};
  vb200_encode_io d = *h;
  enc_stage(io, h, &d, ch, N, nstreams, bps, curves);
  int32_t *dbits = io.out<int32_t>(curves * nb);
  uint8_t *dstr = io.out<uint8_t>((size_t)stride * curves * nb);
  if (io.rc) return io.rc;
  EncScratch S;
  MgdScratch M;
  if ((rc = carve(managed ? c->mgd : c->enc, [&](Carve &k) {
         enc_layout(k, rows, nb, n, nullptr, false, &S);
         if (managed) mgd_layout(k, rows, rows, n, &M);
       }))) return rc;
  if ((rc = scratch_begin(c, st))) return rc;
  if ((rc = encode_launch(c, W, nstreams, bps, blobno, &d, S, st, managed ? &M : nullptr))) return rc;
  if ((rc = encode_entropy_launch(c, W, (int)nb, d.desc, d.posts, d.nonzero, (const int32_t *)d.iwork, stride, dbits,
                                  dstr, st, managed, managed ? (long long)nb : 0))) return rc;
  if ((rc = scratch_end(c, st))) return rc;
  io.back(h->ampmax_out, d.ampmax_out, nb);
  return packets_pack_d2h(io, curves * (int)nb, dstr, stride, dbits, pkt_off, pkt_bits, data, data_cap);
}

extern "C" int vb200_encode_packets(vb200_ctx *c, int W, int nstreams, int bps, int blobno, const vb200_encode_io *h,
                                    int64_t *pkt_off, int32_t *pkt_bits, uint8_t *data, int64_t data_cap) {
  CHECK_CTX(c); CHECK_W(W);
  return encode_packets(c, W, nstreams, bps, blobno, false, "encode_packets", h, pkt_off, pkt_bits, data, data_cap);
}

// ---- bitrate-managed: all VB200_PACKETBLOBS packets of every block ----
extern "C" int vb200_encode_entropy_managed_dev(vb200_ctx *c, int W, int nblocks, int64_t blob_blocks,
                                                const vb200_block_desc *d_desc, const int32_t *d_posts,
                                                const int32_t *d_nonzero, const int32_t *d_iwork, int64_t pkt_stride,
                                                int32_t *d_pkt_bits, uint8_t *d_data, void *stream) {
  CHECK_CTX(c); CHECK_W(W);
  return encode_entropy_dev(c, W, nblocks, true, blob_blocks, d_desc, d_posts, d_nonzero, d_iwork, pkt_stride,
                            d_pkt_bits, d_data, (cudaStream_t)stream);
}

extern "C" int vb200_encode_packets_managed(vb200_ctx *c, int W, int nstreams, int bps, const vb200_encode_io *h,
                                            int64_t *pkt_off, int32_t *pkt_bits, uint8_t *data, int64_t data_cap) {
  CHECK_CTX(c); CHECK_W(W);
  return encode_packets(c, W, nstreams, bps, VB200_PACKETBLOBS / 2, true, "encode_packets_managed", h, pkt_off,
                        pkt_bits, data, data_cap);
}

// ======================================================================== //
// the bitrate manager on the device and whole streams to packets (vb200_bitrate.cuh)
static_assert(sizeof(vb200_bitrate_info) == 48, "vb200_bitrate_info layout (mirrored by vorbis_b200/abi.py)");
static_assert(sizeof(vb200_bitrate_state) == 32, "vb200_bitrate_state layout (mirrored by vorbis_b200/abi.py)");
static_assert(sizeof(vb200_packet_info) == 32, "vb200_packet_info layout (mirrored by vorbis_b200/abi.py)");

extern "C" int vb200_bitrate_setup(vb200_ctx *c, const vb200_bitrate_info *bi) {
  CHECK_CTX(c);
  if (!bi) return fail(VB200_EINVAL, "null bitrate info");
  std::lock_guard<std::mutex> lk(c->mu);
  BitrateDev B{};
  const long long rate = c->setup.rate;
  const int halfsamples = c->setup.blocksizes[0] >> 1;
  const bool managed = bi->reservoir_bits > 0;
  if (managed) {                                     // lib/bitrate.c:34-54, in the reference's evaluation order
    B.short_per_long = c->setup.blocksizes[1] / c->setup.blocksizes[0];
    B.avg_bitsper = (long long)rint(1. * bi->avg_rate * halfsamples / rate);
    B.min_bitsper = (long long)rint(1. * bi->min_rate * halfsamples / rate);
    B.max_bitsper = (long long)rint(1. * bi->max_rate * halfsamples / rate);
    B.desired_fill = (long long)(bi->reservoir_bits * bi->reservoir_bias);
    B.reservoir_bits = bi->reservoir_bits;
    B.slewlimit = 15. / bi->slew_damp;               // lib/bitrate.c:104
    B.rate = (double)rate;
    B.samples[0] = c->setup.blocksizes[0] >> 1;
    B.samples[1] = c->setup.blocksizes[1] >> 1;
  }
  c->br = B;
  c->br_set = true;
  c->br_managed = managed;
  return 0;
}

static int bitrate_check(vb200_ctx *c) {
  if (!c->br_set || !c->br_managed) return fail(VB200_EINVAL, "no managed vb200_bitrate_setup registered");
  return 0;
}

extern "C" int vb200_bitrate_init(vb200_ctx *c, vb200_bitrate_state *state) {
  if (!c) return fail(VB200_EINVAL, "null context");
  int rc;
  if ((rc = bitrate_check(c))) return rc;
  if (!state) return fail(VB200_EINVAL, "null state");
  memset(state, 0, sizeof(*state));
  state->avg_reservoir = state->minmax_reservoir = c->br.desired_fill;
  state->avgfloat = VB200_PACKETBLOBS / 2;
  return 0;
}

extern "C" int vb200_bitrate_addblocks_dev(vb200_ctx *c, int nstreams, int max_blocks, const int32_t *d_count,
                                           const int32_t *d_W, const int32_t *d_pkt_bits, vb200_bitrate_state *d_state,
                                           int32_t *d_choice, int32_t *d_bytes, void *stream) {
  CHECK_CTX(c);
  int rc;
  if ((rc = bitrate_check(c))) return rc;
  if (nstreams <= 0) return 0;
  if (max_blocks < 1) return fail(VB200_EINVAL, "max_blocks");
  if (!d_count || !d_W || !d_pkt_bits || !d_state || !d_choice || !d_bytes) return fail(VB200_EINVAL, "bitrate_addblocks pointers");
  k_bitrate_choose<<<(nstreams + 127) / 128, 128, 0, (cudaStream_t)stream>>>(c->br, nstreams, max_blocks, d_count, d_W,
                                                                            d_pkt_bits, d_state, d_choice, d_bytes, 1);
  return post_launch(c);
}

extern "C" int vb200_bitrate_addblocks(vb200_ctx *c, int nstreams, int max_blocks, const int32_t *count, const int32_t *W,
                                       const int32_t *pkt_bits, vb200_bitrate_state *state, int32_t *choice,
                                       int32_t *bytes) {
  CHECK_CTX(c);
  int rc;
  if ((rc = bitrate_check(c))) return rc;
  if (nstreams <= 0) return 0;
  if (max_blocks < 1) return fail(VB200_EINVAL, "max_blocks");
  if (!count || !W || !pkt_bits || !state || !choice || !bytes) return fail(VB200_EINVAL, "bitrate_addblocks pointers");
  for (int s = 0; s < nstreams; s++)
    if (count[s] < 0 || count[s] > max_blocks) return fail(VB200_EINVAL, "count[s] outside [0, max_blocks]");
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = (size_t)nstreams * max_blocks;
  HostIO io{c};
  const int32_t *dc = io.in(count, nstreams), *dw = io.in(W, n), *db = io.in(pkt_bits, n * VB200_PACKETBLOBS);
  vb200_bitrate_state *ds = io.in(state, nstreams);
  // choice and bytes go in as well: entries past count[s] come back as the caller left them
  int32_t *dch = io.in(choice, n), *dby = io.in(bytes, n);
  if (io.rc) return io.rc;
  if ((rc = vb200_bitrate_addblocks_dev(c, nstreams, max_blocks, dc, dw, db, ds, dch, dby, c->s_main))) return rc;
  io.back(state, ds, nstreams);
  io.back(choice, dch, n);
  io.back(bytes, dby, n);
  return io.sync();
}

// ---- carried streams: the host carry is [nstreams][carry_bytes] of PlanCarry, the mark window (mark_cap bytes),
// the envelope state and a vb200_bitrate_state, each part 8-byte aligned.  One call stages all carries as one buffer
// of arrays (CarryBlob), laid out by carve's rule on the host and used at the same offsets on the device.
static_assert(sizeof(PlanCarry) % 8 == 0 && offsetof(PlanCarry, base) == offsetof(vb200_encode_carry, base) &&
              offsetof(PlanCarry, granulepos) == offsetof(vb200_encode_carry, granulepos) &&
              offsetof(PlanCarry, packetno) == offsetof(vb200_encode_carry, packetno) &&
              offsetof(PlanCarry, done) == offsetof(vb200_encode_carry, done) && sizeof(vb200_encode_carry) == 24,
              "vb200_encode_carry is the head of PlanCarry (mirrored by vorbis_b200/abi.py)");

struct CarryParts { size_t marks, env, br, bytes; };
static CarryParts carry_parts(const vb200_ctx *c, int cap) {
  CarryParts q;
  q.marks = sizeof(PlanCarry);
  q.env = q.marks + (((size_t)cap + 7) & ~(size_t)7);
  q.br = q.env + ((sizeof(int32_t) * VB200_VE_STATE_WORDS(c->setup.channels) + 7) & ~(size_t)7);
  q.bytes = q.br + sizeof(vb200_bitrate_state);
  return q;
}
static int carry_cap(const vb200_ctx *c, int mark_steps) {
  return mark_steps > 0 ? mark_steps : (3 * c->setup.blocksizes[1] / 2 + c->setup.blocksizes[0] / 4) / PLAN_STEP + 8;
}

extern "C" int vb200_encode_carry_bytes(vb200_ctx *c, int mark_steps) {
  CHECK_CTX(c);
  return (int)carry_parts(c, carry_cap(c, mark_steps)).bytes;
}

extern "C" int vb200_encode_carry_init(vb200_ctx *c, int nstreams, int mark_steps, void *carry) {
  CHECK_CTX(c);
  if (nstreams <= 0) return 0;
  if (!carry) return fail(VB200_EINVAL, "null carry");
  const int cap = carry_cap(c, mark_steps);
  const CarryParts q = carry_parts(c, cap);
  for (int s = 0; s < nstreams; s++) {
    char *cs = (char *)carry + (size_t)s * q.bytes;
    memset(cs, 0, q.bytes);
    PlanCarry p{};
    p.packetno = 3;                                  // lib/block.c:311
    p.centerW = p.cursor = c->setup.blocksizes[1] / 2;
    p.gmax = p.prev = -9999.f;
    p.ch = c->setup.channels; p.bs0 = c->setup.blocksizes[0]; p.bs1 = c->setup.blocksizes[1]; p.mark_cap = cap;
    p.br_ready = c->br_set && c->br_managed;
    memcpy(cs, &p, sizeof(p));
    if (p.br_ready) {
      vb200_bitrate_state b;
      vb200_bitrate_init(c, &b);
      memcpy(cs + q.br, &b, sizeof(b));
    }
  }
  return 0;
}

struct CarryBlob {
  PlanCarry *pc; uint8_t *marks; int32_t *env; vb200_bitrate_state *br; int32_t *first, *count, *overflow;
};
static void carry_blob_layout(Carve &k, size_t n, int cap, size_t sw, CarryBlob *b) {
  b->pc = k.take<PlanCarry>(n); b->marks = k.take<uint8_t>(n * cap); b->env = k.take<int32_t>(n * sw);
  b->br = k.take<vb200_bitrate_state>(n); b->first = k.take<int32_t>(n); b->count = k.take<int32_t>(n);
  b->overflow = k.take<int32_t>(1);
}

// checks the carries against the context and the call, and packs them into blob (host memory); *nsteps_env = the
// most envelope steps one stream analyses
static int carry_pack(vb200_ctx *c, int nstreams, bool managed, const vb200_streams_io *h, const void *carry,
                      std::vector<char> &blob, CarryBlob &b, int *cap_out, int *nsteps_env) {
  const PlanCarry *p0 = (const PlanCarry *)carry;
  const int ch = c->setup.channels, cap = p0->mark_cap;
  if (p0->ch != ch || p0->bs0 != c->setup.blocksizes[0] || p0->bs1 != c->setup.blocksizes[1] || cap < 1)
    return fail(VB200_EINVAL, "encode carry of another setup");
  const CarryParts q = carry_parts(c, cap);
  const size_t sw = VB200_VE_STATE_WORDS(ch);
  Carve sz{nullptr, 0};
  carry_blob_layout(sz, nstreams, cap, sw, &b);
  blob.assign(sz.off, 0);
  Carve at{blob.data(), 0};
  carry_blob_layout(at, nstreams, cap, sw, &b);
  const long long nsteps = h->stream_stride / PLAN_STEP - PLAN_VE_WIN;
  int most = 0;
  for (int s = 0; s < nstreams; s++) {
    const char *cs = (const char *)carry + (size_t)s * q.bytes;
    PlanCarry p;
    memcpy(&p, cs, sizeof(p));
    if (p.ch != ch || p.bs0 != p0->bs0 || p.bs1 != p0->bs1 || p.mark_cap != cap)
      return fail(VB200_EINVAL, "encode carries of different setups or mark capacities");
    if (managed && !p.br_ready)
      return fail(VB200_EINVAL, "encode carry made before a managed vb200_bitrate_setup (no bitrate state)");
    int first = 0, count = 0;
    if (!p.done) {
      if (h->pcm_len[s] < p.kept) return fail(VB200_EINVAL, "pcm_len below the samples the carry kept");
      if (h->pcm_len[s] > h->stream_stride) return fail(VB200_EINVAL, "pcm_len above stream_stride");
      if (h->eof && h->eof[s] != 0 && h->eof[s] <= p.base) return fail(VB200_EINVAL, "eof at or before the carry's base");
      long long last = h->pcm_len[s] / PLAN_STEP - PLAN_VE_WIN;    // lib/envelope.c:224-225, as k_plan_blocks clamps it
      if (last > nsteps) last = nsteps;
      first = (int)(p.current / PLAN_STEP);
      count = last > first ? (int)(last - first) : 0;
    }
    b.pc[s] = p;
    memcpy(b.marks + (size_t)s * cap, cs + q.marks, cap);
    memcpy(b.env + (size_t)s * sw, cs + q.env, sizeof(int32_t) * sw);
    memcpy(&b.br[s], cs + q.br, sizeof(vb200_bitrate_state));
    b.first[s] = first; b.count[s] = count;
    if (count > most) most = count;
  }
  *b.overflow = 0;
  *cap_out = cap;
  *nsteps_env = most;
  return 0;
}

static void carry_unpack(vb200_ctx *c, int nstreams, int cap, const CarryBlob &b, void *carry) {
  const CarryParts q = carry_parts(c, cap);
  const size_t sw = VB200_VE_STATE_WORDS(c->setup.channels);
  for (int s = 0; s < nstreams; s++) {
    char *cs = (char *)carry + (size_t)s * q.bytes;
    memcpy(cs, &b.pc[s], sizeof(PlanCarry));
    memcpy(cs + q.marks, b.marks + (size_t)s * cap, cap);
    memcpy(cs + q.env, b.env + (size_t)s * sw, sizeof(int32_t) * sw);
    memcpy(cs + q.br, &b.br[s], sizeof(vb200_bitrate_state));
  }
}

// The device half of every streams packets call, on st: the streams chain into d's device buffers (Kp: carried
// streams), the entropy coder per size, then (k_stream_bits, [k_bitrate_choose], k_packet_offsets, k_stream_gather)
// on the spk arena, carved once when the per-size block counts are known.  dinfo / dpk: the caller's, or when null
// carved here (dpk with data_cap bytes) and returned; *total: the device byte total.  R (the _dev raw-PCM calls): the
// chain runs without waiting for its plan, sized by cap[] (streams_front), and the call's vb200_encode_result is
// written before the gather, which writes bytes only when its rc is 0.
struct SpkResult { vb200_encode_result *res; const int32_t *bad; };
static int spk_chain(vb200_ctx *c, int nstreams, int blobno, bool managed, vb200_streams_io *d, cudaStream_t st,
                     const CarryDev *Kp, int nsteps_env, vb200_packet_info *&dinfo, uint8_t *&dpk, int64_t data_cap,
                     long long **total, const SpkResult *R = nullptr) {
  int rc;
  const int curves = managed ? VB200_PACKETBLOBS : 1;
  const size_t n = (size_t)nstreams * d->max_blocks;
  vb200_block_desc *desc[2] = {nullptr, nullptr};
  const int32_t *d_tot = nullptr;
  if ((rc = encode_streams_launch(c, nstreams, blobno, managed, d, st, desc, Kp, nsteps_env, R ? &d_tot : nullptr)))
    return rc;
  int32_t *bits[2] = {nullptr, nullptr}, *Wb, *sbits, *fbits, *choice = nullptr;
  uint8_t *strided[2] = {nullptr, nullptr};
  long long *off;
  const bool own_info = !dinfo, own_data = !dpk;
  if ((rc = carve(c->spk, [&](Carve &k) {
         for (int w = 0; w < 2; w++) {
           const size_t cnt = d->count[w];
           if (!cnt) continue;
           bits[w] = k.take<int32_t>(curves * cnt);
           strided[w] = k.take<uint8_t>(curves * cnt * (size_t)c->eent.bound[w]);
         }
         Wb = k.take<int32_t>(n); sbits = k.take<int32_t>(n * curves); fbits = k.take<int32_t>(n);
         if (managed) choice = k.take<int32_t>(n);
         off = k.take<long long>(n + 1);
         if (own_info) dinfo = k.take<vb200_packet_info>(n);
         if (own_data) dpk = k.take<uint8_t>((size_t)std::max<int64_t>(data_cap, 1));
       }))) return rc;
  for (int w = 0; w < 2; w++) {
    const int cnt = d->count[w];
    if (!cnt) continue;
    if ((rc = encode_entropy_dev(c, w, cnt, managed, managed ? d->cap[w] : 0, desc[w], d->posts[w], d->nonzero[w],
                                 d->iwork[w], c->eent.bound[w], bits[w], strided[w], st))) return rc;
  }
  k_stream_bits<<<grid_for(c, (int)((n + 255) / 256), 8), 256, 0, st>>>(nstreams, d->max_blocks, d->plan, d->nblocks,
                                                                        curves, bits[0], bits[1], d->count[0],
                                                                        d->count[1], Wb, sbits, fbits);
  if ((rc = post_launch(c))) return rc;
  if (managed) {
    k_bitrate_choose<<<(nstreams + 127) / 128, 128, 0, st>>>(c->br, nstreams, d->max_blocks, d->nblocks, Wb, sbits,
                                                             Kp ? Kp->br : nullptr, choice, fbits, 8);
    if ((rc = post_launch(c))) return rc;
  }
  k_packet_offsets<<<1, 1024, 0, st>>>(fbits, (int)n, off);
  if ((rc = post_launch(c))) return rc;
  if (R) {
    k_pcm_result<<<1, 32, 0, st>>>(R->res, off + n, data_cap, d_tot, d->cap[0], d->cap[1], Kp->overflow, R->bad);
    if ((rc = post_launch(c))) return rc;
  }
  GatherArgs A;
  A.plan = d->plan; A.nblocks = d->nblocks; A.eof = d->eof; A.nstreams = nstreams; A.max_blocks = d->max_blocks;
  A.curves = curves;
  for (int w = 0; w < 2; w++) {
    A.bs[w] = c->setup.blocksizes[w]; A.count[w] = d->count[w]; A.stride[w] = c->eent.bound[w]; A.data[w] = strided[w];
  }
  A.sbits = sbits; A.choice = choice; A.fbits = fbits; A.off = off; A.cap = data_cap; A.info = dinfo; A.dst = dpk;
  A.rc = R ? &R->res->rc : nullptr;
  if (Kp)
    k_stream_gather_carry<<<grid_for(c, (int)n, 8), 256, 0, st>>>(A, Kp->pc);
  else
    k_stream_gather<<<grid_for(c, (int)n, 8), 256, 0, st>>>(A);
  if ((rc = post_launch(c))) return rc;
  *total = off + n;
  return 0;
}

// Both whole-stream packet calls: the streams chain on staged device buffers (spk_chain).  One synchronous round
// trip on s_main.  carry (host): the _resume forms, whose carries are staged as one more buffer and written back only
// when the call succeeds.
static int streams_packets(vb200_ctx *c, int nstreams, int blobno, bool managed, vb200_streams_io *h,
                           vb200_packet_info *info, uint8_t *data, int64_t data_cap, void *carry = nullptr) {
  int rc;
  if ((rc = streams_open(c, h))) return rc;
  if (!c->eent.books) return fail(VB200_EINVAL, "no vb200_encode_entropy_setup registered");
  if (managed && (rc = bitrate_check(c))) return rc;
  if (!managed && (blobno < 0 || blobno >= VB200_PACKETBLOBS)) return fail(VB200_EINVAL, "blobno");
  if (nstreams <= 0) return 0;
  if ((rc = streams_inputs(h, "encode_streams_packets"))) return rc;
  for (int w = 0; w < 2; w++) {
    if (h->posts[w] || h->nonzero[w] || h->iwork[w] || h->ampmax_out[w])
      return fail(VB200_EINVAL, "encode_streams_packets: posts / nonzero / iwork / ampmax_out must be NULL");
    if (h->cap[w] < 0) return fail(VB200_EINVAL, "cap");
  }
  if (!info || (!data && data_cap > 0) || data_cap < 0) return fail(VB200_EINVAL, "encode_streams_packets outputs");
  if ((int64_t)nstreams * h->max_blocks > INT32_MAX / VB200_PACKETBLOBS) return fail(VB200_EINVAL, "nstreams x max_blocks");
  std::vector<char> cblob;
  CarryBlob hb{};
  int ccap = 0, nsteps_env = 0;
  if (carry && (rc = carry_pack(c, nstreams, managed, h, carry, cblob, hb, &ccap, &nsteps_env))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = (size_t)nstreams * h->max_blocks;
  HostIO io{c};
  vb200_streams_io d;
  streams_stage(c, io, nstreams, managed, true, h, &d);
  char *dblob = carry ? io.in(cblob.data(), cblob.size()) : nullptr;
  if (io.rc) return io.rc;
  CarryDev K{}, *Kp = nullptr;
  if (carry) {
    auto dev = [&](auto *hp) { return (decltype(hp))(dblob + ((char *)hp - cblob.data())); };
    K.pc = dev(hb.pc); K.marks = dev(hb.marks); K.cap = ccap; K.env = dev(hb.env); K.br = dev(hb.br);
    K.first = dev(hb.first); K.count = dev(hb.count); K.overflow = dev(hb.overflow);
    Kp = &K;
  }
  vb200_packet_info *dinfo = nullptr;
  uint8_t *dpk = nullptr;
  long long *dtotal;
  rc = spk_chain(c, nstreams, blobno, managed, &d, c->s_main, Kp, nsteps_env, dinfo, dpk, data_cap, &dtotal);
  h->count[0] = d.count[0]; h->count[1] = d.count[1];
  if (rc) return rc;
  long long total = 0;
  if (carry) io.back(cblob.data(), dblob, cblob.size());
  io.back(h->plan, d.plan, n);
  io.back(h->nblocks, d.nblocks, nstreams);
  io.back(info, dinfo, n);
  io.back(&total, dtotal, 1);
  if ((rc = io.sync())) return rc;
  if (total > data_cap) return fail(VB200_EINVAL, "packets exceed data_cap (info filled)");
  if (total) io.back(data, dpk, total);
  if ((rc = io.sync())) return rc;
  if (carry) carry_unpack(c, nstreams, ccap, hb, carry);
  return 0;
}

extern "C" int vb200_encode_streams_packets(vb200_ctx *c, int nstreams, int blobno, vb200_streams_io *io,
                                            vb200_packet_info *info, uint8_t *data, int64_t data_cap) {
  CHECK_CTX(c);
  return streams_packets(c, nstreams, blobno, false, io, info, data, data_cap);
}

extern "C" int vb200_encode_streams_packets_managed(vb200_ctx *c, int nstreams, vb200_streams_io *io,
                                                    vb200_packet_info *info, uint8_t *data, int64_t data_cap) {
  CHECK_CTX(c);
  return streams_packets(c, nstreams, 0, true, io, info, data, data_cap);
}

extern "C" int vb200_encode_streams_packets_resume(vb200_ctx *c, int nstreams, int blobno, vb200_streams_io *io,
                                                   void *carry, vb200_packet_info *info, uint8_t *data,
                                                   int64_t data_cap) {
  CHECK_CTX(c);
  if (!carry) return fail(VB200_EINVAL, "null carry");
  return streams_packets(c, nstreams, blobno, false, io, info, data, data_cap, carry);
}

extern "C" int vb200_encode_streams_packets_managed_resume(vb200_ctx *c, int nstreams, vb200_streams_io *io,
                                                           void *carry, vb200_packet_info *info, uint8_t *data,
                                                           int64_t data_cap) {
  CHECK_CTX(c);
  if (!carry) return fail(VB200_EINVAL, "null carry");
  return streams_packets(c, nstreams, 0, true, io, info, data, data_cap, carry);
}

// ---- raw PCM to packets: vorbis_analysis_wrote's LPC preamble and tail on the device, in front of the carried streams
// packets path.  The host carry of a stream is a PcmCarry, then the encode carry (carry_parts bytes), then the filters
// of every channel (LPC_FILTER_FLOATS floats: the order-16 preamble coefficients and prime, the order-32 tail
// coefficients and prime), each part 8-byte aligned.
static_assert(offsetof(PcmCarry, raw_base) == offsetof(vb200_pcm_carry, raw_base) &&
              offsetof(PcmCarry, written) == offsetof(vb200_pcm_carry, written) &&
              offsetof(PcmCarry, ended) == offsetof(vb200_pcm_carry, ended) &&
              offsetof(PcmCarry, drained) == offsetof(vb200_pcm_carry, drained) && sizeof(vb200_pcm_carry) == 48 &&
              sizeof(PcmCarry) % 8 == 0, "vb200_pcm_carry is the head of PcmCarry (mirrored by vorbis_b200/abi.py)");

static size_t pcm_filt_bytes(const vb200_ctx *c) { return sizeof(float) * LPC_FILTER_FLOATS * c->setup.channels; }

extern "C" int vb200_encode_pcm_carry_bytes(vb200_ctx *c, int mark_steps) {
  CHECK_CTX(c);
  return (int)(sizeof(PcmCarry) + carry_parts(c, carry_cap(c, mark_steps)).bytes + pcm_filt_bytes(c));
}

extern "C" int vb200_encode_pcm_carry_init(vb200_ctx *c, int nstreams, int mark_steps, void *carry) {
  CHECK_CTX(c);
  if (nstreams <= 0) return 0;
  if (!carry) return fail(VB200_EINVAL, "null carry");
  const size_t eb = carry_parts(c, carry_cap(c, mark_steps)).bytes, pb = sizeof(PcmCarry) + eb + pcm_filt_bytes(c);
  for (int s = 0; s < nstreams; s++) {
    char *cs = (char *)carry + (size_t)s * pb;
    memset(cs, 0, pb);
    int rc;
    if ((rc = vb200_encode_carry_init(c, 1, mark_steps, cs + sizeof(PcmCarry)))) return rc;
    PcmCarry p{};
    memcpy(&p.enc, cs + sizeof(PcmCarry), sizeof(p.enc));
    p.drained = 1;
    p.ch = c->setup.channels; p.bs1 = c->setup.blocksizes[1];
    memcpy(cs, &p, sizeof(p));
  }
  return 0;
}

// The device buffers of one raw-PCM call, and what the chain gives back
struct PcmCall {
  const void *pcm;
  int s16, max_blocks, mark_cap, cap[2];
  int64_t stride;
  const int64_t *pcm_len, *first;        // first: null for the carries' raw_base
  const int32_t *end;
  unsigned char *carry;                  // [nstreams][vb200_encode_pcm_carry_bytes]
  vb200_stream_block *plan;
  int32_t *nblocks, *status;
  vb200_packet_info *info;               // info and data: the caller's, or null for the spk arena's (returned)
  uint8_t *data;
  int64_t data_cap;
  vb200_encode_result *res;              // the _dev forms: the result and the refusals on the device
  int count[2];                          // out: the plan's totals
  long long *total;                      // out: the byte total (device)
  int32_t *bad;                          // out: some stream was refused (device)
};

// The raw-PCM chain of both forms on st.  Launches: k_pcm_pack, k_lpc_filter<16> (the preamble filters due this
// call), k_pcm_timeline<false> (the timelines up to eof), k_lpc_filter<32> (the tail filters due, which read those
// timelines), k_pcm_timeline<true> (the tails), the streams packets chain on the timelines ([k_pcm_result] for the
// _dev forms), then k_pcm_unpack: six more than the _resume calls, whatever the stream count.  The timeline stride is
// known from the input stride, so nothing here waits for the host; the streams chain waits once for its plan.
static int pcm_chain(vb200_ctx *c, int nstreams, int blobno, bool managed, PcmCall &P, cudaStream_t st) {
  int rc;
  const int ch = c->setup.channels, bs1 = c->setup.blocksizes[1], half = bs1 / 2;
  const CarryParts q = carry_parts(c, P.mark_cap);
  const size_t sw = VB200_VE_STATE_WORDS(ch), curves = managed ? VB200_PACKETBLOBS : 1;
  const long long tstride = (P.stride + half + 3LL * bs1 + 3) & ~3LL;     // the longest timeline a stream passes
  const int nsteps = (int)(tstride / PLAN_STEP) - PLAN_VE_WIN;
  PcmPackArgs A{};
  vb200_streams_io d{};
  float *dtl;
  int32_t *flags;                        // the mark window overflow, then bad
  if ((rc = carve(c->ptl, [&](Carve &k) {
         dtl = k.take<float>((size_t)nstreams * ch * tstride);
         A.ps = k.take<PcmStream>(nstreams); A.tl_len = k.take<int64_t>(nstreams); A.eof = k.take<int64_t>(nstreams);
         A.jobs = k.take<LpcJob>(2 * (size_t)nstreams * ch);
         A.filt = k.take<float>((size_t)nstreams * ch * LPC_FILTER_FLOATS);
         A.head = k.take<PcmCarry>(nstreams); A.pc = k.take<PlanCarry>(nstreams);
         A.mk = k.take<uint8_t>((size_t)nstreams * P.mark_cap); A.envs = k.take<int32_t>(nstreams * sw);
         A.brs = k.take<vb200_bitrate_state>(nstreams);
         A.first_step = k.take<int32_t>(nstreams); A.count = k.take<int32_t>(nstreams);
         flags = k.take<int32_t>(2);
         for (int w = 0; w < 2; w++) {
           if (P.cap[w] <= 0) continue;
           const size_t rows = curves * P.cap[w] * ch, n = c->dx[w].N / 2;
           d.posts[w] = k.take<int32_t>(rows * VB200_FLOOR1_STRIDE); d.nonzero[w] = k.take<int32_t>(rows);
           d.iwork[w] = k.take<int32_t>(rows * n); d.ampmax_out[w] = k.take<float>(P.cap[w]);
         }
       }))) return rc;
  if ((rc = scratch_begin(c, st))) return rc;
  CU(cudaMemsetAsync(dtl, 0, sizeof(float) * nstreams * ch * tstride, st));   // columns past a stream's len read as 0
  CU(cudaMemsetAsync(flags, 0, 2 * sizeof(int32_t), st));
  A.carry = P.carry; A.pb = (long long)(sizeof(PcmCarry) + q.bytes + pcm_filt_bytes(c));
  A.marks = q.marks; A.env = q.env; A.br = q.br;
  A.nstreams = nstreams; A.ch = ch; A.bs0 = c->setup.blocksizes[0]; A.bs1 = bs1; A.cap = P.mark_cap;
  A.managed = managed; A.env_words = (int)sw;
  A.pcm_len = P.pcm_len; A.first = P.first; A.end = P.end; A.in_stride = P.stride; A.tl_stride = tstride;
  A.nsteps = nsteps; A.in = P.pcm; A.s16 = P.s16; A.tl = dtl; A.status = P.status; A.bad = flags + 1;
  k_pcm_pack<<<(nstreams + 127) / 128, 128, 0, st>>>(A);
  if ((rc = post_launch(c))) return rc;
  PcmTimelineArgs T;
  T.in = P.pcm; T.s16 = P.s16; T.ch = ch; T.half = half; T.in_stride = P.stride; T.tl_stride = tstride;
  T.st = A.ps; T.filt = A.filt; T.tl = dtl; T.nstreams = nstreams;
  const int pairs = nstreams * ch, lg = grid_for(c, (pairs + LPC_WARPS - 1) / LPC_WARPS, 8);
  k_lpc_filter<LPC_PRE><<<lg, 32 * LPC_WARPS, 0, st>>>(A.jobs, pairs, 1);
  if ((rc = post_launch(c))) return rc;
  k_pcm_timeline<false><<<grid_for(c, pairs, 8), 256, 0, st>>>(T);
  if ((rc = post_launch(c))) return rc;
  k_lpc_filter<LPC_TAIL><<<lg, 32 * LPC_WARPS, 0, st>>>(A.jobs + pairs, pairs, 1);
  if ((rc = post_launch(c))) return rc;
  k_pcm_timeline<true><<<(pairs + 255) / 256, 256, 0, st>>>(T);
  if ((rc = post_launch(c))) return rc;
  d.pcm = dtl; d.pcm_fmt = VB200_PCM_F32_PLANAR; d.max_blocks = P.max_blocks; d.stream_stride = tstride;
  d.pcm_len = A.tl_len; d.eof = A.eof; d.plan = P.plan; d.nblocks = P.nblocks;
  d.cap[0] = P.cap[0]; d.cap[1] = P.cap[1];
  CarryDev K;
  K.pc = A.pc; K.marks = A.mk; K.cap = P.mark_cap; K.env = A.envs; K.br = A.brs; K.first = A.first_step;
  K.count = A.count; K.overflow = flags;
  const SpkResult R{P.res, A.bad};
  P.bad = A.bad;
  rc = spk_chain(c, nstreams, blobno, managed, &d, st, &K, nsteps, P.info, P.data, P.data_cap, &P.total,
                 P.res ? &R : nullptr);
  P.count[0] = d.count[0]; P.count[1] = d.count[1];
  if (rc) return rc;
  k_pcm_unpack<<<(nstreams + 127) / 128, 128, 0, st>>>(A, P.nblocks, P.max_blocks, P.res ? &P.res->rc : nullptr);
  return post_launch(c);
}

// the checks both forms make on the host, in the host form's order after its own first ones
static int pcm_call_check(vb200_ctx *c, int nstreams, int blobno, bool managed, const vb200_pcm_io *h,
                          const void *info, const uint8_t *data, int64_t data_cap) {
  int rc;
  if ((rc = plan_check(c))) return rc;
  if (!c->eent.books) return fail(VB200_EINVAL, "no vb200_encode_entropy_setup registered");
  if (managed && (rc = bitrate_check(c))) return rc;
  if (!managed && (blobno < 0 || blobno >= VB200_PACKETBLOBS)) return fail(VB200_EINVAL, "blobno");
  if (!h->plan || !h->nblocks) return fail(VB200_EINVAL, "encode_streams_packets: pcm, pcm_len, plan, nblocks");
  if (h->cap[0] < 0 || h->cap[1] < 0) return fail(VB200_EINVAL, "cap");
  if (!info || (!data && data_cap > 0) || data_cap < 0) return fail(VB200_EINVAL, "encode_streams_packets outputs");
  if ((int64_t)nstreams * h->max_blocks > INT32_MAX / VB200_PACKETBLOBS) return fail(VB200_EINVAL, "nstreams x max_blocks");
  return cqn_channels_check(c);
}

static int pcm_packets(vb200_ctx *c, int nstreams, int blobno, bool managed, vb200_pcm_io *h, void *carry,
                       vb200_packet_info *info, uint8_t *data, int64_t data_cap) {
  int rc;
  if (!h) return fail(VB200_EINVAL, "null io");
  h->count[0] = h->count[1] = 0;
  if (h->pcm_fmt != VB200_PCM_F32_PLANAR && h->pcm_fmt != VB200_PCM_S16_INTERLEAVED) return fail(VB200_EINVAL, "pcm format");
  if (nstreams <= 0) return 0;
  if (!carry) return fail(VB200_EINVAL, "null carry");
  if (!h->pcm || !h->pcm_len || h->stream_stride < 0 || h->max_blocks < 1) return fail(VB200_EINVAL, "encode_pcm_packets: pcm, pcm_len, stride, max_blocks");
  const int ch = c->setup.channels, bs1 = c->setup.blocksizes[1];
  PcmCarry p0;
  memcpy(&p0, carry, sizeof(p0));
  if (p0.ch != ch || p0.bs1 != bs1) return fail(VB200_EINVAL, "pcm carry of another setup");
  const int mark_cap = ((const PlanCarry *)((const char *)carry + sizeof(PcmCarry)))->mark_cap;
  const size_t pb = sizeof(PcmCarry) + carry_parts(c, mark_cap).bytes + pcm_filt_bytes(c);
  // the refusals k_pcm_pack reports on the device, here with their messages (keep the two in step)
  for (int s = 0; s < nstreams; s++) {
    const char *cs = (const char *)carry + (size_t)s * pb;
    PcmCarry p;
    memcpy(&p, cs, sizeof(p));
    if (p.ch != ch || p.bs1 != bs1) return fail(VB200_EINVAL, "pcm carries of different setups");
    const int64_t kept = p.written - p.raw_base, fresh = h->pcm_len[s] - kept;
    const bool end = h->end && h->end[s];
    if (fresh < 0) return fail(VB200_EINVAL, "pcm_len below the input samples the carry kept");
    if (h->pcm_len[s] > h->stream_stride) return fail(VB200_EINVAL, "pcm_len above stream_stride");
    if (p.ended && fresh) return fail(VB200_EINVAL, "samples after the end");
    if (end && p.ended) return fail(VB200_EINVAL, "a second end");
    if (end && fresh) return fail(VB200_EINVAL, "an end call with new samples (end is vorbis_analysis_wrote(v, 0))");
    if (end && !p.drained) return fail(VB200_EINVAL, "an end call on a carry max_blocks left undrained");
  }
  if ((rc = pcm_call_check(c, nstreams, blobno, managed, h, info, data, data_cap))) return rc;
  for (int s = 0; s < nstreams; s++) {
    PlanCarry q;
    memcpy(&q, (const char *)carry + (size_t)s * pb + sizeof(PcmCarry), sizeof(q));
    if (q.ch != ch || q.bs0 != c->setup.blocksizes[0] || q.bs1 != bs1 || q.mark_cap != mark_cap || mark_cap < 1)
      return fail(VB200_EINVAL, "encode carries of different setups or mark capacities");
    if (managed && !q.br_ready)
      return fail(VB200_EINVAL, "encode carry made before a managed vb200_bitrate_setup (no bitrate state)");
  }
  std::lock_guard<std::mutex> lk(c->mu);
  const size_t n = (size_t)nstreams * h->max_blocks;
  HostIO io{c};
  PcmCall P{};
  P.s16 = h->pcm_fmt == VB200_PCM_S16_INTERLEAVED;
  const size_t in_bytes = (size_t)nstreams * ch * (size_t)h->stream_stride * (P.s16 ? 2 : 4);
  P.pcm = io.in(in_bytes ? h->pcm : nullptr, std::max<size_t>(in_bytes, 1));
  P.max_blocks = h->max_blocks; P.mark_cap = mark_cap; P.cap[0] = h->cap[0]; P.cap[1] = h->cap[1];
  P.stride = h->stream_stride;
  P.pcm_len = io.in(h->pcm_len, nstreams);
  P.end = h->end ? io.in(h->end, nstreams) : nullptr;
  P.carry = (unsigned char *)io.in((const char *)carry, nstreams * pb);
  P.plan = io.out<vb200_stream_block>(n); P.nblocks = io.out<int32_t>(nstreams); P.status = io.out<int32_t>(nstreams);
  P.data_cap = data_cap;
  if (io.rc) return io.rc;
  rc = pcm_chain(c, nstreams, blobno, managed, P, c->s_main);
  h->count[0] = P.count[0]; h->count[1] = P.count[1];
  if (rc) return rc;
  if ((rc = scratch_end(c, c->s_main))) return rc;
  long long total = 0;
  int bad = 0;
  io.back(h->plan, P.plan, n);
  io.back(h->nblocks, P.nblocks, nstreams);
  io.back(info, P.info, n);
  io.back(&total, P.total, 1);
  io.back(&bad, P.bad, 1);
  if ((rc = io.sync())) return rc;
  if (bad) return fail(VB200_EINVAL, "pcm carry inconsistent with its encode carry");
  if (total > data_cap) return fail(VB200_EINVAL, "packets exceed data_cap (info filled)");
  if (total) io.back(data, P.data, total);
  io.back((char *)carry, (const char *)P.carry, nstreams * pb);
  return io.sync();
}

extern "C" int vb200_encode_pcm_packets(vb200_ctx *c, int nstreams, int blobno, vb200_pcm_io *io, void *carry,
                                        vb200_packet_info *info, uint8_t *data, int64_t data_cap) {
  CHECK_CTX(c);
  return pcm_packets(c, nstreams, blobno, false, io, carry, info, data, data_cap);
}

extern "C" int vb200_encode_pcm_packets_managed(vb200_ctx *c, int nstreams, vb200_pcm_io *io, void *carry,
                                                vb200_packet_info *info, uint8_t *data, int64_t data_cap) {
  CHECK_CTX(c);
  return pcm_packets(c, nstreams, 0, true, io, carry, info, data, data_cap);
}

static int pcm_packets_dev(vb200_ctx *c, int nstreams, int blobno, bool managed, int mark_steps, const vb200_pcm_io *h,
                           const int64_t *d_first, void *d_carry, vb200_packet_info *d_info, uint8_t *d_data,
                           int64_t data_cap, int32_t *d_status, vb200_encode_result *d_result, void *stream) {
  int rc;
  if (!h) return fail(VB200_EINVAL, "null io");
  if (h->pcm_fmt != VB200_PCM_F32_PLANAR && h->pcm_fmt != VB200_PCM_S16_INTERLEAVED) return fail(VB200_EINVAL, "pcm format");
  if (nstreams <= 0) return 0;
  if (!h->pcm || !h->pcm_len || h->stream_stride < 0 || h->max_blocks < 1) return fail(VB200_EINVAL, "encode_pcm_packets: pcm, pcm_len, stride, max_blocks");
  if (!d_carry || !d_status || !d_result) return fail(VB200_EINVAL, "encode_pcm_packets_dev: carry, status, result");
  if ((rc = pcm_call_check(c, nstreams, blobno, managed, h, d_info, d_data, data_cap))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  PcmCall P{};
  P.pcm = h->pcm; P.s16 = h->pcm_fmt == VB200_PCM_S16_INTERLEAVED; P.max_blocks = h->max_blocks;
  P.mark_cap = carry_cap(c, mark_steps); P.cap[0] = h->cap[0]; P.cap[1] = h->cap[1]; P.stride = h->stream_stride;
  P.pcm_len = h->pcm_len; P.first = d_first; P.end = h->end; P.carry = (unsigned char *)d_carry;
  P.plan = h->plan; P.nblocks = h->nblocks; P.status = d_status; P.info = d_info; P.data = d_data;
  P.data_cap = data_cap; P.res = d_result;
  if ((rc = pcm_chain(c, nstreams, blobno, managed, P, st))) return rc;
  return scratch_end(c, st);
}

extern "C" int vb200_encode_pcm_packets_dev(vb200_ctx *c, int nstreams, int blobno, int mark_steps,
                                            const vb200_pcm_io *d_io, const int64_t *d_first, void *d_carry,
                                            vb200_packet_info *d_info, uint8_t *d_data, int64_t data_cap,
                                            int32_t *d_status, vb200_encode_result *d_result, void *stream) {
  CHECK_CTX(c);
  return pcm_packets_dev(c, nstreams, blobno, false, mark_steps, d_io, d_first, d_carry, d_info, d_data, data_cap,
                         d_status, d_result, stream);
}

extern "C" int vb200_encode_pcm_packets_managed_dev(vb200_ctx *c, int nstreams, int mark_steps,
                                                    const vb200_pcm_io *d_io, const int64_t *d_first, void *d_carry,
                                                    vb200_packet_info *d_info, uint8_t *d_data, int64_t data_cap,
                                                    int32_t *d_status, vb200_encode_result *d_result, void *stream) {
  CHECK_CTX(c);
  return pcm_packets_dev(c, nstreams, 0, true, mark_steps, d_io, d_first, d_carry, d_info, d_data, data_cap, d_status,
                         d_result, stream);
}

extern "C" int vb200_lpc_extrapolate(vb200_ctx *c, int nrows, int order, const float *data, int64_t data_stride,
                                     const int32_t *n, int32_t count, float *coeff, float *out, int64_t out_stride) {
  CHECK_CTX(c);
  if (order != LPC_PRE && order != LPC_TAIL) return fail(VB200_EINVAL, "lpc order must be 16 or 32");
  if (nrows <= 0) return 0;
  if (!data || !n || !coeff || (count > 0 && !out) || count < 0 || out_stride < count) return fail(VB200_EINVAL, "lpc_extrapolate arguments");
  for (int r = 0; r < nrows; r++)
    if (n[r] < order || n[r] > data_stride) return fail(VB200_EINVAL, "lpc_extrapolate: n[r] outside [order, data_stride]");
  std::lock_guard<std::mutex> lk(c->mu);
  cudaStream_t st = c->s_main;
  HostIO io{c};
  const float *dd = io.in(data, (size_t)nrows * data_stride);
  float *dc = io.out<float>((size_t)nrows * order), *dp = io.out<float>((size_t)nrows * order);
  float *dout = count > 0 ? io.out<float>((size_t)nrows * out_stride) : nullptr;
  std::vector<LpcJob> jobs(nrows);
  for (int r = 0; r < nrows; r++) {
    LpcJob &J = jobs[r];
    J = LpcJob{};
    J.src = dd; J.off = (long long)r * data_stride; J.step = 1; J.n = n[r];
    J.coef = dc + (size_t)r * order; J.prime = dp + (size_t)r * order;
  }
  const LpcJob *dj = io.in(jobs.data(), nrows);
  if (io.rc) return io.rc;
  const int grid = grid_for(c, (nrows + LPC_WARPS - 1) / LPC_WARPS, 8);
  if (order == LPC_PRE) k_lpc_filter<LPC_PRE><<<grid, 32 * LPC_WARPS, 0, st>>>(dj, nrows, 0);
  else k_lpc_filter<LPC_TAIL><<<grid, 32 * LPC_WARPS, 0, st>>>(dj, nrows, 0);
  int rc;
  if ((rc = post_launch(c))) return rc;
  if (count > 0) {
    if (order == LPC_PRE)
      k_lpc_predict<LPC_PRE><<<(nrows + 127) / 128, 128, 0, st>>>(nrows, dc, dp, count, dout, out_stride);
    else
      k_lpc_predict<LPC_TAIL><<<(nrows + 127) / 128, 128, 0, st>>>(nrows, dc, dp, count, dout, out_stride);
    if ((rc = post_launch(c))) return rc;
    CU(cudaMemcpy2DAsync(out, sizeof(float) * out_stride, dout, sizeof(float) * out_stride, sizeof(float) * count,
                         nrows, cudaMemcpyDeviceToHost, st));
  }
  io.back(coeff, dc, (size_t)nrows * order);
  return io.sync();
}

// ======================================================================== //
// envelope / block-switch detector
static int env_check(vb200_ctx *c, int nstreams, const void *pcm, int fmt, int64_t stride, int first, int nsteps,
                     const void *state, const void *ret) {
  if (!pcm || !state || !ret) return fail(VB200_EINVAL, "envelope pointers");
  if (nstreams <= 0 || nsteps < 0 || first < 0) return fail(VB200_EINVAL, "nstreams/steps");
  if (fmt != VB200_PCM_F32_PLANAR && fmt != VB200_PCM_S16_INTERLEAVED) return fail(VB200_EINVAL, "pcm format");
  if ((int64_t)ENV_STEP * ((int64_t)first + nsteps - 1) + ENV_N > stride && nsteps > 0)
    return fail(VB200_EINVAL, "steps exceed the stream buffer");
  (void)c;
  return 0;
}

// d_first_per_stream (with d_steps_per_stream): stream s analyses steps d_first_per_stream[s] + j, j < its count,
// and first_step is 0
static int envelope_search_launch(vb200_ctx *c, int nstreams, const void *d_pcm, int fmt, int64_t stride,
                                  int first_step, int nsteps, int32_t *d_state, uint8_t *d_ret, void *stream,
                                  const int32_t *d_steps_per_stream, const int32_t *d_first_per_stream) {
  CHECK_CTX(c);
  int rc;
  if ((rc = env_check(c, nstreams, d_pcm, fmt, stride, first_step, nsteps, d_state, d_ret))) return rc;
  if (nsteps == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int ch = c->setup.channels;
  // bounded scratch: the spectra of at most ~4M (stream, channel, step) items at a time
  long per_step = (long)nstreams * ch;
  int chunk = (int)((1L << 22) / per_step);
  if (chunk < 1) chunk = 1;
  if (chunk > nsteps) chunk = nsteps;
  float *p_t, *p_v;
  if ((rc = carve(c->env_scratch, [&](Carve &k) {
         p_t = k.take<float>((size_t)per_step * chunk);
         p_v = k.take<float>((size_t)per_step * chunk * 32);
       }))) return rc;
  EnvSrc src; src.base = d_pcm; src.fmt = fmt; src.stride = stride; src.ch = ch;
  if ((rc = scratch_begin(c, st))) return rc;
  for (int j0 = 0; j0 < nsteps; j0 += chunk) {
    const int ns = nsteps - j0 < chunk ? nsteps - j0 : chunk;
    const long items = per_step * ns;
    const int grid = grid_for(c, (int)((items + ENV_WARPS - 1) / ENV_WARPS), 16);
    if (d_first_per_stream)
      k_env_spectrum_var<<<grid, 32 * ENV_WARPS, 0, st>>>(c->env, src, nstreams, j0, ns, p_t, p_v, d_first_per_stream,
                                                          d_steps_per_stream);
    else
      k_env_spectrum<<<grid, 32 * ENV_WARPS, 0, st>>>(c->env, src, nstreams, first_step + j0, ns, p_t, p_v);
    if ((rc = post_launch(c))) return rc;
    k_env_filter<<<(nstreams + ENV_WARPS - 1) / ENV_WARPS, 32 * ENV_WARPS, 0, st>>>(
        c->env, nstreams, ch, ns, nsteps, j0, p_t, p_v, d_state, d_ret, d_steps_per_stream);
    if ((rc = post_launch(c))) return rc;
  }
  return scratch_end(c, st);
}

extern "C" int vb200_envelope_search_dev(vb200_ctx *c, int nstreams, const void *d_pcm, int fmt, int64_t stride,
                                         int first_step, int nsteps, int32_t *d_state, uint8_t *d_ret, void *stream) {
  return envelope_search_launch(c, nstreams, d_pcm, fmt, stride, first_step, nsteps, d_state, d_ret, stream, nullptr,
                                nullptr);
}

static int envelope_search_host(vb200_ctx *c, int nstreams, const void *pcm, int fmt, int64_t stride,
                                int first_step, int nsteps, int32_t *state, uint8_t *ret, const int32_t *steps_per_stream) {
  CHECK_CTX(c);
  int rc;
  if ((rc = env_check(c, nstreams, pcm, fmt, stride, first_step, nsteps, state, ret))) return rc;
  if (nsteps == 0) return 0;
  std::lock_guard<std::mutex> lk(c->mu);
  const int ch = c->setup.channels;
  const size_t pcm_bytes = (fmt == VB200_PCM_S16_INTERLEAVED ? sizeof(int16_t) : sizeof(float)) * (size_t)nstreams * ch * (size_t)stride;
  const size_t st_len = (size_t)nstreams * VB200_VE_STATE_WORDS(ch);
  HostIO io{c};
  const int32_t *dn = steps_per_stream ? io.in(steps_per_stream, nstreams) : nullptr;
  const void *dp = io.in(pcm, pcm_bytes);
  int32_t *ds = io.in(state, st_len);
  uint8_t *dr = io.out<uint8_t>((size_t)nstreams * nsteps);
  if (io.rc) return io.rc;
  if ((rc = envelope_search_launch(c, nstreams, dp, fmt, stride, first_step, nsteps, ds, dr, c->s_main, dn, nullptr)))
    return rc;
  io.back(state, ds, st_len);
  io.back(ret, dr, (size_t)nstreams * nsteps);
  return io.sync();
}

extern "C" int vb200_envelope_search(vb200_ctx *c, int nstreams, const void *pcm, int fmt, int64_t stride,
                                     int first_step, int nsteps, int32_t *state, uint8_t *ret) {
  return envelope_search_host(c, nstreams, pcm, fmt, stride, first_step, nsteps, state, ret, nullptr);
}

// streams with different amounts of new data in one call: stream s analyses its first steps_per_stream[s]
// (<= nsteps) steps, its later ret entries are left untouched
extern "C" int vb200_envelope_search_var(vb200_ctx *c, int nstreams, const void *pcm, int fmt, int64_t stride,
                                         int nsteps, const int32_t *steps_per_stream, int32_t *state, uint8_t *ret) {
  if (!steps_per_stream) return fail(VB200_EINVAL, "steps_per_stream");
  return envelope_search_host(c, nstreams, pcm, fmt, stride, 0, nsteps, state, ret, steps_per_stream);
}

// lib/envelope.c:254-264, replayed on the host from the per-step trigger bits (plain C, no CUDA)
extern "C" void vb200_envelope_apply_marks(const uint8_t *ret, int first_step, int nsteps, int32_t *mark) {
  for (int k = 0; k < nsteps; k++) {
    const int j = first_step + k;
    mark[j + 2] = 0;                                    // VE_POST
    if (ret[k] & 1) { mark[j] = 1; mark[j + 1] = 1; }
    if (ret[k] & 2) { mark[j] = 1; if (j > 0) mark[j - 1] = 1; }
  }
}

// ======================================================================== //
// Ogg files in: the page demux (vb200_ogg.cuh) and the reference's tabulated windows
static_assert(sizeof(vb200_ogg_stream) == 72 && offsetof(vb200_ogg_stream, hdr_offset) == 32 &&
              offsetof(vb200_ogg_stream, hdr_bytes) == 56, "vb200_ogg_stream layout (OGG_STREAM_DTYPE in abi.py)");
extern "C" int vb200_ogg_demux_dev(int nfiles, const uint8_t *d_bytes, const int64_t *d_file_off, int max_packets,
                                   vb200_packet_info *d_info, int32_t *d_npkt, uint8_t *d_data,
                                   vb200_ogg_stream *d_streams, void *stream) {
  if (nfiles < 0 || max_packets < 1) return fail(VB200_EINVAL, "ogg_demux: nfiles < 0 or max_packets < 1");
  if (nfiles == 0) return 0;
  if (!d_bytes || !d_file_off || !d_info || !d_npkt || !d_data || !d_streams)
    return fail(VB200_EINVAL, "ogg_demux: null pointer");
  const int grid = (nfiles + OGG_WARPS - 1) / OGG_WARPS;
  k_ogg_demux<<<grid, 32 * OGG_WARPS, 0, (cudaStream_t)stream>>>(nfiles, d_bytes, d_file_off, max_packets, d_info,
                                                                  d_npkt, d_data, d_streams);
  CU(cudaGetLastError());
  return 0;
}

extern "C" int vb200_ogg_demux(int nfiles, const uint8_t *bytes, const int64_t *file_off, int max_packets,
                               vb200_packet_info *info, int32_t *npkt, uint8_t *data, vb200_ogg_stream *streams) {
  if (nfiles < 0 || max_packets < 1) return fail(VB200_EINVAL, "ogg_demux: nfiles < 0 or max_packets < 1");
  if (nfiles == 0) return 0;
  if (!file_off || !info || !npkt || !streams) return fail(VB200_EINVAL, "ogg_demux: null pointer");
  if (file_off[0] < 0) return fail(VB200_EINVAL, "ogg_demux: file_off[0] < 0");
  for (int f = 0; f < nfiles; f++)
    if (file_off[f + 1] < file_off[f]) return fail(VB200_EINVAL, "ogg_demux: file_off decreases");
  const size_t total = (size_t)file_off[nfiles];
  if (total && (!bytes || !data)) return fail(VB200_EINVAL, "ogg_demux: null pointer");
  const size_t n_info = (size_t)nfiles * max_packets;
  DevBuf buf;                                             // freed on return
  uint8_t *db, *dd;
  int64_t *doff;
  vb200_packet_info *dinfo;
  int32_t *dn;
  vb200_ogg_stream *ds;
  int rc = carve(buf, [&](Carve &c) {
    db = c.take<uint8_t>(total); doff = c.take<int64_t>(nfiles + 1); dinfo = c.take<vb200_packet_info>(n_info);
    dn = c.take<int32_t>(nfiles); dd = c.take<uint8_t>(total); ds = c.take<vb200_ogg_stream>(nfiles);
  });
  if (rc) return rc;
  if (total) CU(cudaMemcpy(db, bytes, total, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(doff, file_off, sizeof(int64_t) * (nfiles + 1), cudaMemcpyHostToDevice));
  if (total) CU(cudaMemset(dd, 0, total));
  if ((rc = vb200_ogg_demux_dev(nfiles, db, doff, max_packets, dinfo, dn, dd, ds, nullptr))) return rc;
  CU(cudaMemcpy(npkt, dn, sizeof(int32_t) * nfiles, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(streams, ds, sizeof(vb200_ogg_stream) * nfiles, cudaMemcpyDeviceToHost));
  std::vector<vb200_packet_info> rows(n_info);
  CU(cudaMemcpy(rows.data(), dinfo, sizeof(vb200_packet_info) * n_info, cudaMemcpyDeviceToHost));
  for (int f = 0; f < nfiles; f++)                        // entries past npkt[f] are not written
    memcpy(info + (size_t)f * max_packets, rows.data() + (size_t)f * max_packets, sizeof(vb200_packet_info) * npkt[f]);
  if (total) CU(cudaMemcpy(data, dd, total, cudaMemcpyDeviceToHost));
  return 0;
}

// the links of chained files (k_ogg_links_* in vb200_ogg.cuh)
extern "C" int vb200_ogg_links_dev(int nfiles, const uint8_t *d_bytes, const int64_t *d_file_off, int64_t *d_link_first,
                                   int64_t *d_link_off, int64_t link_cap, void *stream) {
  if (nfiles < 0 || link_cap < 0) return fail(VB200_EINVAL, "ogg_links: nfiles < 0 or link_cap < 0");
  if (!d_file_off || !d_link_first || (link_cap && !d_link_off)) return fail(VB200_EINVAL, "ogg_links: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (nfiles == 0) {
    CU(cudaMemsetAsync(d_link_first, 0, sizeof(int64_t), st));
    if (d_link_off) CU(cudaMemcpyAsync(d_link_off, d_file_off, sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  if (!d_bytes) return fail(VB200_EINVAL, "ogg_links: null pointer");
  long long *first = (long long *)d_link_first;
  const int grid = (nfiles + OGG_WARPS - 1) / OGG_WARPS;
  k_ogg_links_count<<<grid, 32 * OGG_WARPS, 0, st>>>(nfiles, d_bytes, d_file_off, first);
  k_ds_scan<<<1, 1024, 0, st>>>(nfiles, first);
  k_ogg_links_write<<<grid, 32 * OGG_WARPS, 0, st>>>(nfiles, d_bytes, d_file_off, first, d_link_off, link_cap);
  CU(cudaGetLastError());
  return 0;
}

extern "C" int vb200_ogg_links(int nfiles, const uint8_t *bytes, const int64_t *file_off, int64_t *link_first,
                               int64_t *link_off, int64_t link_cap) {
  if (nfiles < 0 || link_cap < 0) return fail(VB200_EINVAL, "ogg_links: nfiles < 0 or link_cap < 0");
  if (!file_off || !link_first || (link_cap && !link_off)) return fail(VB200_EINVAL, "ogg_links: null pointer");
  if (file_off[0] < 0) return fail(VB200_EINVAL, "ogg_links: file_off[0] < 0");
  for (int f = 0; f < nfiles; f++)
    if (file_off[f + 1] < file_off[f]) return fail(VB200_EINVAL, "ogg_links: file_off decreases");
  const size_t total = (size_t)file_off[nfiles];
  if (total && !bytes) return fail(VB200_EINVAL, "ogg_links: null pointer");
  link_first[0] = 0;
  if (nfiles == 0) {
    if (link_off) link_off[0] = file_off[0];
    return 0;
  }
  // every link after a file's first starts at a captured page of 27 bytes or more: the device table needs no more rows
  const int64_t cap = std::min<int64_t>(link_cap, nfiles + (int64_t)(total / 27));
  DevBuf buf;                                             // freed on return
  uint8_t *db;
  int64_t *doff, *dfirst, *dlinks;
  int rc = carve(buf, [&](Carve &c) {
    db = c.take<uint8_t>(total); doff = c.take<int64_t>(nfiles + 1); dfirst = c.take<int64_t>(nfiles + 1);
    dlinks = c.take<int64_t>((size_t)cap + 1);
  });
  if (rc) return rc;
  if (total) CU(cudaMemcpy(db, bytes, total, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(doff, file_off, sizeof(int64_t) * (nfiles + 1), cudaMemcpyHostToDevice));
  if ((rc = vb200_ogg_links_dev(nfiles, db, doff, dfirst, dlinks, cap, nullptr))) return rc;
  CU(cudaMemcpy(link_first, dfirst, sizeof(int64_t) * (nfiles + 1), cudaMemcpyDeviceToHost));
  const int64_t links = link_first[nfiles];
  if (links > link_cap) return fail(VB200_EINVAL, "ogg_links: link_cap below the link count");
  CU(cudaMemcpy(link_off, dlinks, sizeof(int64_t) * (links + 1), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int vb200_vorbis_window(int n, float *out) {
  if (n < 64 || n > 8192 || !pow2(n) || !out) return fail(VB200_EINVAL, "vorbis_window: n must be 64, 128, .. 8192");
  vbh::window(n, out);
  return 0;
}

// ======================================================================== //
// Ogg files grouped by setup (vb200_ogg_group.cuh) and the header packets to a decode description (vb200_headers.h)
static_assert(sizeof(vb200_file_group) == 12, "vb200_file_group layout (FILE_GROUP_DTYPE in abi.py)");
static_assert(offsetof(vb200_vorbis_headers, setup) == 32 &&
              offsetof(vb200_vorbis_headers, entropy) == 32 + sizeof(vb200_setup),
              "vb200_vorbis_headers layout (abi.VorbisHeaders)");

// the scratch of one grouping call, in the order k_ogg_group_* use it; base = nullptr: sizes only
static size_t ogg_group_layout(int nfiles, char *base, OggGroupScratch *sc) {
  Carve c{base, 0};
  const uint32_t slots = ogg_group_slots(nfiles);
  sc->hash = c.take<unsigned long long>(nfiles);
  sc->rep = c.take<int32_t>(nfiles);
  sc->cnt = c.take<int32_t>(nfiles);
  sc->first = c.take<int32_t>(nfiles);
  sc->run = c.take<int32_t>(nfiles);
  sc->tkey = c.take<unsigned long long>(slots);
  sc->tmin = c.take<int32_t>(slots);
  sc->slots = slots;
  return c.off;
}

extern "C" size_t vb200_ogg_group_scratch_bytes(int nfiles, int max_packets) {
  (void)max_packets;
  OggGroupScratch sc;
  return ogg_group_layout(nfiles < 0 ? 0 : nfiles, nullptr, &sc);
}

extern "C" int vb200_ogg_group_dev(int nfiles, const uint8_t *d_data, const vb200_ogg_stream *d_streams,
                                   int max_packets, const int32_t *d_npkt, const vb200_packet_info *d_info,
                                   int32_t *d_status, int32_t *d_order, int32_t *d_npkt_out,
                                   vb200_packet_info *d_info_out, vb200_file_group *d_groups, int32_t *d_ngroups,
                                   void *d_scratch, size_t scratch_bytes, void *stream) {
  if (nfiles < 0 || max_packets < 1) return fail(VB200_EINVAL, "ogg_group: nfiles < 0 or max_packets < 1");
  if (!d_ngroups) return fail(VB200_EINVAL, "ogg_group: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (nfiles == 0) { CU(cudaMemsetAsync(d_ngroups, 0, sizeof(int32_t), s)); return 0; }
  if (!d_data || !d_streams || !d_npkt || !d_info || !d_status || !d_order || !d_npkt_out || !d_info_out ||
      !d_groups || !d_scratch)
    return fail(VB200_EINVAL, "ogg_group: null pointer");
  if (((uintptr_t)d_info | (uintptr_t)d_info_out) & 15) return fail(VB200_EINVAL, "ogg_group: info not 16-byte aligned");
  if ((uintptr_t)d_scratch & 7) return fail(VB200_EINVAL, "ogg_group: scratch not 8-byte aligned");
  OggGroupScratch sc;
  if (scratch_bytes < ogg_group_layout(nfiles, nullptr, &sc)) return fail(VB200_EINVAL, "ogg_group: scratch too small");
  ogg_group_layout(nfiles, (char *)d_scratch, &sc);
  const int wgrid = (nfiles + OGG_GROUP_WARPS - 1) / OGG_GROUP_WARPS;
  k_ogg_group_key<<<wgrid, 32 * OGG_GROUP_WARPS, 0, s>>>(nfiles, d_data, d_streams, d_status, sc);
  k_ogg_group_insert<<<(nfiles + 255) / 256, 256, 0, s>>>(nfiles, d_status, sc);
  k_ogg_group_rep<<<wgrid, 32 * OGG_GROUP_WARPS, 0, s>>>(nfiles, d_data, d_streams, d_status, sc);
  k_ogg_group_order<<<1, OGG_GROUP_ORDER_THREADS, 0, s>>>(nfiles, d_status, d_order, d_groups, d_ngroups, sc);
  k_ogg_group_gather<<<wgrid, 32 * OGG_GROUP_WARPS, 0, s>>>(nfiles, max_packets, d_order, d_npkt, d_info, d_npkt_out,
                                                            d_info_out);
  CU(cudaGetLastError());
  return 0;
}

extern "C" int vb200_ogg_group(int nfiles, const uint8_t *data, int64_t data_bytes, const vb200_ogg_stream *streams,
                               int max_packets, const int32_t *npkt, const vb200_packet_info *info, int32_t *status,
                               int32_t *order, int32_t *npkt_out, vb200_packet_info *info_out,
                               vb200_file_group *groups, int32_t *ngroups) {
  if (nfiles < 0 || max_packets < 1 || data_bytes < 0) return fail(VB200_EINVAL, "ogg_group: bad sizes");
  if (!ngroups) return fail(VB200_EINVAL, "ogg_group: null pointer");
  *ngroups = 0;
  if (nfiles == 0) return 0;
  if (!streams || !npkt || !info || !status || !order || !npkt_out || !info_out || !groups || (data_bytes && !data))
    return fail(VB200_EINVAL, "ogg_group: null pointer");
  for (int f = 0; f < nfiles; f++) {
    if (npkt[f] < 0 || npkt[f] > max_packets) return fail(VB200_EINVAL, "ogg_group: npkt outside 0..max_packets");
    if (streams[f].status != 0 && streams[f].status != VB200_EINVAL) continue;
    for (int k = 0; k < 3; k++)
      if (streams[f].hdr_offset[k] < 0 || streams[f].hdr_bytes[k] < 0 ||
          streams[f].hdr_offset[k] + streams[f].hdr_bytes[k] > data_bytes)
        return fail(VB200_EINVAL, "ogg_group: a header packet outside data");
  }
  const size_t n_info = (size_t)nfiles * max_packets;
  const size_t sbytes = vb200_ogg_group_scratch_bytes(nfiles, max_packets);
  DevBuf buf;                                             // freed on return
  uint8_t *dd; vb200_ogg_stream *ds; int32_t *dn, *dst, *dord, *dno, *dng; vb200_packet_info *di, *dio;
  vb200_file_group *dg; char *dscr;
  int rc = carve(buf, [&](Carve &c) {
    dd = c.take<uint8_t>((size_t)data_bytes); ds = c.take<vb200_ogg_stream>(nfiles); dn = c.take<int32_t>(nfiles);
    di = c.take<vb200_packet_info>(n_info); dst = c.take<int32_t>(nfiles); dord = c.take<int32_t>(nfiles);
    dno = c.take<int32_t>(nfiles); dio = c.take<vb200_packet_info>(n_info); dg = c.take<vb200_file_group>(nfiles);
    dng = c.take<int32_t>(1); dscr = c.take<char>(sbytes);
  });
  if (rc) return rc;
  if (data_bytes) CU(cudaMemcpy(dd, data, (size_t)data_bytes, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(ds, streams, sizeof(vb200_ogg_stream) * nfiles, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(dn, npkt, sizeof(int32_t) * nfiles, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(di, info, sizeof(vb200_packet_info) * n_info, cudaMemcpyHostToDevice));
  if ((rc = vb200_ogg_group_dev(nfiles, dd, ds, max_packets, dn, di, dst, dord, dno, dio, dg, dng, dscr, sbytes,
                                nullptr)))
    return rc;
  CU(cudaMemcpy(status, dst, sizeof(int32_t) * nfiles, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(order, dord, sizeof(int32_t) * nfiles, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(npkt_out, dno, sizeof(int32_t) * nfiles, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(ngroups, dng, sizeof(int32_t), cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(groups, dg, sizeof(vb200_file_group) * *ngroups, cudaMemcpyDeviceToHost));
  std::vector<vb200_packet_info> rows(n_info);
  CU(cudaMemcpy(rows.data(), dio, sizeof(vb200_packet_info) * n_info, cudaMemcpyDeviceToHost));
  for (int p = 0; p < nfiles; p++)                        // rows past npkt_out[p] are not written
    memcpy(info_out + (size_t)p * max_packets, rows.data() + (size_t)p * max_packets,
           sizeof(vb200_packet_info) * npkt_out[p]);
  return 0;
}

// ======================================================================== //
// Ogg files out: the page mux (vb200_ogg_mux.cuh)
static_assert(sizeof(vb200_ogg_mux_carry) == 24 && offsetof(vb200_ogg_mux_carry, kept_segs) == 16,
              "vb200_ogg_mux_carry layout (OGG_MUX_CARRY_DTYPE in abi.py)");
extern "C" int vb200_ogg_mux_dev(int nstreams, const uint8_t *d_data, int64_t data_bytes, const vb200_packet_info *d_hdr,
                                 int max_packets, const int32_t *d_npkt, const vb200_packet_info *d_info,
                                 vb200_ogg_mux_carry *d_carry, uint8_t *d_out, int64_t out_cap, int64_t *d_out_off,
                                 int32_t *d_status, void *stream) {
  if (nstreams < 0 || max_packets < 1 || data_bytes < 0 || out_cap < 0)
    return fail(VB200_EINVAL, "ogg_mux: nstreams < 0, max_packets < 1 or a negative size");
  if (!d_out_off) return fail(VB200_EINVAL, "ogg_mux: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (nstreams == 0) { CU(cudaMemsetAsync(d_out_off, 0, sizeof(int64_t), st)); return 0; }
  if (!d_npkt || !d_info || !d_carry || !d_status || (data_bytes && !d_data) || (out_cap && !d_out))
    return fail(VB200_EINVAL, "ogg_mux: null pointer");
  OggMuxArgs A{nstreams, d_data, data_bytes, d_hdr, max_packets, d_npkt, d_info, d_carry, d_out, out_cap,
               (long long *)d_out_off, d_status};
  const int grid = (nstreams + OGG_MUX_WARPS - 1) / OGG_MUX_WARPS;
  k_ogg_mux_count<<<grid, 32 * OGG_MUX_WARPS, 0, st>>>(A);
  k_ds_scan<<<1, 1024, 0, st>>>(nstreams, A.out_off);
  k_ogg_mux_write<<<grid, 32 * OGG_MUX_WARPS, 0, st>>>(A);
  CU(cudaGetLastError());
  return 0;
}

extern "C" int vb200_ogg_mux(int nstreams, const uint8_t *data, int64_t data_bytes, const vb200_packet_info *hdr,
                             int max_packets, const int32_t *npkt, const vb200_packet_info *info,
                             vb200_ogg_mux_carry *carry, uint8_t *out, int64_t out_cap, int64_t *out_off,
                             int32_t *status) {
  if (nstreams < 0 || max_packets < 1 || data_bytes < 0 || out_cap < 0)
    return fail(VB200_EINVAL, "ogg_mux: nstreams < 0, max_packets < 1 or a negative size");
  if (!out_off) return fail(VB200_EINVAL, "ogg_mux: null pointer");
  out_off[0] = 0;
  if (nstreams == 0) return 0;
  if (!npkt || !info || !carry || !status || (data_bytes && !data) || (out_cap && !out))
    return fail(VB200_EINVAL, "ogg_mux: null pointer");
  const size_t n_info = (size_t)nstreams * max_packets;
  DevBuf buf;                                             // freed on return
  uint8_t *dd, *dout;
  vb200_packet_info *dh, *di;
  int32_t *dn, *dst;
  vb200_ogg_mux_carry *dc;
  int64_t *doff;
  int rc = carve(buf, [&](Carve &c) {
    dd = c.take<uint8_t>((size_t)data_bytes); dh = c.take<vb200_packet_info>(hdr ? (size_t)nstreams * 3 : 0);
    dn = c.take<int32_t>(nstreams); di = c.take<vb200_packet_info>(n_info); dc = c.take<vb200_ogg_mux_carry>(nstreams);
    dout = c.take<uint8_t>((size_t)out_cap); doff = c.take<int64_t>(nstreams + 1); dst = c.take<int32_t>(nstreams);
  });
  if (rc) return rc;
  if (data_bytes) CU(cudaMemcpy(dd, data, (size_t)data_bytes, cudaMemcpyHostToDevice));
  if (hdr) CU(cudaMemcpy(dh, hdr, sizeof(vb200_packet_info) * nstreams * 3, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(dn, npkt, sizeof(int32_t) * nstreams, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(di, info, sizeof(vb200_packet_info) * n_info, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(dc, carry, sizeof(vb200_ogg_mux_carry) * nstreams, cudaMemcpyHostToDevice));
  if ((rc = vb200_ogg_mux_dev(nstreams, dd, data_bytes, hdr ? dh : nullptr, max_packets, dn, di, dc,
                              out_cap ? dout : nullptr, out_cap, doff, dst, nullptr)))
    return rc;
  CU(cudaMemcpy(out_off, doff, sizeof(int64_t) * (nstreams + 1), cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(status, dst, sizeof(int32_t) * nstreams, cudaMemcpyDeviceToHost));
  if (out_off[nstreams] > out_cap) return fail(VB200_EINVAL, "ogg_mux: out_cap below the pages' bytes");
  if (out_off[nstreams]) CU(cudaMemcpy(out, dout, (size_t)out_off[nstreams], cudaMemcpyDeviceToHost));
  for (int s = 0; s < nstreams; s++)
    if (status[s]) return fail(VB200_EINVAL, "ogg_mux: a stream's rows or carry are invalid (see status)");
  CU(cudaMemcpy(carry, dc, sizeof(vb200_ogg_mux_carry) * nstreams, cudaMemcpyDeviceToHost));
  return 0;
}

// ======================================================================== //
// device memory helpers
extern "C" int vb200_malloc_device(vb200_ctx *c, size_t bytes, void **dptr) {
  CHECK_CTX(c);
  CU(cudaMalloc(dptr, bytes ? bytes : 1));
  return 0;
}
extern "C" int vb200_free_device(vb200_ctx *c, void *dptr) { CHECK_CTX(c); CU(cudaFree(dptr)); return 0; }
extern "C" int vb200_memcpy_h2d(vb200_ctx *c, void *dptr, const void *src, size_t bytes) {
  CHECK_CTX(c); CU(cudaMemcpy(dptr, src, bytes, cudaMemcpyHostToDevice)); return 0;
}
extern "C" int vb200_memcpy_d2h(vb200_ctx *c, void *dst, const void *dptr, size_t bytes) {
  CHECK_CTX(c); CU(cudaMemcpy(dst, dptr, bytes, cudaMemcpyDeviceToHost)); return 0;
}
extern "C" int vb200_synchronize(vb200_ctx *c) { CHECK_CTX(c); CU(cudaDeviceSynchronize()); return 0; }
