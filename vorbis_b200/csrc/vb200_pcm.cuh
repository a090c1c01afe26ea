// vb200_pcm.cuh — the per-call bookkeeping of the raw-PCM packet calls (vb200_encode_pcm_packets[_managed][_dev]) on
// the device, so that the host and the _dev forms share it and a carry never has to be read on the host.
//
//   k_pcm_pack     one thread per stream: checks the stream's carry and write (vorbis_analysis_wrote's refusals) into
//                  status[s]; takes the write as the reference would (lib/block.c:480, :525: which preamble and tail
//                  filters are due, the timeline length and eof); fills the LPC jobs' fixed slots; and packs the
//                  encode carry into the CarryDev arrays the streams chain reads, with the envelope steps to analyse.
//                  A refused stream passes nothing: no jobs, no timeline, a done plan.
//   k_pcm_unpack   one thread per stream, unless the call's rc is nonzero: the new carry from the packed one, the new
//                  filters and the new head (raw_base, drained).
//   k_pcm_result   vb200_encode_result of a _dev call.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"
#include "vb200_streams.cuh"
#include "vb200_lpc.cuh"

namespace vb200 {

// The host carry of a raw-PCM stream starts with a PcmCarry, then the encode carry (PlanCarry, its mark window, the
// envelope state, a vb200_bitrate_state), then the filters of every channel (LPC_FILTER_FLOATS floats each).
struct PcmCarry {
  vb200_encode_carry enc;            // a copy of the encode carry's head, refreshed by every call (vb200_pcm_carry)
  long long raw_base, written;
  int ended, drained;
  int pre_done;                      // v->preextrapolate: the preamble filter has been made
  int ch, bs1, pad;
};

struct PcmPackArgs {
  unsigned char *carry;              // [nstreams][pb]
  long long pb, marks, env, br;      // the carry stride; where the mark window, envelope and bitrate state start
  int nstreams, ch, bs0, bs1, cap, managed, env_words;
  const int64_t *pcm_len, *first;    // first: null for the carries' raw_base
  const int32_t *end;                // or null
  long long in_stride, tl_stride;
  int nsteps;                        // envelope steps of a tl_stride timeline
  const void *in;                    // the caller's rows
  int s16;
  const float *tl;                   // the timelines, [nstreams][ch][tl_stride]
  PcmStream *ps;
  int64_t *tl_len, *eof;
  LpcJob *jobs;                      // [2][nstreams][ch]: the preamble jobs, then the tail jobs; n < 0: not due
  float *filt;                       // [nstreams][ch][LPC_FILTER_FLOATS]
  PcmCarry *head;                    // the updated heads; k_pcm_unpack completes them
  PlanCarry *pc;
  uint8_t *mk;
  int32_t *envs;
  vb200_bitrate_state *brs;
  int32_t *first_step, *count;       // the envelope steps each stream analyses
  int32_t *status;                   // [nstreams]
  int32_t *bad;                      // any nonzero status
};

__global__ void __launch_bounds__(128) k_pcm_pack(PcmPackArgs A) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= A.nstreams) return;
  const unsigned char *cs = A.carry + (size_t)s * A.pb, *ec = cs + sizeof(PcmCarry);
  PcmCarry p;
  PlanCarry q;
  memcpy(&p, cs, sizeof(p));
  memcpy(&q, ec, sizeof(q));
  const long long half = A.bs1 / 2, len = A.pcm_len[s];
  const long long first = A.first ? (long long)A.first[s] : p.raw_base;
  const bool end = A.end && A.end[s];
  const long long fresh = first + len - p.written;
  // the refusals of the host form's checks in pcm_packets (vb200.cu), which give them their messages: keep in step
  bool ok = p.ch == A.ch && p.bs1 == A.bs1 && q.ch == A.ch && q.bs0 == A.bs0 && q.bs1 == A.bs1 &&
            q.mark_cap == A.cap && (!A.managed || q.br_ready) && first >= 0 && first <= p.raw_base && fresh >= 0 &&
            len <= A.in_stride && !(p.ended && fresh) && !(end && p.ended) && !(end && fresh) && !(end && !p.drained);
  PcmStream t{};
  int pre_due = 0, tail_due = 0, first_step = 0, count = 0;
  if (ok) {
    p.written += fresh;
    pre_due = !p.pre_done && (p.written > A.bs1 || end);
    tail_due = end;
    p.pre_done |= pre_due;
    p.ended |= end;
    t.base = q.base; t.raw_base = first;
    t.eof = p.ended ? half + p.written : 0;
    t.len = q.done || !p.pre_done ? 0 : (p.ended ? t.eof + 3LL * A.bs1 : half + p.written) - q.base;
    if (!q.done) {
      // the checks and the steps of the carried streams path (vb200_encode_streams_packets_resume) on the timeline
      if (t.len < q.kept || t.len > A.tl_stride || (t.eof != 0 && t.eof <= q.base)) ok = false;
      long long last = t.len / PLAN_STEP - PLAN_VE_WIN;    // lib/envelope.c:224-225, as k_plan_blocks clamps it
      if (last > A.nsteps) last = A.nsteps;
      first_step = (int)(q.current / PLAN_STEP);
      count = last > first_step ? (int)(last - first_step) : 0;
    }
  }
  if (!ok) {
    t = PcmStream{};
    pre_due = tail_due = 0;
    q.done = 1;                                          // the planner passes the stream by
    first_step = count = 0;
    atomicOr(A.bad, 1);
  }
  A.status[s] = ok ? 0 : VB200_EINVAL;
  A.ps[s] = t;
  A.tl_len[s] = t.len; A.eof[s] = t.eof;
  A.head[s] = p;
  A.pc[s] = q;
  A.first_step[s] = first_step; A.count[s] = count;
  memcpy(A.mk + (size_t)s * A.cap, ec + A.marks, A.cap);
  memcpy(A.envs + (size_t)s * A.env_words, ec + A.env, sizeof(int32_t) * A.env_words);
  memcpy(&A.brs[s], ec + A.br, sizeof(vb200_bitrate_state));
  const long long nf = (long long)A.ch * LPC_FILTER_FLOATS;
  const float *cf = (const float *)(ec + A.br + sizeof(vb200_bitrate_state));
  for (long long i = 0; i < nf; i++) A.filt[s * nf + i] = cf[i];
  for (int k = 0; k < A.ch; k++) {
    const long long r = (long long)s * A.ch + k;
    for (int pass = 0; pass < 2; pass++) {
      LpcJob J{};
      float *f = A.filt + r * LPC_FILTER_FLOATS + (pass ? 2 * LPC_PRE : 0);
      J.coef = f; J.prime = f + (pass ? LPC_TAIL : LPC_PRE);
      J.n = -1;
      if (!pass && pre_due) {
        // _preextrapolate_helper: the input [0, P) time-reversed (raw_base, and so first, is 0 before the preamble)
        const long long P = p.written;
        J.src = A.in; J.s16 = A.s16; J.n = P;
        J.off = A.s16 ? ((long long)s * A.in_stride + P - 1 - first) * A.ch + k : r * A.in_stride + P - 1 - first;
        J.step = A.s16 ? -A.ch : -1;
      } else if (pass && tail_due) {
        // vorbis_analysis_wrote(v, 0): timeline [eof - n, eof), n = min(eof - base, blocksizes[1])
        const long long n = min(t.eof - t.base, (long long)A.bs1);
        J.src = A.tl; J.s16 = 0; J.n = n; J.off = r * A.tl_stride + t.eof - n - t.base; J.step = 1;
      }
      A.jobs[((long long)pass * A.nstreams + s) * A.ch + k] = J;
    }
  }
}

// rc: the call's vb200_encode_result rc, or null (a host form, which copies the carries back only when it succeeds)
__global__ void __launch_bounds__(128) k_pcm_unpack(PcmPackArgs A, const int32_t *__restrict__ nblocks, int max_blocks,
                                                    const int32_t *rc) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= A.nstreams || (rc && *rc)) return;
  unsigned char *cs = A.carry + (size_t)s * A.pb, *ec = cs + sizeof(PcmCarry);
  PcmCarry p = A.head[s];
  const PlanCarry &q = A.pc[s];
  memcpy(&p.enc, &q, sizeof(p.enc));
  p.raw_base = max(0LL, (long long)p.enc.base - A.bs1 / 2);
  p.drained = nblocks[s] < max_blocks;
  memcpy(cs, &p, sizeof(p));
  memcpy(ec, &q, sizeof(q));
  memcpy(ec + A.marks, A.mk + (size_t)s * A.cap, A.cap);
  memcpy(ec + A.env, A.envs + (size_t)s * A.env_words, sizeof(int32_t) * A.env_words);
  memcpy(ec + A.br, &A.brs[s], sizeof(vb200_bitrate_state));
  const long long nf = (long long)A.ch * LPC_FILTER_FLOATS;
  float *cf = (float *)(ec + A.br + sizeof(vb200_bitrate_state));
  for (long long i = 0; i < nf; i++) cf[i] = A.filt[s * nf + i];
}

// total: the byte total; tot: the plan's block totals (the _dev forms size their launches by cap[], so a plan past cap[]
// or a mark window overflow is only known here, and the bytes are then not known)
__global__ void k_pcm_result(vb200_encode_result *r, const long long *total, int64_t data_cap, const int32_t *tot,
                             int cap0, int cap1, const int32_t *overflow, const int32_t *bad) {
  if (threadIdx.x || blockIdx.x) return;
  const bool fits = tot[0] <= cap0 && tot[1] <= cap1 && !*overflow;
  const long long bytes = fits ? *total : 0;
  r->bytes = bytes;
  r->count[0] = tot[0]; r->count[1] = tot[1];
  r->rc = !fits || *bad || bytes > data_cap ? VB200_EINVAL : 0;
  r->pad = 0;
}

}  // namespace vb200
