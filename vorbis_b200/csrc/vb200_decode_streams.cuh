// vb200_decode_streams.cuh — whole streams from packets (vb200_decode_streams_packets[_dev]): what a stock decoder's
// vorbis_synthesis -> vorbis_synthesis_blockin -> vorbis_synthesis_pcmout loop does around mapping0_inverse, on the
// device.
//
//   k_ds_header  one thread per packet slot: the packet header of vorbis_synthesis (lib/synthesis.c:41-71)
//   k_ds_plan    one thread per stream, walking its packets in order: the dropped packets, the compacted block
//                tables k_decode_packets<true> reads, and blockin's sample bookkeeping (lib/block.c:741-751,
//                835-941), which never reads a sample value: each block's returned window [lo, hi) of the samples
//                it finishes, its samples and granulepos
//   k_ds_scan    pcm_base, the prefix sums of the streams' returned samples
// then k_decode_packets<true> and k_synthesis_trim (vb200.cu), which writes only [lo, hi) of each block.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"
#include "vb200_entropy.cuh"

// The readable part of a stream's carry: the state of vorbis_dsp_state / private_state that blockin's bookkeeping
// keeps.  W = -1 after vorbis_synthesis_restart: no block since (pcm_returned == -1), and the synthesis primes.  The
// carry is DS_HEAD_BYTES of head, then the overlap tail of every channel (blocksizes[1]/2 floats each).
struct DsHead {
  long long granulepos;      // v->granulepos
  long long sample_count;    // b->sample_count
  long long sequence;        // v->sequence
  int W;                     // the last block's flag, -1 = nothing decoded since the restart
  int rate;                  // DS_RATE_FULL or DS_RATE_HALF: the mode the carry belongs to
};
constexpr int DS_HEAD_BYTES = 64;
constexpr int DS_RATE_FULL = 1, DS_RATE_HALF = 2;
static_assert(sizeof(DsHead) <= DS_HEAD_BYTES, "carry head");

// what k_synthesis_trim needs besides the arguments of k_synthesis_carry
struct DsTrim {
  const int2 *win;           // [nstreams][nblk] the returned window [lo, hi) of each block's finished samples
  const long long *base;     // [nstreams + 1] pcm_base
  const int *W_in;           // [nstreams] the carried flag k_ds_plan read (-1: block 0 primes)
  const DsHead *head;        // [nstreams] the heads after this call
  unsigned char *carry;      // [nstreams][carry_bytes]
  long long carry_bytes;
  long long cap;             // pcm_cap
  int tail_stride;           // blocksizes[1] / 2
  __device__ __forceinline__ float *tail(int st, int c) const {
    return reinterpret_cast<float *>(carry + (size_t)st * carry_bytes + DS_HEAD_BYTES) + (size_t)c * tail_stride;
  }
  __device__ __forceinline__ DsHead *carried(int st) const {
    return reinterpret_cast<DsHead *>(carry + (size_t)st * carry_bytes);
  }
};

// a finished-sample sink that keeps only [lo, hi), written from index 0
template <class B>
struct SinkTrim {
  B b;
  int lo, hi;
  __device__ __forceinline__ void put(int i, float v) const { if (i >= lo && i < hi) b.put(i - lo, v); }
};

// the packet header as vorbis_synthesis reads it: the block flag, or OV_ENOTAUDIO / OV_EBADPACKET.  Modes 0 and 1
// have block flags 0 and 1 (every vorbisenc setup); a higher mode number has no mode_param.  r: the packet's bits.
__device__ __forceinline__ int ds_packet_header(EntReader r, int modebits) {
  int v;
  if (r.read(1) != 0) v = -135;                            // OV_ENOTAUDIO, also for an empty packet
  else {
    const int mode = r.read(modebits);
    if (mode < 0 || mode > 1) v = -136;                    // OV_EBADPACKET
    else if (mode == 1) {
      r.read(1);                                           // lW: only the window selection reads it
      v = r.read(1) == -1 ? -136 : 1;                      // nW
    } else v = 0;
  }
  return v;
}

// one packet slot per thread; hdr of slots past npkt[s] is not written
__global__ void __launch_bounds__(256)
k_ds_header(int nstreams, int max_packets, int modebits, const int *__restrict__ npkt,
            const vb200_packet_info *__restrict__ info, const unsigned char *__restrict__ data, int *__restrict__ hdr) {
  const long long slot = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= (long long)nstreams * max_packets) return;
  const int st = (int)(slot / max_packets), k = (int)(slot - (long long)st * max_packets);
  if (k >= npkt[st]) return;
  const vb200_packet_info p = info[slot];
  hdr[slot] = ds_packet_header(EntReader{data + p.offset, 8ll * (p.bytes > 0 ? p.bytes : 0), 0}, modebits);
}

// blockin's bookkeeping for one packet that vorbis_synthesis accepted (block flag W): h advances, and [lo, hi) is
// the window of the block's finished samples that pcmout returns (lib/block.c:741-751, 835-941, >> hs at half rate).
// bs: blocksizes.  k_ds_plan runs the same step written out in its loop: called from there, this function changes
// that kernel's register allocation, so its SASS would not stay as it was; the index and ranges tests check that the
// two give the same windows.
__device__ __forceinline__ void ds_blockin(DsHead &h, int W, const vb200_packet_info &p, const int *bs, int hs,
                                           long long &lo_, long long &hi_) {
  const int lW = h.W;
  const long long fin = lW >= 0 ? (long long)((bs[lW] / 4 + bs[W] / 4) >> hs) : 0;
  if (h.sequence == -1 || h.sequence + 1 != (long long)p.packetno) { h.granulepos = -1; h.sample_count = -1; }
  h.sequence = p.packetno;
  long long lo = 0, hi = fin;                              // pcm_returned, pcm_current past prevCenter
  if (h.sample_count == -1) h.sample_count = 0;
  else h.sample_count += bs[lW] / 4 + bs[W] / 4;
  if (h.granulepos == -1) {
    if (p.granulepos != -1) {
      h.granulepos = p.granulepos;
      if (h.sample_count > h.granulepos) {
        long long extra = h.sample_count - p.granulepos;
        if (extra < 0) extra = 0;
        if (p.e_o_s) {                                     // trim the end
          if (extra > (hi - lo) << hs) extra = (hi - lo) << hs;
          hi -= extra >> hs;
        } else {                                           // trim the beginning
          lo += extra >> hs;
          if (lo > hi) lo = hi;
        }
      }
    }
  } else {
    h.granulepos += bs[lW] / 4 + bs[W] / 4;
    if (p.granulepos != -1 && h.granulepos != p.granulepos) {
      if (h.granulepos > p.granulepos) {
        long long extra = h.granulepos - p.granulepos;
        if (extra && p.e_o_s) {                            // partial last frame
          if (extra > (hi - lo) << hs) extra = (hi - lo) << hs;
          if (extra < 0) extra = 0;
          hi -= extra >> hs;
        }
      }
      h.granulepos = p.granulepos;
    }
  }
  h.W = W;
  lo_ = lo; hi_ = hi;
}

struct DsPlanArgs {
  int nstreams, max_packets, ch, hs;
  int bs[2];
  const int *npkt;
  const vb200_packet_info *info;
  const int *hdr;
  const unsigned char *carry;
  long long carry_bytes;
  // outputs: the compacted block tables (block j of stream s at s*max_packets + j) ...
  int *Wseq, *pkt_bytes, *count;
  long long *pkt_off, *coef_off, *pcm_off;
  int2 *win;
  // ... and per stream / per packet
  int *W_in;
  DsHead *head;
  long long *pcm_base;       // pcm_base[s + 1] = the stream's returned samples (k_ds_scan turns them into offsets)
  vb200_decoded_packet *out;
};

__global__ void __launch_bounds__(128)
k_ds_plan(DsPlanArgs A) {
  const int st = blockIdx.x * blockDim.x + threadIdx.x;
  if (st >= A.nstreams) return;
  DsHead h = *reinterpret_cast<const DsHead *>(A.carry + (size_t)st * A.carry_bytes);
  A.W_in[st] = h.W;
  const int n = A.npkt[st], hs = A.hs;
  const long long rows = (long long)A.ch * (A.bs[1] / 2);  // residue scratch per packet slot
  long long pos = 0;
  int j = 0;
  for (int k = 0; k < n; k++) {
    const size_t slot = (size_t)st * A.max_packets + k;
    const int v = A.hdr[slot];
    vb200_decoded_packet o;
    o.pcm_offset = pos;
    if (v < 0) {                                           // vorbis_synthesis failed: no blockin, nothing changes
      o.granulepos = h.granulepos; o.samples = 0; o.status = v;
      A.out[slot] = o;
      continue;
    }
    const vb200_packet_info p = A.info[slot];
    const int lW = h.W, W = v;
    const long long fin = lW >= 0 ? (long long)((A.bs[lW] / 4 + A.bs[W] / 4) >> hs) : 0;
    if (h.sequence == -1 || h.sequence + 1 != (long long)p.packetno) { h.granulepos = -1; h.sample_count = -1; }
    h.sequence = p.packetno;
    long long lo = 0, hi = fin;                            // pcm_returned, pcm_current past prevCenter
    if (h.sample_count == -1) h.sample_count = 0;
    else h.sample_count += A.bs[lW] / 4 + A.bs[W] / 4;
    if (h.granulepos == -1) {
      if (p.granulepos != -1) {
        h.granulepos = p.granulepos;
        if (h.sample_count > h.granulepos) {
          long long extra = h.sample_count - p.granulepos;
          if (extra < 0) extra = 0;
          if (p.e_o_s) {                                   // trim the end
            if (extra > (hi - lo) << hs) extra = (hi - lo) << hs;
            hi -= extra >> hs;
          } else {                                         // trim the beginning
            lo += extra >> hs;
            if (lo > hi) lo = hi;
          }
        }
      }
    } else {
      h.granulepos += A.bs[lW] / 4 + A.bs[W] / 4;
      if (p.granulepos != -1 && h.granulepos != p.granulepos) {
        if (h.granulepos > p.granulepos) {
          long long extra = h.granulepos - p.granulepos;
          if (extra && p.e_o_s) {                          // partial last frame
            if (extra > (hi - lo) << hs) extra = (hi - lo) << hs;
            if (extra < 0) extra = 0;
            hi -= extra >> hs;
          }
        }
        h.granulepos = p.granulepos;
      }
    }
    h.W = W;
    const size_t b = (size_t)st * A.max_packets + j;
    A.Wseq[b] = W;
    A.pkt_off[b] = p.offset;
    A.pkt_bytes[b] = p.bytes;
    A.coef_off[b] = (long long)b * rows;
    A.pcm_off[b] = pos;
    A.win[b] = make_int2((int)lo, (int)hi);
    o.granulepos = h.granulepos; o.samples = (int)(hi - lo); o.status = 0;
    A.out[slot] = o;
    pos += hi - lo;
    j++;
  }
  A.count[st] = j;
  A.head[st] = h;
  A.pcm_base[st + 1] = pos;
}

// pcm_base[0] = 0 and pcm_base[1 .. n] turned from counts into their inclusive prefix sums, one CTA
__global__ void __launch_bounds__(1024)
k_ds_scan(int n, long long *__restrict__ base) {
  __shared__ long long s_warp[32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int per = (n + 1023) / 1024, a = tid * per, b = min(n, a + per);
  long long sum = 0;
  for (int k = a; k < b; k++) sum += base[k + 1];
  long long inc = sum;
  for (int d = 1; d < 32; d <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += y; }
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  long long run = inc - sum;
  for (int k = 0; k < wid; k++) run += s_warp[k];
  for (int k = a; k < b; k++) { run += base[k + 1]; base[k + 1] = run; }
  if (tid == 0) base[0] = 0;
}
