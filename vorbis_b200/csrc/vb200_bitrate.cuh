// vb200_bitrate.cuh — the bitrate manager's choice on the device, and whole streams' packets in stream order.
//
//  k_bitrate_choose   lib/bitrate.c:73-227   vorbis_bitrate_addblock replayed operation for operation: the
//                                            avg-reservoir slew search and slew limit (fp64, rint), the min and
//                                            max loops, truncation to maxsize bytes or zero padding up to minsize,
//                                            and both reservoir updates with the final size.  One thread per
//                                            stream, blocks in stream order (the state is a strict chain; its
//                                            exactness is the point, not its speed).
//  k_stream_bits      the per-size packet bit counts of vb200_encode_entropy[_managed]_dev (curve-major,
//                     k*count[W] + slot) gathered into stream order through the plan
//  k_stream_gather    every block's vb200_packet_info (granulepos, e_o_s, packetno as vorbis_analysis_blockout
//                     and vorbis_bitrate_flushpacket set them, lib/block.c:618-687, lib/bitrate.c:229-252) and the
//                     chosen packet's bytes copied from its strided slot, cut at the truncation point or followed
//                     by zero bytes of padding; k_stream_gather_carry the same for carried streams
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"
#include "vb200_streams.cuh"

namespace vb200 {

// what vorbis_bitrate_init derives from bitrate_manager_info and the codec setup (lib/bitrate.c:28-56)
struct BitrateDev {
  long long avg_bitsper, min_bitsper, max_bitsper;
  long long short_per_long;
  long long desired_fill;          // (long)(reservoir_bits * reservoir_bias)
  long long reservoir_bits;
  double slewlimit;                // 15. / slew_damp
  double rate;                     // vi->rate
  int samples[2];                  // blocksizes[W] >> 1
};

__device__ __forceinline__ long long br_bits(const int *__restrict__ pb, int k) {
  return (long long)((pb[k] + 7) >> 3) * 8;          // oggpack_bytes(packetblob[k]) * 8
}

// Stream s runs blocks 0 .. count[s]-1 of its row.  pkt_bits [nstreams][max_blocks][VB200_PACKETBLOBS]; state
// [nstreams] read and written in place, or nullptr: start from vorbis_bitrate_init's state and keep nothing.
// choice [nstreams][max_blocks] the packet kept; out [nstreams][max_blocks] its final length in bytes times
// out_scale (1: bytes; 8: bits, the input of k_packet_offsets).  W entries other than 0 read as 1.
__global__ void __launch_bounds__(128)
k_bitrate_choose(BitrateDev B, int nstreams, int max_blocks, const int32_t *__restrict__ count,
                 const int32_t *__restrict__ Wb, const int32_t *__restrict__ pkt_bits,
                 vb200_bitrate_state *__restrict__ state, int32_t *__restrict__ choice_out, int32_t *__restrict__ out,
                 int out_scale) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nstreams) return;
  long long avg_res = B.desired_fill, minmax_res = B.desired_fill;
  double avgfloat = VB200_PACKETBLOBS / 2;
  int last = 0;
  if (state) {
    avg_res = state[s].avg_reservoir; minmax_res = state[s].minmax_reservoir;
    avgfloat = state[s].avgfloat; last = state[s].choice;
  }
  const int nb = count[s];
  const size_t row = (size_t)s * max_blocks;
  for (int k = 0; k < nb; k++) {
    const int W = Wb[row + k] ? 1 : 0;
    const int *pb = pkt_bits + (row + k) * VB200_PACKETBLOBS;
    int choice = (int)rint(avgfloat);
    long long this_bits = br_bits(pb, choice);
    const long long min_target = W ? B.min_bitsper * B.short_per_long : B.min_bitsper;
    const long long max_target = W ? B.max_bitsper * B.short_per_long : B.max_bitsper;
    const int samples = W ? B.samples[1] : B.samples[0];   // (a dynamic index would put B on the stack)
    if (B.avg_bitsper > 0) {
      const long long avg_target = W ? B.avg_bitsper * B.short_per_long : B.avg_bitsper;
      if (avg_res + (this_bits - avg_target) > B.desired_fill) {
        while (choice > 0 && this_bits > avg_target && avg_res + (this_bits - avg_target) > B.desired_fill) {
          choice--;
          this_bits = br_bits(pb, choice);
        }
      } else if (avg_res + (this_bits - avg_target) < B.desired_fill) {
        while (choice + 1 < VB200_PACKETBLOBS && this_bits < avg_target &&
               avg_res + (this_bits - avg_target) < B.desired_fill) {
          choice++;
          this_bits = br_bits(pb, choice);
        }
      }
      double slew = rint((double)choice - avgfloat) / (double)samples * B.rate;
      if (slew < -B.slewlimit) slew = -B.slewlimit;
      if (slew > B.slewlimit) slew = B.slewlimit;
      avgfloat += slew / B.rate * (double)samples;
      choice = (int)rint(avgfloat);
      this_bits = br_bits(pb, choice);
    }
    if (B.min_bitsper > 0 && this_bits < min_target) {
      while (minmax_res - (min_target - this_bits) < 0) {
        choice++;
        if (choice >= VB200_PACKETBLOBS) break;
        this_bits = br_bits(pb, choice);
      }
    }
    if (B.max_bitsper > 0 && this_bits > max_target) {
      while (minmax_res + (this_bits - max_target) > B.reservoir_bits) {
        choice--;
        if (choice < 0) break;
        this_bits = br_bits(pb, choice);
      }
    }
    long long bytes;
    if (choice < 0) {
      // oggpack_writetrunc at a byte boundary keeps the first maxsize bytes (C's truncating division)
      long long maxsize = (max_target + (B.reservoir_bits - minmax_res)) / 8;
      if (maxsize < 0) maxsize = 0;
      choice = 0;
      bytes = (pb[0] + 7) >> 3;
      if (bytes > maxsize) bytes = maxsize;
    } else {
      long long minsize = (min_target - minmax_res + 7) / 8;
      if (choice >= VB200_PACKETBLOBS) choice = VB200_PACKETBLOBS - 1;
      bytes = (pb[choice] + 7) >> 3;
      minsize -= bytes;
      if (minsize > 0) bytes += minsize;                 // oggpack_write(0, 8) per missing byte
    }
    this_bits = bytes * 8;
    if (B.min_bitsper > 0 || B.max_bitsper > 0) {
      if (max_target > 0 && this_bits > max_target) {
        minmax_res += this_bits - max_target;
      } else if (min_target > 0 && this_bits < min_target) {
        minmax_res += this_bits - min_target;
      } else if (minmax_res > B.desired_fill) {
        if (max_target > 0) {
          minmax_res += this_bits - max_target;
          if (minmax_res < B.desired_fill) minmax_res = B.desired_fill;
        } else {
          minmax_res = B.desired_fill;
        }
      } else {
        if (min_target > 0) {
          minmax_res += this_bits - min_target;
          if (minmax_res > B.desired_fill) minmax_res = B.desired_fill;
        } else {
          minmax_res = B.desired_fill;
        }
      }
    }
    if (B.avg_bitsper > 0) avg_res += this_bits - (W ? B.avg_bitsper * B.short_per_long : B.avg_bitsper);
    choice_out[row + k] = choice;
    out[row + k] = (int32_t)(bytes * out_scale);
    last = choice;
  }
  if (state) {
    state[s].avg_reservoir = avg_res; state[s].minmax_reservoir = minmax_res;
    state[s].avgfloat = avgfloat; state[s].choice = last;
  }
}

// Block k of stream s (entry t = s*max_blocks + k): W[t] and, for every curve c, sbits[t*curves + c] =
// bits_W[c*count[W] + slot].  fbits[t] = 0 past nblocks[s]; with one curve (un-managed) fbits[t] is that packet's
// bit count, with VB200_PACKETBLOBS the chooser fills it.
__global__ void __launch_bounds__(256)
k_stream_bits(int nstreams, int max_blocks, const vb200_stream_block *__restrict__ plan,
              const int32_t *__restrict__ nblocks, int curves, const int32_t *__restrict__ bits0,
              const int32_t *__restrict__ bits1, int count0, int count1, int32_t *__restrict__ Wb,
              int32_t *__restrict__ sbits, int32_t *__restrict__ fbits) {
  const long long total = (long long)nstreams * max_blocks;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(t / max_blocks), k = (int)(t - (long long)s * max_blocks);
    if (k >= nblocks[s]) { fbits[t] = 0; continue; }
    const int W = plan[t].W, slot = plan[t].slot;
    const int32_t *b = W ? bits1 : bits0;
    const long long cnt = W ? count1 : count0;
    Wb[t] = W;
    for (int c = 0; c < curves; c++) sbits[t * curves + c] = b[c * cnt + slot];
    if (curves == 1) fbits[t] = b[slot];
  }
}

struct GatherArgs {
  const vb200_stream_block *plan;
  const int32_t *nblocks;
  const int64_t *eof;               // [nstreams] or nullptr
  int nstreams, max_blocks, curves;
  int bs[2];
  long long count[2], stride[2];
  const uint8_t *data[2];           // strided packets of each size: packet (c, slot) at (c*count + slot)*stride
  const int32_t *sbits;             // [t][curves] natural bit counts
  const int32_t *choice;            // [t] or nullptr (un-managed: curve 0, reported as VB200_PACKETBLOBS/2)
  const int32_t *fbits;             // [t] final length in bits (a whole number of bytes when managed)
  const long long *off;             // [t + 1] byte offsets (k_packet_offsets of fbits)
  long long cap;
  vb200_packet_info *info;
  uint8_t *dst;
};

// one CTA per block in a grid-stride loop; info is always written, the bytes only when all of them fit cap.
// CARRY: positions are relative to the call's buffer, which starts at timeline sample pc[s].base_in; packet numbers
// continue from pc[s].packetno_in, and the last block's granulepos goes to the carry.
template <bool CARRY>
__device__ __forceinline__ void stream_gather_body(const GatherArgs &A, PlanCarry *pc) {
  const long long total = (long long)A.nstreams * A.max_blocks;
  const bool fits = A.off[total] <= A.cap;
  for (long long t = blockIdx.x; t < total; t += gridDim.x) {
    const int s = (int)(t / A.max_blocks), k = (int)(t - (long long)s * A.max_blocks);
    const long long o = A.off[t];
    if (k >= A.nblocks[s]) {
      if (threadIdx.x == 0) {
        vb200_packet_info z;
        z.offset = o; z.granulepos = 0; z.bytes = 0; z.e_o_s = 0; z.packetno = 0; z.choice = 0;
        A.info[t] = z;
      }
      continue;
    }
    const vb200_stream_block b = A.plan[t];
    const int c = A.choice ? A.choice[t] : 0;
    const long long natural = (A.sbits[t * A.curves + (A.curves > 1 ? c : 0)] + 7) >> 3;
    const long long bytes = (A.fbits[t] + 7) >> 3;       // as k_packet_offsets counts it
    if (threadIdx.x == 0) {
      // vb->granulepos is v->granulepos when the block is cut: the sum of the moves so far (the block's centre
      // minus blocksizes[1]/2 on the timeline), clipped at the end of stream (lib/block.c:676-687)
      const long long centre = (CARRY ? pc[s].base_in : 0) + (long long)b.pos + A.bs[b.W] / 2, half1 = A.bs[1] / 2;
      const long long e = A.eof ? (long long)A.eof[s] : 0;
      long long g = centre - half1;
      if (e > 0 && g > e - half1) g = e - half1;
      vb200_packet_info in;
      in.offset = o; in.granulepos = g; in.bytes = (int32_t)bytes;
      in.e_o_s = (e > 0 && centre >= e) ? 1 : 0;       // lib/block.c:649-655
      in.packetno = (CARRY ? pc[s].packetno_in : 3) + k;  // v->sequence starts at 3 (lib/block.c:311)
      in.choice = A.choice ? c : VB200_PACKETBLOBS / 2;
      A.info[t] = in;
      if (CARRY && k == A.nblocks[s] - 1) pc[s].granulepos = g;
    }
    if (!fits) continue;
    const uint8_t *src = A.data[b.W] + ((long long)c * A.count[b.W] + b.slot) * A.stride[b.W];
    for (long long j = threadIdx.x; j < bytes; j += blockDim.x) A.dst[o + j] = j < natural ? src[j] : 0;
  }
}

__global__ void __launch_bounds__(256)
k_stream_gather(GatherArgs A) {
  stream_gather_body<false>(A, nullptr);
}

__global__ void __launch_bounds__(256)
k_stream_gather_carry(GatherArgs A, PlanCarry *pc) {
  stream_gather_body<true>(A, pc);
}

}  // namespace vb200
