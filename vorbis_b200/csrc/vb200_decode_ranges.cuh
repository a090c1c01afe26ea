// vb200_decode_ranges.cuh — sample ranges of many streams from packets (vb200_decode_ranges[_dev]): for each request
// r, samples [start, start + length) of what vb200_decode_streams_packets returns for its stream from a fresh carry,
// decoding only the blocks that finish those samples plus the one block before them that primes the overlap.
//
//   k_dr_plan    one warp per request, walking its stream's packets from packet 0 to the range's end: the header of
//                32 packets at a time (ds_packet_header, one per lane), then blockin's bookkeeping over them in order
//                (ds_blockin, the step of k_ds_plan), the compacted block tables k_decode_packets<true> reads and each
//                block's window, intersected with the range, with its offset in the request's output row
// then k_decode_packets<true> with requests as its streams and k_synthesis_range (vb200.cu).
//
// A block's finished samples depend on its own packet and on the previous decoded block's (the right half of its
// IMDCT and its flag); nothing else of the stream's past reaches them.  So block j0, the first whose returned
// samples meet the range, is decoded after block j0 - 1 alone, which primes as block 0 of a fresh decode does.
// j0 >= 1 always: the first decoded block of a stream returns nothing.
//
// Capacity.  A request's scratch is fixed from out_stride alone:
//   blocks   dr_blocks = (out_stride << hs) / (blocksizes[0]/2) + 3
//   residue  dr_residue = ch * (2 * (out_stride << hs) + 3 * blocksizes[1]/2) floats, rounded up to a multiple of
//            64 floats: request r's region starts at r * dr_residue, and every block's spectrum inside it is a multiple
//            of 32 floats, so each block starts on a 16-byte boundary as the synthesis' float4 loads need (an odd
//            channel count with an odd out_stride would otherwise put every other request 8 bytes off)
// The kept blocks are the priming block, the first and the last block that meet the range (the same block when
// one does) and the interior blocks between those two.  Every returned sample of an interior block lies inside
// the range.  An interior block that returns all it finishes returns F = (bs[lW]/4 + bs[W]/4) >> hs samples, so
//   - F << hs >= blocksizes[0]/2 (even quarters; bs[lW]/4 + bs[W]/4 >= 2 * blocksizes[0]/4): at most
//     (length << hs) / (blocksizes[0]/2) such blocks;
//   - its spectrum is ch * bs[W]/2 floats, and bs[W]/2 <= 2 * (bs[lW]/4 + bs[W]/4) = 2 * (F << hs): at most
//     ch * 2 * (length << hs) floats for all of them;
// and the three edge blocks take at most 3 * ch * blocksizes[1]/2 floats.  With length <= out_stride that is the
// bound above.  A trim or a packetno gap can make an interior block return fewer samples (a crafted stream can
// make it return none), which the bound does not cover: k_dr_plan checks every kept block against both
// capacities, writes nothing past them and reports such a request as got[r] = VB200_EINVAL with count 0, so its
// row stays zero.  A larger out_stride serves it.
#pragma once
#include <climits>
#include "vb200_decode_streams.cuh"

struct DrPlanArgs {
  int nstreams, max_packets, nreq, ch, hs, modebits;
  int bs[2];
  int out_stride;
  int nblk;                  // block slots per request (dr_blocks)
  long long res_cap;         // residue floats per request (dr_residue)
  const int *npkt;
  const vb200_packet_info *info;
  const unsigned char *data;
  const vb200_pcm_range *req;
  // outputs: the compacted block tables of request r at r*nblk + k (block 0 primes) ...
  int *Wseq, *pkt_bytes, *count;
  long long *pkt_off, *coef_off, *pcm_off;
  int2 *win;
  // ... and per request
  long long *base;           // [nreq + 1] r * out_stride: the output rows, as pcm_base of k_synthesis_trim
  int *got;
};

__global__ void __launch_bounds__(128)
k_dr_plan(DrPlanArgs A) {
  const int lane = threadIdx.x & 31;
  const int r = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (r >= A.nreq) return;                                 // warp-uniform
  const vb200_pcm_range q = A.req[r];
  if (lane == 0) {
    A.base[r] = (long long)r * A.out_stride;
    if (r == A.nreq - 1) A.base[r + 1] = (long long)A.nreq * A.out_stride;
  }
  long long got = 0;
  int keep = 0;                                            // blocks up to the last that meets the range
  if (q.stream < 0 || q.stream >= A.nstreams || q.start < 0 || q.length < 0 || q.length > A.out_stride) {
    got = VB200_EINVAL;
  } else if (q.length > 0) {
    const int st = q.stream, n = min(max(A.npkt[st], 0), A.max_packets);
    // t1 saturates: a start near INT64_MAX lies past every stream's end and gives got = 0
    const long long t0 = q.start, t1 = q.start > LLONG_MAX - q.length ? LLONG_MAX : q.start + q.length;
    const size_t row = (size_t)r * A.nblk;
    const long long res0 = (long long)r * A.res_cap;
    DsHead h;
    h.granulepos = -1; h.sample_count = -1; h.sequence = -1; h.W = -1; h.rate = 0;
    long long pos = 0;                                     // the stream's output before the current block
    long long coef = 0, coef_keep = 0;                     // residue floats of the blocks kept so far
    int nb = 0;                                            // blocks written (0 until the range is met)
    int pW = 0, pbytes = 0;                                // the last decoded block: the priming candidate
    long long poff = 0;
    bool done = false, over = false;
    // block k of the request: its tables, if it fits both capacities
    auto put = [&](int k, int W, long long off, int bytes, long long lo, long long hi, long long o) {
      const long long need = (long long)A.ch * (A.bs[W] / 2);
      if (lane == 0 && k < A.nblk && coef + need <= A.res_cap) {
        A.Wseq[row + k] = W;
        A.pkt_off[row + k] = off;
        A.pkt_bytes[row + k] = bytes;
        A.coef_off[row + k] = res0 + coef;
        A.pcm_off[row + k] = o;
        A.win[row + k] = make_int2((int)lo, (int)hi);
      }
      coef += need;
    };
    for (int k0 = 0; k0 < n && !done; k0 += 32) {
      const int k = k0 + lane;
      vb200_packet_info p{};
      int v = -135;
      if (k < n) {
        p = A.info[(size_t)st * A.max_packets + k];
        v = ds_packet_header(EntReader{A.data + p.offset, 8ll * (p.bytes > 0 ? p.bytes : 0), 0}, A.modebits);
      }
      const int m = min(32, n - k0);
      for (int i = 0; i < m; i++) {
        const int W = __shfl_sync(0xffffffffu, v, i);
        if (W < 0) continue;                               // dropped: nothing changes
        vb200_packet_info pi;
        pi.offset = __shfl_sync(0xffffffffu, p.offset, i);
        pi.granulepos = __shfl_sync(0xffffffffu, p.granulepos, i);
        pi.bytes = __shfl_sync(0xffffffffu, p.bytes, i);
        pi.e_o_s = __shfl_sync(0xffffffffu, p.e_o_s, i);
        pi.packetno = __shfl_sync(0xffffffffu, p.packetno, i);
        long long lo, hi;
        ds_blockin(h, W, pi, A.bs, A.hs, lo, hi);
        const long long ns = hi - lo;
        if (nb == 0) {
          if (ns == 0 || pos + ns <= t0) {                 // before the range: a priming candidate
            pW = W; poff = pi.offset; pbytes = pi.bytes;
            pos += ns;
            continue;
          }
          put(0, pW, poff, pbytes, 0, 0, 0);               // the block before primes
          nb = 1;
        }
        const long long a = max(pos, t0), b = min(pos + ns, t1);
        if (a < b) put(nb, W, pi.offset, pi.bytes, lo + (a - pos), lo + (b - pos), a - t0);
        else put(nb, W, pi.offset, pi.bytes, 0, 0, 0);
        nb++;
        if (a < b) {
          keep = nb; coef_keep = coef;
          if (keep > A.nblk || coef_keep > A.res_cap) { over = true; done = true; break; }
        }
        pos += ns;
        if (pos >= t1) { done = true; break; }
      }
    }
    got = over ? VB200_EINVAL : max(0ll, min(pos, t1) - t0);
    if (over) keep = 0;
  }
  if (lane == 0) {
    A.count[r] = keep;
    A.got[r] = (int)got;
  }
}
