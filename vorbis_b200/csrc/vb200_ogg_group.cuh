// vb200_ogg_group.cuh — Ogg files grouped by their identification and setup header bytes (vb200_ogg_group_dev).
//
// Five kernels, whatever nfiles and the number of groups:
//   k_ogg_group_key     one warp per file: the comment-header check of vorbis_synthesis_headerin (status), a 64-bit
//                       hash of (identification, setup) bytes; clears the hash table and the per-file counters
//   k_ogg_group_insert  one thread per grouped file: open addressing on the hash, the lowest file index per hash
//   k_ogg_group_rep     one warp per grouped file: rep = the lowest file whose header bytes are the same.  The
//                       table's candidate is compared byte for byte; when it differs (a hash collision) the warp scans
//                       the lower files with the same hash in order and compares each.  Counts the group sizes.
//   k_ogg_group_order   one block: scans in file order give each group its first position and number, then each
//                       file its rank inside its group (a chunk of 1024 files at a time, with running per-group counts)
//   k_ogg_group_gather  one warp per output position: npkt and the info rows of the file placed there
#pragma once
#include <climits>

#define OGG_GROUP_WARPS 8
#define OGG_GROUP_ORDER_THREADS 1024
// The bits of the 64-bit key hash that are kept.  A build with a narrow mask (tests/test_gpu_ogg_headers.py compiles
// one) makes hash collisions common, so that the byte comparison and the collision scan decide every group.
#ifndef VB200_OGG_GROUP_HASH_MASK
#define VB200_OGG_GROUP_HASH_MASK 0xffffffffffffffffULL
#endif

// a file with all three header packets and a comment header vorbis_synthesis_headerin takes: status 0, or
// VB200_EINVAL (max_packets cut its table, which holds the first max_packets audio packets)
__device__ __forceinline__ bool og_grouped(int status) { return status == 0 || status == VB200_EINVAL; }

struct OggGroupScratch {
  unsigned long long *hash;     // [nfiles] key hash, 0 where the file is not grouped
  int32_t *rep;                 // [nfiles] lowest file index with the same header bytes
  int32_t *cnt;                 // [nfiles] files in the group whose rep is this file
  int32_t *first;               // [nfiles] a rep's first output position; for a file left out its rank among
                                //          the files left out
  int32_t *run;                 // [nfiles] files of the group placed so far (k_ogg_group_order)
  unsigned long long *tkey;     // [slots] hash, 0 = empty
  int32_t *tmin;                // [slots] lowest file index inserted with that hash
  uint32_t slots;               // power of two >= 2 * nfiles
};

static inline uint32_t ogg_group_slots(int nfiles) {
  uint32_t s = 64;
  while (s < 2u * (uint32_t)nfiles) s <<= 1;
  return s;
}

__device__ __forceinline__ unsigned long long og_mix(unsigned long long x) {   // splitmix64's finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27; x *= 0x94d049bb133111ebULL;
  return x ^ (x >> 31);
}

// the warp's hash of bytes [p, p + n): lane-strided 8-byte words, each mixed with its word index and the salt, summed
__device__ unsigned long long og_warp_hash(const uint8_t *p, int n, unsigned long long salt, int lane) {
  unsigned long long h = 0;
  for (int w = lane; w * 8 < n; w += 32) {
    unsigned long long v = 0;
    const int at = w * 8, m = n - at < 8 ? n - at : 8;
    for (int b = 0; b < m; b++) v |= (unsigned long long)p[at + b] << (8 * b);
    h += og_mix(v ^ og_mix(salt + (unsigned long long)w));
  }
  for (int o = 16; o; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  return og_mix(h ^ (salt * 0x9e3779b97f4a7c15ULL) ^ (unsigned long long)n);
}

__device__ __forceinline__ int og_le32(const uint8_t *p) {
  return (int)((uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24);
}

// vorbis_synthesis_headerin on a comment packet (lib/info.c:247-275, 386-426).  Every field is byte aligned, and any
// read past the end makes a later check fail, so a byte position stands in for the bit reader.
__device__ bool og_comment_ok(const uint8_t *p, long n) {
  const char magic[7] = {3, 'v', 'o', 'r', 'b', 'i', 's'};
  if (n < 7) return false;
  for (int i = 0; i < 7; i++)
    if (p[i] != (uint8_t)magic[i]) return false;
  long at = 7;
  if (at + 4 > n) return false;
  const int vendorlen = og_le32(p + at);
  at += 4;
  if (vendorlen < 0 || vendorlen > n - 8 || at + vendorlen > n) return false;
  at += vendorlen;
  if (at + 4 > n) return false;
  const int count = og_le32(p + at);
  at += 4;
  if (count < 0 || count > ((n - at) >> 2)) return false;
  for (int i = 0; i < count; i++) {
    if (at + 4 > n) return false;
    const int len = og_le32(p + at);
    at += 4;
    if (len < 0 || len > n - at) return false;
    at += len;
  }
  return at < n && (p[at] & 1);                        // the end-of-packet bit
}

// the warp compares the header bytes of files a and b (identification and setup)
__device__ bool og_same(const uint8_t *data, const vb200_ogg_stream *st, int a, int b, int lane) {
  for (int k = 0; k < 3; k += 2) {
    const int n = st[a].hdr_bytes[k];
    if (n != st[b].hdr_bytes[k]) return false;
    const uint8_t *x = data + st[a].hdr_offset[k], *y = data + st[b].hdr_offset[k];
    for (int i = 0; i < n; i += 32) {
      const bool diff = i + lane < n && x[i + lane] != y[i + lane];
      if (__any_sync(0xffffffffu, diff)) return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(32 * OGG_GROUP_WARPS)
k_ogg_group_key(int nfiles, const uint8_t *__restrict__ data, const vb200_ogg_stream *__restrict__ st,
                int32_t *__restrict__ status, OggGroupScratch sc) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < sc.slots; i += gridDim.x * blockDim.x) {
    sc.tkey[i] = 0;
    sc.tmin[i] = INT_MAX;
  }
  const int f = blockIdx.x * OGG_GROUP_WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (f >= nfiles) return;
  int s = st[f].status;
  if (s == 0 || s == VB200_EINVAL) {
    bool ok = false;
    if (lane == 0) ok = og_comment_ok(data + st[f].hdr_offset[1], st[f].hdr_bytes[1]);
    if (!__shfl_sync(0xffffffffu, ok, 0)) s = VB200_EBADHEADER;
  }
  unsigned long long h = 0;
  if (og_grouped(s)) {
    const unsigned long long a = og_warp_hash(data + st[f].hdr_offset[0], st[f].hdr_bytes[0], 1, lane);
    const unsigned long long b = og_warp_hash(data + st[f].hdr_offset[2], st[f].hdr_bytes[2], 2, lane);
    h = og_mix(a * 0x9e3779b97f4a7c15ULL + b) & VB200_OGG_GROUP_HASH_MASK;
    if (!h) h = 1;
  }
  if (lane == 0) {
    status[f] = s;
    sc.hash[f] = h;
    sc.rep[f] = -1;
    sc.cnt[f] = 0;
    sc.run[f] = 0;
  }
}

__global__ void k_ogg_group_insert(int nfiles, const int32_t *__restrict__ status, OggGroupScratch sc) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nfiles || !og_grouped(status[f])) return;
  const unsigned long long h = sc.hash[f];
  for (uint32_t i = (uint32_t)h & (sc.slots - 1);; i = (i + 1) & (sc.slots - 1)) {
    const unsigned long long was = atomicCAS(&sc.tkey[i], 0ULL, h);
    if (was == 0 || was == h) { atomicMin(&sc.tmin[i], f); return; }
  }
}

__global__ void __launch_bounds__(32 * OGG_GROUP_WARPS)
k_ogg_group_rep(int nfiles, const uint8_t *__restrict__ data, const vb200_ogg_stream *__restrict__ st,
                const int32_t *__restrict__ status, OggGroupScratch sc) {
  const int f = blockIdx.x * OGG_GROUP_WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (f >= nfiles || !og_grouped(status[f])) return;
  const unsigned long long h = sc.hash[f];
  int g = f;
  if (lane == 0) {
    uint32_t i = (uint32_t)h & (sc.slots - 1);
    while (sc.tkey[i] != h) i = (i + 1) & (sc.slots - 1);
    g = sc.tmin[i];
  }
  g = __shfl_sync(0xffffffffu, g, 0);
  int rep = f;
  if (g != f) {
    if (og_same(data, st, f, g, lane)) {
      rep = g;
    } else {                                           // a hash collision: the lowest lower file with equal bytes
      for (int base = 0; base < f && rep == f; base += 32) {
        const int c = base + lane;
        unsigned m = __ballot_sync(0xffffffffu, c < f && og_grouped(status[c]) && sc.hash[c] == h);
        for (; m && rep == f; m &= m - 1) {
          const int cand = base + __ffs(m) - 1;
          if (og_same(data, st, f, cand, lane)) rep = cand;
        }
      }
    }
  }
  if (lane == 0) {
    sc.rep[f] = rep;
    atomicAdd(&sc.cnt[rep], 1);
  }
}

// exclusive block scan of v; *total gets the block's sum.  All threads of the block call it.
__device__ int og_block_exscan(int v, int *s_warp, int *total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();                                     // s_warp free from an earlier call
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nw ? s_warp[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    s_warp[lane] = w;                                  // inclusive over warps
  }
  __syncthreads();
  *total = s_warp[nw - 1];
  return x - v + (warp ? s_warp[warp - 1] : 0);
}

__global__ void __launch_bounds__(OGG_GROUP_ORDER_THREADS)
k_ogg_group_order(int nfiles, const int32_t *__restrict__ status, int32_t *__restrict__ order,
                  vb200_file_group *__restrict__ groups, int32_t *__restrict__ ngroups, OggGroupScratch sc) {
  __shared__ int s_warp[32];
  __shared__ int s_rep[OGG_GROUP_ORDER_THREADS];
  const int t = threadIdx.x, B = blockDim.x;
  int ngrp = 0, nused = 0, nrest = 0;
  // groups: first position and number of each rep, in file order; ranks of the files left out
  for (int base = 0; base < nfiles; base += B) {
    const int f = base + t;
    const bool in = f < nfiles, used = in && og_grouped(status[f]), isrep = used && sc.rep[f] == f;
    const int size = isrep ? sc.cnt[f] : 0;
    int tg, ts, tr;
    const int eg = og_block_exscan(isrep, s_warp, &tg);
    const int es = og_block_exscan(size, s_warp, &ts);
    const int er = og_block_exscan(in && !used, s_warp, &tr);
    if (isrep) {
      sc.first[f] = nused + es;
      groups[ngrp + eg] = vb200_file_group{nused + es, size, f};
    } else if (in && !used) {
      sc.first[f] = nrest + er;
    }
    ngrp += tg; nused += ts; nrest += tr;
  }
  if (t == 0) *ngroups = ngrp;
  __syncthreads();
  // positions: a group's first position + the files of the group before this one
  for (int base = 0; base < nfiles; base += B) {
    const int f = base + t;
    const bool in = f < nfiles, used = in && og_grouped(status[f]);
    const int r = used ? sc.rep[f] : -1;
    s_rep[t] = r;
    __syncthreads();
    int k = 0;
    bool last = used;
    if (used) {
      for (int u = 0; u < t; u++) k += s_rep[u] == r;
      for (int u = t + 1; u < B && last; u++) last = s_rep[u] != r;
      order[sc.first[r] + sc.run[r] + k] = f;
    } else if (in) {
      order[nused + sc.first[f]] = f;
    }
    __syncthreads();                                   // every file of the chunk has read run[]
    if (last) sc.run[r] += k + 1;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(32 * OGG_GROUP_WARPS)
k_ogg_group_gather(int nfiles, int max_packets, const int32_t *__restrict__ order, const int32_t *__restrict__ npkt,
                   const vb200_packet_info *__restrict__ info, int32_t *__restrict__ npkt_out,
                   vb200_packet_info *__restrict__ info_out) {
  static_assert(sizeof(vb200_packet_info) == 2 * sizeof(int4), "a packet row is two 16-byte words");
  const int p = blockIdx.x * OGG_GROUP_WARPS + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (p >= nfiles) return;
  const int f = order[p], m = npkt[f];
  if (lane == 0) npkt_out[p] = m;
  const int4 *src = (const int4 *)(info + (size_t)f * max_packets);
  int4 *dst = (int4 *)(info_out + (size_t)p * max_packets);
  for (int i = lane; i < 2 * m; i += 32) dst[i] = src[i];
}
