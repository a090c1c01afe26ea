// vb200_entropy.cuh — the entropy half of mapping0_inverse (lib/mapping0.c:714-751) on the device.
//
// The bitstream of a packet is sequential, so one thread decodes one packet: the floor-1 fit values of every
// channel (floor1_inverse1, lib/floor1.c:955-1039), the nonzero propagation over the coupling steps, then the
// residue of every submap (types 1 and 2, lib/res0.c:651-711, 812-864) added into zeroed rows in the
// reference's order.  Parallelism comes from packets.
//
// Codewords are looked up in multi-level tables built by vb200_decode_entropy_setup: a table of 2^k entries is
// indexed by the next k stream bits (LSb first); an entry is either a leaf, (codeword << 6) | total length, or
// (bit 31) a sub-table, (offset << 5) | its k.  Every tree is complete (checked at setup), so every index of
// every table holds one or the other; each level consumes at least one bit, so a lookup takes at most 32 levels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vorbis_b200.h"

struct EntBook {
  int dim, used, k, pad;               // k: bits of the first-level table
  int tab_off, vec_off, ent_off, pad2;
};

struct EntFloor {                      // vb200_floor_decode, bounded at setup
  int partitions, qbits, quant_q, posts;
  unsigned char pclass[32], cdim[16], csubs[16];
  short cbook[16];
  short subbook[16][8];
};

struct EntRes {                        // vb200_residue_decode, bounded at setup; type -1 = nothing to decode
  int type, begin, end, grouping, partvals, groupbook, stages, ppw, partitions;
  short stagebook[64][8];
};

struct EntDev {
  const EntBook *books;
  const uint32_t *tab;
  const float *vec;
  const int *ent;
  const EntFloor *floor[2];            // [VB200_MAX_SUBMAPS] per block size
  const EntRes *res[2];
  const unsigned char *chmux[2];
  const int *mag[2], *ang[2];
  int steps[2], submaps[2], n[2];      // n: lines per channel (blocksize / 2)
  int ch, modebits, cls_cap;
};

// bit reader of lib/bitwise.c as oracle/shim/bitpack.c reads: a read of k bits succeeds only if k bits remain;
// a failed read returns -1 and leaves the reader exhausted (pos = nbits + 1), so every later read fails.
// Bytes are read only below nbits / 8.
struct EntReader {
  const unsigned char *p;
  long long nbits, pos;
  __device__ __forceinline__ uint32_t peek(long long at, int k) const {   // k <= 32 bits at `at`, zero past the end
    const long long byte = at >> 3, nbytes = nbits >> 3;
    const int sh = (int)(at & 7), need = (sh + k + 7) >> 3;
    unsigned long long acc = 0;
    for (int i = 0; i < need; i++)
      if (byte + i < nbytes) acc |= (unsigned long long)p[byte + i] << (8 * i);
    return (uint32_t)((acc >> sh) & ((1ull << k) - 1));
  }
  __device__ __forceinline__ int read(int k) {
    if (pos + k > nbits) { pos = nbits + 1; return -1; }
    const int v = (int)peek(pos, k);
    pos += k;
    return v;
  }
};

// decode_packed_entry_number for a complete tree: the codeword that is a prefix of the remaining bits, or -1
// (and the reader exhausted) when there is none.  Returns the codeword's index.
__device__ __forceinline__ int ent_codeword(const EntDev &E, const EntBook &B, EntReader &r) {
  if (r.pos > r.nbits) return -1;
  const uint32_t *tab = E.tab + B.tab_off;
  long long at = r.pos;
  int k = B.k;
  for (int level = 0; level < 32; level++) {
    const uint32_t e = tab[r.peek(at, k)];
    if (!(e & 0x80000000u)) {
      const int len = (int)(e & 63);
      if (r.pos + len > r.nbits) break;
      r.pos += len;
      return (int)(e >> 6);
    }
    if (r.nbits - at < k) break;
    at += k;
    tab = E.tab + B.tab_off + ((e >> 5) & 0x3ffffffu);
    k = (int)(e & 31);
  }
  r.pos = r.nbits + 1;
  return -1;
}

// vorbis_book_decode: the entry number or -1 (also for a book without a codelist, which reads nothing)
__device__ __forceinline__ int ent_book_decode(const EntDev &E, int book, EntReader &r) {
  const EntBook B = E.books[book];
  if (B.used == 0) return -1;
  const int cw = ent_codeword(E, B, r);
  return cw < 0 ? -1 : E.ent[B.ent_off + cw];
}

// vorbis_book_decodev_add (lib/codebook.c:428-443)
__device__ __forceinline__ int ent_decodev_add(const EntDev &E, int book, float *a, EntReader &r, int n) {
  const EntBook B = E.books[book];
  if (B.used == 0) return 0;
  for (int i = 0; i < n;) {
    const int cw = ent_codeword(E, B, r);
    if (cw < 0) return -1;
    const float *t = E.vec + B.vec_off + (size_t)cw * B.dim;
    for (int j = 0; i < n && j < B.dim;) a[i++] += t[j++];
  }
  return 0;
}

// vorbis_book_decodevv_add (lib/codebook.c:472-495): rows[] are the bundle's channels, each `stride` floats apart
__device__ __forceinline__ int ent_decodevv_add(const EntDev &E, int book, float *base, const unsigned char *rows,
                                                int stride, long offset, int ch, EntReader &r, int n) {
  const EntBook B = E.books[book];
  if (B.used == 0) return 0;
  int chptr = 0;
  const long m = (offset + n) / ch;
  for (long i = offset / ch; i < m;) {
    const int cw = ent_codeword(E, B, r);
    if (cw < 0) return -1;
    const float *t = E.vec + B.vec_off + (size_t)cw * B.dim;
    for (int j = 0; i < m && j < B.dim; j++) {
      base[(size_t)rows[chptr++] * stride + i] += t[j];
      if (chptr == ch) { chptr = 0; i++; }
    }
  }
  return 0;
}

// floor1_inverse1: true with fit[] filled (0x8000 on predicted posts), or false (the row is absent)
__device__ __forceinline__ bool ent_floor1(const EntDev &E, const EntFloor &F, const Floor1Dev &L, EntReader &r,
                                           int32_t *fit) {
  if (r.read(1) != 1) return false;
  fit[0] = r.read(F.qbits);
  fit[1] = r.read(F.qbits);
  for (int i = 0, j = 2; i < F.partitions; i++) {
    const int cls = F.pclass[i], cdim = F.cdim[cls], csubbits = F.csubs[cls], csub = 1 << csubbits;
    int cval = 0;
    if (csubbits) {
      cval = ent_book_decode(E, F.cbook[cls], r);
      if (cval == -1) return false;
    }
    for (int k = 0; k < cdim; k++) {
      const int book = F.subbook[cls][cval & (csub - 1)];
      cval >>= csubbits;
      if (book >= 0) {
        if ((fit[j + k] = ent_book_decode(E, book, r)) == -1) return false;
      } else {
        fit[j + k] = 0;
      }
    }
    j += cdim;
  }
  for (int i = 2; i < F.posts; i++) {
    const int ln = L.lo[i - 2], hn = L.hi[i - 2];
    int predicted;
    {                                                      // render_point, lib/floor1.c:362-374
      const int x0 = L.postlist[ln], x1 = L.postlist[hn], y0 = fit[ln] & 0x7fff, y1 = fit[hn] & 0x7fff;
      const int dy = y1 - y0, adx = x1 - x0, ady = abs(dy);
      const int off = ady * (L.postlist[i] - x0) / adx;
      predicted = dy < 0 ? y0 - off : y0 + off;
    }
    const int hiroom = F.quant_q - predicted, loroom = predicted;
    const int room = (hiroom < loroom ? hiroom : loroom) << 1;
    int val = fit[i];
    if (val) {
      if (val >= room) val = hiroom > loroom ? val - loroom : -1 - (val - hiroom);
      else val = (val & 1) ? -((val + 1) >> 1) : val >> 1;
      fit[i] = (val + predicted) & 0x7fff;
      fit[ln] &= 0x7fff;
      fit[hn] &= 0x7fff;
    } else {
      fit[i] = predicted | 0x8000;
    }
  }
  return true;
}

// the residue of one submap: `rows` lists the bundle's channels (type 1: the nonzero ones only), nrows of them.
// Partition classes go to cls (at most E.cls_cap bytes, checked at setup).  A failed read stops the submap.
__device__ __forceinline__ void ent_residue(const EntDev &E, const EntRes &R, float *base, int stride,
                                            const unsigned char *rows, int nrows, EntReader &r, unsigned char *cls) {
  const int two = R.type == 2;
  const int max = two ? stride * nrows : stride;        // (pcmend * ch) >> 1 for type 2, pcmend >> 1 for type 1
  const int end = R.end < max ? R.end : max, n = end - R.begin;
  if (n <= 0 || nrows == 0) return;
  const int spp = R.grouping, partvals = n / spp, ppw = R.ppw, per = two ? 1 : nrows;
  for (int s = 0; s < R.stages; s++) {
    for (int i = 0, l = 0; i < partvals; l++) {
      if (s == 0) {
        for (int j = 0; j < per; j++) {                    // the partition word of each channel (type 2: one)
          int temp = ent_book_decode(E, R.groupbook, r);
          if (temp == -1 || temp >= R.partvals) return;
          for (int k = ppw - 1; k >= 0; k--) {             // decodemap (lib/res0.c:300-311), last digit first
            const int at = l * ppw + k;
            if (at < partvals) cls[(size_t)j * partvals + at] = (unsigned char)(temp % R.partitions);
            temp /= R.partitions;
          }
        }
      }
      for (int k = 0; k < ppw && i < partvals; k++, i++) {
        if (two) {
          const int book = R.stagebook[cls[i]][s];
          if (book >= 0 && ent_decodevv_add(E, book, base, rows, stride, (long)i * spp + R.begin, nrows, r, spp) == -1)
            return;
        } else {
          for (int j = 0; j < nrows; j++) {
            const int book = R.stagebook[cls[(size_t)j * partvals + i]][s];
            if (book >= 0 &&
                ent_decodev_add(E, book, base + (size_t)rows[j] * stride + R.begin + (size_t)i * spp, r, spp) == -1)
              return;
          }
        }
      }
    }
  }
}

// One packet of block size W into zeroed rows: res [ch][n_W], posts [ch][VB200_FLOOR1_STRIDE] (zeroed),
// present [ch].  nz, rows: ch bytes each; cls: E.cls_cap bytes.  Run by one thread.
__device__ __noinline__ void ent_block(const EntDev &E, const Floor1Dev *__restrict__ floors, int W,
                                       const unsigned char *pkt, int bytes, float *res, int32_t *posts,
                                       int32_t *present, unsigned char *nz, unsigned char *rows, unsigned char *cls) {
  EntReader r{pkt, 8ll * (bytes > 0 ? bytes : 0), 1 + E.modebits + (W ? 2 : 0)};
  if (r.pos > r.nbits) r.pos = r.nbits + 1;
  const int ch = E.ch, n = E.n[W];
  const unsigned char *chmux = E.chmux[W];
  const EntFloor *fl = E.floor[W];
  for (int c = 0; c < ch; c++) {
    const int sm = chmux[c];
    int32_t *fit = posts + (size_t)c * VB200_FLOOR1_STRIDE;
    const bool ok = ent_floor1(E, fl[sm], floors[sm], r, fit);
    if (!ok) for (int j = 0; j < VB200_FLOOR1_STRIDE; j++) fit[j] = 0;
    present[c] = ok;
    nz[c] = ok;
  }
  for (int i = 0; i < E.steps[W]; i++) {
    const int m = E.mag[W][i], a = E.ang[W][i];
    if (nz[m] || nz[a]) nz[m] = nz[a] = 1;
  }
  for (int sm = 0; sm < E.submaps[W]; sm++) {
    const EntRes &R = E.res[W][sm];
    if (R.type < 0) continue;
    int nrows = 0, any = 0;
    for (int c = 0; c < ch; c++)
      if (chmux[c] == sm) {
        any |= nz[c];
        if (R.type == 2 || nz[c]) rows[nrows++] = (unsigned char)c;
      }
    if (R.type == 2 && !any) continue;
    ent_residue(E, R, res, n, rows, nrows, r, cls);
  }
}
