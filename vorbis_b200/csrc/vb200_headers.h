// vb200_headers.h — the three Vorbis header packets to a decode description (vb200_vorbis_headers_parse).
//
// Plain host C++ (no CUDA): vb200.cu includes it, and a test compiles it alone with g++ and sanitizers.
// It restates the reference decoder's acceptance and tables: vorbis_synthesis_headerin ×3 (lib/info.c:211-450,
// the book unpack of lib/codebook.c:147-285, floor1_unpack, floor0_unpack, res0_unpack, mapping0_unpack) and the
// failure points of vorbis_synthesis_init, which are those of vorbis_book_init_decode (lib/sharedbook.c:393-519).
// Its output is what vorbis_b200/host/vb200_decode.c derives from a live decoder after those calls: vb200md_setup's
// vb200_setup and vb200md_entropy_new's vb200_entropy_setup.
#pragma once
#include <cmath>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <type_traits>
#include <utility>
#include <vector>

#include "vorbis_b200.h"

namespace vbh {

// The reader of libogg's oggpack_*: LSb first; a read past the end returns -1 and so does every read after it, and
// bytes() is then storage + 1.  Every check below that compares a count with storage - bytes() relies on that.
struct Reader {
  const uint8_t *p;
  long storage;
  long pos = 0;                 // bits consumed
  bool over = false;
  Reader(const uint8_t *d, long n) : p(d), storage(n) {}
  long read(int bits) {
    if (over) return -1;
    if (bits < 0 || bits > 32 || pos + bits > storage * 8) { over = true; return -1; }
    uint64_t v = 0;
    for (int got = 0; got < bits;) {
      const long at = (pos + got) >> 3;
      const int sh = (int)((pos + got) & 7), take = 8 - sh < bits - got ? 8 - sh : bits - got;
      v |= (uint64_t)((p[at] >> sh) & ((1u << take) - 1)) << got;
      got += take;
    }
    pos += bits;
    return (long)v;
  }
  void skip_bytes(long n) {     // n reads of 8 bits whose values are dropped (_v_readstring)
    if (over || n <= 0) return;
    if (n > storage || pos + 8 * n > storage * 8) { over = true; return; }
    pos += 8 * n;
  }
  long bytes() const { return over ? storage + 1 : (pos + 7) >> 3; }
};

// vb200_vorbis_window's table: the closed form in double, printed with "%.10f" and read back with strtof
inline void window(int n, float *out) {
  char txt[64];
  for (int i = 0; i < n / 2; i++) {
    const double s = sin((i + .5) / n * M_PI);
    snprintf(txt, sizeof(txt), "%.10f", sin(.5 * M_PI * (s * s)));
    out[i] = strtof(txt, nullptr);
  }
}

inline int ilog(uint32_t v) { int r = 0; while (v) { r++; v >>= 1; } return r; }
inline int popcount(uint32_t v) { int r = 0; while (v) { r += v & 1; v >>= 1; } return r; }
inline uint32_t bitrev(uint32_t x) {
  uint32_t r = 0;
  for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i);
  return r;
}

// The packed float of a book's minimum and delta: 21-bit mantissa, 10-bit exponent biased by 768 + 20, the
// exponent clamped to [-63, 63], evaluated as ldexp of a double and rounded to float once.
inline float unpack_float32(uint32_t v) {
  double mant = (double)(v & 0x1fffff);
  if (v & 0x80000000u) mant = -mant;
  long e = (long)((v & 0x7fe00000u) >> 21) - 20 - 768;
  e = e > 63 ? 63 : e < -63 ? -63 : e;
  return (float)ldexp(mant, (int)e);
}

// The largest v with v^dim <= entries, from the reference's float first guess and its integer walk.
inline long maptype1_quantvals(long dim, long entries) {
  if (entries < 1) return 0;
  long v = (long)floor(pow((double)(float)entries, (double)(1.f / dim)));
  if (v < 1) v = 1;
  for (;;) {
    long acc = 1, acc1 = 1;
    int i;
    for (i = 0; i < dim; i++) {
      if (entries / v < acc) break;
      acc *= v;
      acc1 = LONG_MAX / (v + 1) < acc1 ? LONG_MAX : acc1 * (v + 1);
    }
    if (i >= dim && acc <= entries && acc1 > entries) return v;
    if (i < dim || acc > entries) v--; else v++;
  }
}

struct Book {
  int dim = 0;                  // after the (signed char) cast
  int32_t entries = 0;
  bool ordered = false;
  std::vector<int8_t> len;      // unordered: per entry, 0 = unused
  int minlength = 0, maxlength = 0;
  int32_t cum[32] = {};         // ordered: entries of lengths minlength .. minlength + l, cumulative
  int maptype = 0, q_quant = 0, q_sequencep = 0;
  uint32_t q_min = 0, q_delta = 0;
  std::vector<uint16_t> quant;
};

struct Floor {
  int type = 0;
  vb200_floor_decode dec;       // floor 1: the decode fields, zeros where the unpack read nothing
  int posts = 0;
  int32_t postlist[VB200_VIF_POSIT + 2] = {};
  int mult = 0;
};

struct Residue {
  int type = 0;
  long begin = 0, end = 0;
  int grouping = 0, partitions = 0, groupbook = 0, partvals = 0;
  int secondstages[64] = {};
  int booklist[64 * 8] = {};
};

struct Mapping {
  int submaps = 1, coupling_steps = 0;
  int mag[256] = {}, ang[256] = {};
  int chmux[256] = {};
  int floorsubmap[16] = {}, residuesubmap[16] = {};
};

struct Mode { int blockflag, mapping; };

// what the returned vb200_vorbis_headers points to
struct Owned {
  vb200_vorbis_headers pub;     // first: the pointer handed out
  std::vector<float> window[2];
  std::vector<vb200_codebook> books;
  std::vector<uint8_t> length;
  std::vector<uint32_t> bits;
  std::vector<int32_t> entry;
  std::vector<float> value;
};
static_assert(std::is_standard_layout<Owned>::value, "Owned must start with its public struct");

// _vorbis_unpack_info after the packet type and magic
inline int unpack_info(Reader &r, vb200_vorbis_headers *h) {
  const int version = (int)r.read(32);
  if (version != 0) return VB200_EVERSION;
  const long channels = r.read(8), rate = r.read(32);
  h->bitrate_upper = (int32_t)r.read(32);
  h->bitrate_nominal = (int32_t)r.read(32);
  h->bitrate_lower = (int32_t)r.read(32);
  const long b0 = r.read(4);
  if (b0 < 0) return VB200_EBADHEADER;
  const long b1 = r.read(4);
  if (b1 < 0) return VB200_EBADHEADER;
  const long bs0 = 1L << b0, bs1 = 1L << b1;
  if (rate < 1 || channels < 1 || bs0 < 64 || bs1 < bs0 || bs1 > 8192) return VB200_EBADHEADER;
  if (r.read(1) != 1) return VB200_EBADHEADER;
  h->channels = (int32_t)channels;
  h->rate = (int32_t)rate;
  h->blocksizes[0] = (int32_t)bs0;
  h->blocksizes[1] = (int32_t)bs1;
  return 0;
}

// _vorbis_unpack_comment: validated only, nothing kept
inline int unpack_comment(Reader &r) {
  const int vendorlen = (int)r.read(32);
  if (vendorlen < 0 || vendorlen > r.storage - 8) return VB200_EBADHEADER;
  r.skip_bytes(vendorlen);
  const int n = (int)r.read(32);
  if (n < 0 || n > ((r.storage - r.bytes()) >> 2)) return VB200_EBADHEADER;
  for (int i = 0; i < n; i++) {
    const int len = (int)r.read(32);
    if (len < 0 || len > r.storage - r.bytes()) return VB200_EBADHEADER;
    r.skip_bytes(len);
  }
  return r.read(1) == 1 ? 0 : VB200_EBADHEADER;
}

// the book unpack: false where the reference fails it
inline bool unpack_book(Reader &r, Book &b) {
  if (r.read(24) != 0x564342) return false;
  b.dim = (signed char)r.read(16);
  b.entries = (int32_t)r.read(24);
  if (b.entries == -1) return false;
  if (ilog((uint32_t)b.dim) + ilog((uint32_t)b.entries) > 24) return false;
  switch ((int)r.read(1)) {
    case 0: {
      const long unused = r.read(1);
      if (((long)b.entries * (unused ? 1 : 5) + 7) >> 3 > r.storage - r.bytes()) return false;
      b.len.assign((size_t)b.entries, 0);
      for (long i = 0; i < b.entries; i++) {
        if (unused && !r.read(1)) continue;       // a read past the end here takes the "used" branch's -1 next
        const long num = r.read(5);
        if (num == -1) return false;
        b.len[i] = (int8_t)(num + 1);
      }
      break;
    }
    case 1: {
      b.ordered = true;
      long minlength = r.read(5) + 1, length = minlength, maxlength = minlength;
      if (minlength == 0) return false;
      for (long i = 0; i < b.entries; length++) {
        const long num = r.read(ilog((uint32_t)(b.entries - i)));
        if (num == -1) return false;
        if (length > 32 || num > b.entries - i || (num > 0 && ((num - 1) >> (length - 1)) > 1)) return false;
        i += num;
        b.cum[length - minlength] = (int32_t)i;
        if (i == 0) minlength++;                    // leading lengths without entries are skipped
        maxlength = length;
      }
      b.minlength = (signed char)minlength;
      b.maxlength = (signed char)maxlength;
      break;
    }
    default:
      return false;
  }
  b.maptype = (signed char)r.read(4);
  if (b.maptype == 0) return true;
  if (b.maptype != 1 && b.maptype != 2) return false;
  b.q_min = (uint32_t)r.read(32);
  b.q_delta = (uint32_t)r.read(32);
  b.q_quant = (signed char)r.read(4) + 1;
  b.q_sequencep = (signed char)r.read(1);
  if (b.q_sequencep == -1) return false;
  const int quantvals = b.maptype == 1 ? (b.dim == 0 ? 0 : (int)maptype1_quantvals(b.dim, b.entries))
                                       : b.entries * b.dim;
  if (((long)quantvals * b.q_quant + 7) >> 3 > r.storage - r.bytes()) return false;
  b.quant.resize(quantvals > 0 ? quantvals : 0);
  long q = 0;
  for (int i = 0; i < quantvals; i++) { q = r.read(b.q_quant); b.quant[i] = (uint16_t)q; }
  return q != -1;
}

// floor1_unpack
inline bool unpack_floor1(Reader &r, int nbooks, Floor &f) {
  vb200_floor_decode &d = f.dec;
  int maxclass = -1;
  d.type = 1;
  d.partitions = (int)r.read(5);
  for (int j = 0; j < d.partitions; j++) {
    d.partitionclass[j] = (int)r.read(4);
    if (d.partitionclass[j] < 0) return false;
    if (maxclass < d.partitionclass[j]) maxclass = d.partitionclass[j];
  }
  for (int j = 0; j < maxclass + 1; j++) {
    d.class_dim[j] = (int)r.read(3) + 1;
    d.class_subs[j] = (int)r.read(2);
    if (d.class_subs[j] < 0) return false;
    if (d.class_subs[j]) d.class_book[j] = (int)r.read(8);
    if (d.class_book[j] < 0 || d.class_book[j] >= nbooks) return false;
    for (int k = 0; k < (1 << d.class_subs[j]); k++) {
      d.class_subbook[j][k] = (int)r.read(8) - 1;
      if (d.class_subbook[j][k] < -1 || d.class_subbook[j][k] >= nbooks) return false;
    }
  }
  f.mult = (int)r.read(2) + 1;
  const int rangebits = (int)r.read(4);
  if (rangebits < 0) return false;
  int count = 0;
  for (int j = 0, k = 0; j < d.partitions; j++) {
    count += d.class_dim[d.partitionclass[j]];
    if (count > VB200_VIF_POSIT) return false;
    for (; k < count; k++) {
      const int t = f.postlist[k + 2] = (int)r.read(rangebits);
      if (t < 0 || t >= (1 << rangebits)) return false;
    }
  }
  f.postlist[0] = 0;
  f.postlist[1] = 1 << rangebits;
  f.posts = count + 2;
  for (int a = 0; a < f.posts; a++)                  // no repeated post positions
    for (int b = a + 1; b < f.posts; b++)
      if (f.postlist[a] == f.postlist[b]) return false;
  return true;
}

// floor0_unpack: only whether the reference takes it
inline bool unpack_floor0(Reader &r, const std::vector<Book> &books) {
  const long order = r.read(8), rate = r.read(16), barkmap = r.read(16);
  r.read(6);
  r.read(8);
  const long numbooks = r.read(4) + 1;
  if (order < 1 || rate < 1 || barkmap < 1 || numbooks < 1) return false;
  for (long j = 0; j < numbooks; j++) {
    const long b = r.read(8);
    if (b < 0 || b >= (long)books.size() || books[b].maptype == 0 || books[b].dim < 1) return false;
  }
  return true;
}

// res0_unpack (all three residue types)
inline bool unpack_residue(Reader &r, const std::vector<Book> &books, Residue &s) {
  s.begin = r.read(24);
  s.end = r.read(24);
  s.grouping = (int)r.read(24) + 1;
  s.partitions = (int)r.read(6) + 1;
  s.groupbook = (int)r.read(8);
  if (s.groupbook < 0) return false;
  int acc = 0;
  for (int j = 0; j < s.partitions; j++) {
    int cascade = (int)r.read(3);
    const long cflag = r.read(1);
    if (cflag < 0) return false;
    if (cflag) {
      const long c = r.read(5);
      if (c < 0) return false;
      cascade |= (int)(c << 3);
    }
    s.secondstages[j] = cascade;
    acc += popcount((uint32_t)cascade);
  }
  for (int j = 0; j < acc; j++) {
    s.booklist[j] = (int)r.read(8);
    if (s.booklist[j] < 0) return false;
  }
  const int nbooks = (int)books.size();
  if (s.groupbook >= nbooks) return false;
  for (int j = 0; j < acc; j++)
    if (s.booklist[j] >= nbooks || books[s.booklist[j]].maptype == 0) return false;
  const int entries = books[s.groupbook].entries;
  int dim = books[s.groupbook].dim, partvals = 1;
  if (dim < 1) return false;
  for (; dim > 0; dim--) {
    partvals *= s.partitions;
    if (partvals > entries) return false;
  }
  s.partvals = partvals;
  return true;
}

// mapping0_unpack
inline bool unpack_mapping(Reader &r, int channels, int floors, int residues, Mapping &m) {
  long b = r.read(1);
  if (b < 0) return false;
  if (b) {
    m.submaps = (int)r.read(4) + 1;
    if (m.submaps <= 0) return false;
  }
  b = r.read(1);
  if (b < 0) return false;
  if (b) {
    m.coupling_steps = (int)r.read(8) + 1;
    if (m.coupling_steps <= 0) return false;
    for (int i = 0; i < m.coupling_steps; i++) {
      const int M = m.mag[i] = (int)r.read(ilog((uint32_t)(channels - 1)));
      const int A = m.ang[i] = (int)r.read(ilog((uint32_t)(channels - 1)));
      if (M < 0 || A < 0 || M == A || M >= channels || A >= channels) return false;
    }
  }
  if (r.read(2) != 0) return false;
  if (m.submaps > 1)
    for (int i = 0; i < channels; i++) {
      m.chmux[i] = (int)r.read(4);
      if (m.chmux[i] >= m.submaps || m.chmux[i] < 0) return false;
    }
  for (int i = 0; i < m.submaps; i++) {
    r.read(8);
    m.floorsubmap[i] = (int)r.read(8);
    if (m.floorsubmap[i] >= floors || m.floorsubmap[i] < 0) return false;
    m.residuesubmap[i] = (int)r.read(8);
    if (m.residuesubmap[i] >= residues || m.residuesubmap[i] < 0) return false;
  }
  return true;
}

// The codewords of one book as the reference's decoder sees them, appended to o (length, stream bits, original
// entry, value row); *rows = how many.  False where vorbis_book_init_decode fails the book.  o = nullptr: only the
// check and the count, with no per-entry work for an ordered book.
inline bool book_codewords(const Book &b, Owned *o, long *rows) {
  *rows = 0;
  std::vector<std::pair<uint32_t, int32_t>> words;    // (codeword left-aligned in 32 bits, entry)
  std::vector<uint8_t> lens;
  if (!b.ordered) {
    // Canonical codewords in entry order, lowest value first: next[l] is the next free codeword of length l.
    // Taking one shifts the free codewords of every other length off the node it occupies.
    uint32_t next[33] = {};
    long used = 0;
    for (long i = 0; i < b.entries; i++) {
      const int l = b.len[i];
      if (l <= 0) continue;
      uint32_t w = next[l];
      if (l < 32 && (w >> l)) return false;            // over-populated
      words.push_back({l == 32 ? w : w << (32 - l), (int32_t)i});
      lens.push_back((uint8_t)l);
      used++;
      for (int j = l; j > 0; j--) {                    // the taken node's parents move on
        if (next[j] & 1) { next[j] = j == 1 ? next[1] + 1 : next[j - 1] << 1; break; }
        next[j]++;
      }
      for (int j = l + 1; j < 33; j++) {               // codewords that hung below the taken node move below the new one
        if ((next[j] >> 1) != w) break;
        w = next[j];
        next[j] = next[j - 1] << 1;
      }
    }
    if (used == 0) return true;                        // no codelist: vorbis_book_decode returns -1
    *rows = used;
    if (!(used == 1 && next[2] == 2))                  // under-populated, except the single-entry book
      for (int i = 1; i < 33; i++)
        if (next[i] & (0xffffffffu >> (32 - i))) return false;
  } else if (b.entries > 0) {
    const int nl = b.maxlength - b.minlength + 1;
    uint32_t code = 0, prev = 0;
    for (int l = 0; l < nl; l++) {
      const int length = b.minlength + l;
      const uint32_t n = (uint32_t)b.cum[l] - prev;
      if (l + 1 < nl && (unsigned long)n > ((0xffffffffUL - code) >> (32 - length))) return false;
      for (uint32_t e = prev; o && e < (uint32_t)b.cum[l]; e++) {
        words.push_back({code + ((e - prev) << (32 - length)), (int32_t)e});
        lens.push_back((uint8_t)length);
      }
      code += n << (32 - length);
      prev = (uint32_t)b.cum[l];
    }
    if (code - 1 != 0xffffffffu && !(b.entries == 1 && b.maxlength == 1)) return false;
    *rows = b.entries;
  } else {
    return true;
  }
  if (!o) return true;
  const bool values = b.maptype == 1 || b.maptype == 2;
  const float mindel = unpack_float32(b.q_min), delta = unpack_float32(b.q_delta);
  const long quantvals = b.maptype == 1 && b.dim > 0 ? maptype1_quantvals(b.dim, b.entries) : 0;
  for (size_t i = 0; i < words.size(); i++) {
    o->length.push_back(lens[i]);
    o->bits.push_back(bitrev(words[i].first));
    o->entry.push_back(words[i].second);
    if (!values) continue;
    const long j = words[i].second;
    float last = 0.f;
    long div = 1;
    for (int k = 0; k < b.dim; k++) {
      const float q = b.maptype == 1 ? (float)b.quant[(j / div) % quantvals] : (float)b.quant[j * b.dim + k];
      const float v = (float)(fabs((double)q) * delta + mindel + last);   // in double, rounded once
      if (b.q_sequencep) last = v;
      o->value.push_back(v);
      div *= quantvals;
    }
  }
  return true;
}

inline int check_magic(Reader &r, int type) {
  const long t = r.read(8);
  static const char magic[] = "vorbis";
  bool ok = true;
  for (int i = 0; i < 6; i++) ok = (char)r.read(8) == magic[i] && ok;
  if (!ok) return VB200_ENOTVORBIS;
  return t == type ? 0 : VB200_EBADHEADER;
}

inline int parse(const uint8_t *id, int32_t id_bytes, const uint8_t *comment, int32_t comment_bytes,
                 const uint8_t *setup, int32_t setup_bytes, Owned &o) {
  vb200_vorbis_headers *h = &o.pub;
  int rc;
  {
    Reader r(id, id_bytes);
    if ((rc = check_magic(r, 1)) || (rc = unpack_info(r, h))) return rc;
  }
  {
    Reader r(comment, comment_bytes);
    if ((rc = check_magic(r, 3)) || (rc = unpack_comment(r))) return rc;
  }
  Reader r(setup, setup_bytes);
  if ((rc = check_magic(r, 5))) return rc;
  const int ch = h->channels;
  std::vector<Book> books((size_t)(r.read(8) + 1));
  if (books.empty()) return VB200_EBADHEADER;
  for (Book &b : books)
    if (!unpack_book(r, b)) return VB200_EBADHEADER;
  const long times = r.read(6) + 1;
  if (times <= 0) return VB200_EBADHEADER;
  for (long i = 0; i < times; i++)
    if (r.read(16) != 0) return VB200_EBADHEADER;
  std::vector<Floor> floors((size_t)(r.read(6) + 1));
  if (floors.empty()) return VB200_EBADHEADER;
  for (Floor &f : floors) {
    memset(&f.dec, 0, sizeof(f.dec));
    f.type = (int)r.read(16);
    if (f.type == 1 ? !unpack_floor1(r, (int)books.size(), f) : f.type != 0 || !unpack_floor0(r, books))
      return VB200_EBADHEADER;
  }
  std::vector<Residue> residues((size_t)(r.read(6) + 1));
  if (residues.empty()) return VB200_EBADHEADER;
  for (Residue &s : residues) {
    s.type = (int)r.read(16);
    if (s.type < 0 || s.type > 2 || !unpack_residue(r, books, s)) return VB200_EBADHEADER;
  }
  std::vector<Mapping> maps((size_t)(r.read(6) + 1));
  if (maps.empty()) return VB200_EBADHEADER;
  for (Mapping &m : maps)
    if (r.read(16) != 0 || !unpack_mapping(r, ch, (int)floors.size(), (int)residues.size(), m))
      return VB200_EBADHEADER;
  std::vector<Mode> modes((size_t)(r.read(6) + 1));
  if (modes.empty()) return VB200_EBADHEADER;
  for (Mode &m : modes) {
    m.blockflag = (int)r.read(1);
    const long window = r.read(16), transform = r.read(16);
    m.mapping = (int)r.read(8);
    if (window >= 1 || transform >= 1 || m.mapping >= (int)maps.size() || m.mapping < 0) return VB200_EBADHEADER;
  }
  if (r.read(1) != 1) return VB200_EBADHEADER;
  // vorbis_synthesis_init: every book's decode tables, first checked and counted
  long rows = 0, values = 0;
  for (const Book &b : books) {
    long n;
    if (!book_codewords(b, nullptr, &n)) return VB200_EBADHEADER;
    rows += n;
    if (b.maptype == 1 || b.maptype == 2) values += n * (b.dim > 0 ? b.dim : 0);
  }
  // the reference takes the header set; what the output cannot describe
  if (rows > VB200_HEADERS_MAX_CODEWORDS || values > VB200_HEADERS_MAX_VALUES) return VB200_EIMPL;
  if (modes.size() != 2 || modes[0].blockflag != 0 || modes[1].blockflag != 1) return VB200_EIMPL;
  for (const Book &b : books)
    if (b.dim < 1 || b.dim > 127) return VB200_EIMPL;
  for (int w = 0; w < 2; w++) {
    const Mapping &m = maps[modes[w].mapping];
    if (m.submaps > VB200_MAX_SUBMAPS) return VB200_EIMPL;
    for (int j = 0; j < m.submaps; j++)
      if (floors[m.floorsubmap[j]].type != 1) return VB200_EIMPL;
  }
  std::vector<size_t> first(books.size() + 1), vfirst(books.size() + 1);
  o.length.reserve(rows); o.bits.reserve(rows); o.entry.reserve(rows); o.value.reserve(values);
  for (size_t i = 0; i < books.size(); i++) {
    long n;
    first[i] = o.length.size();
    vfirst[i] = o.value.size();
    book_codewords(books[i], &o, &n);
  }
  first[books.size()] = o.length.size();
  vfirst[books.size()] = o.value.size();
  // vb200md_setup's vb200_setup
  vb200_setup *s = &h->setup;
  s->channels = h->channels;
  s->rate = h->rate;
  s->blocksizes[0] = h->blocksizes[0];
  s->blocksizes[1] = h->blocksizes[1];
  for (int w = 0; w < 2; w++) {
    o.window[w].resize(h->blocksizes[w] / 2);
    window(h->blocksizes[w], o.window[w].data());
    s->window[w] = o.window[w].data();
    const Mapping &m = maps[modes[w].mapping];
    s->coupling_steps[w] = m.coupling_steps;
    for (int k = 0; k < m.coupling_steps; k++) { s->coupling_mag[w][k] = m.mag[k]; s->coupling_ang[w][k] = m.ang[k]; }
    s->submaps[w] = m.submaps;
    for (int c = 0; c < ch; c++) s->chmux[w][c] = (uint8_t)m.chmux[c];
    for (int j = 0; j < VB200_MAX_SUBMAPS; j++) s->residue[w][j].type = -1;
    for (int j = 0; j < m.submaps; j++) {
      const Floor &f = floors[m.floorsubmap[j]];
      const Residue &rs = residues[m.residuesubmap[j]];
      vb200_floor1_setup *fo = &s->floor1[w][j];
      fo->posts = f.posts;
      for (int k = 0; k < f.posts; k++) fo->postlist[k] = f.postlist[k];
      fo->mult = f.mult;
      fo->n = f.postlist[1];
      // vb200md_entropy_new's floor and residue decode fields
      h->entropy.floor[w][j] = f.dec;
      vb200_residue_decode *ro = &h->entropy.residue[w][j];
      ro->type = rs.type;
      ro->begin = (int32_t)rs.begin; ro->end = (int32_t)rs.end; ro->grouping = rs.grouping;
      ro->partitions = rs.partitions; ro->partvals = rs.partvals; ro->groupbook = rs.groupbook;
      for (int c = 0, acc = 0; c < 64; c++) {          // res0_look's layout of the stage books
        const int stages = c < rs.partitions ? ilog((uint32_t)rs.secondstages[c]) : 0;
        for (int k = 0; k < 8; k++)
          ro->stagebook[c][k] = k < stages && (rs.secondstages[c] & (1 << k)) ? rs.booklist[acc++] : -1;
      }
    }
  }
  h->entropy.nbooks = (int32_t)books.size();
  h->entropy.modebits = ilog((uint32_t)(modes.size() - 1));
  o.books.resize(books.size());
  for (size_t i = 0; i < books.size(); i++) {
    vb200_codebook *c = &o.books[i];
    const size_t n = first[i + 1] - first[i];
    c->dim = books[i].dim;
    c->used = (int32_t)n;
    c->length = o.length.data() + first[i];
    c->bits = o.bits.data() + first[i];
    c->entry = o.entry.data() + first[i];
    c->value = (books[i].maptype == 1 || books[i].maptype == 2) && n ? o.value.data() + vfirst[i] : nullptr;
  }
  h->entropy.books = o.books.data();
  return 0;
}

}  // namespace vbh

extern "C" int vb200_vorbis_headers_parse(const uint8_t *id, int32_t id_bytes, const uint8_t *comment,
                                          int32_t comment_bytes, const uint8_t *setup, int32_t setup_bytes,
                                          vb200_vorbis_headers **out) {
  if (!out || id_bytes < 0 || comment_bytes < 0 || setup_bytes < 0 || (id_bytes && !id) ||
      (comment_bytes && !comment) || (setup_bytes && !setup))
    return VB200_EINVAL;
  *out = nullptr;
  vbh::Owned *o = new (std::nothrow) vbh::Owned();
  if (!o) return VB200_EFAULT;
  memset(&o->pub, 0, sizeof(o->pub));
  int rc;
  try {
    rc = vbh::parse(id, id_bytes, comment, comment_bytes, setup, setup_bytes, *o);
  } catch (const std::bad_alloc &) {
    rc = VB200_EFAULT;
  }
  if (rc) { delete o; return rc; }
  *out = &o->pub;
  return 0;
}

extern "C" void vb200_vorbis_headers_free(vb200_vorbis_headers *h) {
  delete reinterpret_cast<vbh::Owned *>(h);
}
