// cuemu.h — a tiny CPU emulation of the CUDA execution model, enough to run the kernels of
// vorbis_b200/csrc/vb200.cu unmodified on host threads.
//
// DEVELOPMENT TOOL ONLY.  It exists so that kernel changes can be checked for logic / indexing
// errors against the oracle in this (GPU-less) container before a GPU box is spent on them.
// It is not part of the product: libvorbis_b200.so never contains or falls back to this code,
// nothing under vorbis_b200/ references it, and nothing measured or shipped runs through it.
// tools/cuemu/build_emu.py rewrites the `<<<...>>>` launches of a COPY of vb200.cu into
// cuemu::launch() calls and compiles that copy with g++ into tools/cuemu/_build/.
//
// Model: one CTA at a time; every CUDA thread of the CTA is an OS thread; __syncthreads and the
// warp collectives are futex barriers; `__shared__` statics are plain statics (one CTA runs at a
// time), dynamic shared memory is one buffer per launch; global memory is host memory.
#pragma once
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sched.h>
#include <thread>
#include <vector>

// ---- qualifiers ---------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __restrict__ __restrict
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static
#define __grid_constant__

// ---- vector types -------------------------------------------------------------------------
struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct alignas(8) float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(4) short2 { short x, y; };
struct alignas(8) short4 { short x, y, z, w; };
struct alignas(16) double2 { double x, y; };
static inline float2 make_float2(float a, float b) { return float2{a, b}; }
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
static inline int2 make_int2(int a, int b) { return int2{a, b}; }
static inline int4 make_int4(int a, int b, int c, int d) { return int4{a, b, c, d}; }
static inline uint2 make_uint2(unsigned a, unsigned b) { return uint2{a, b}; }
static inline short2 make_short2(short a, short b) { return short2{a, b}; }
static inline short4 make_short4(short a, short b, short c, short d) { return short4{a, b, c, d}; }

namespace cuemu {

// futex-backed barrier for a varying set of participants (all of them pass the same n)
struct Barrier {
  std::atomic<unsigned> count{0}, gen{0};
  void wait(unsigned n) {
    if (n <= 1) return;
    const unsigned g = gen.load(std::memory_order_acquire);
    if (count.fetch_add(1, std::memory_order_acq_rel) + 1 == n) {
      count.store(0, std::memory_order_relaxed);
      gen.fetch_add(1, std::memory_order_acq_rel);
      gen.notify_all();
    } else {
      while (gen.load(std::memory_order_acquire) == g) gen.wait(g, std::memory_order_acquire);
    }
  }
};

struct WarpSlot {                       // one collective context per distinct participation mask
  std::atomic<unsigned> mask{0};
  Barrier bar;
  uint64_t val[32];
};
struct Warp {
  WarpSlot slot[16];
  WarpSlot &get(unsigned mask) {
    for (;;) {
      for (auto &s : slot) {
        unsigned m = s.mask.load(std::memory_order_acquire);
        if (m == mask) return s;
        if (m == 0) {
          unsigned z = 0;
          if (s.mask.compare_exchange_strong(z, mask) || z == mask) return s;
        }
      }
      fprintf(stderr, "cuemu: more than 16 distinct warp masks in one warp\n");
      abort();
    }
  }
};

struct Cta {
  unsigned nthreads = 0;
  Barrier bar;                          // __syncthreads
  Barrier named[16];                    // bar.sync id, n
  std::vector<Warp> warps;
  unsigned char *smem = nullptr;
};

struct ThreadCtx {
  Cta *cta = nullptr;
  unsigned lane = 0, warp = 0;
};
extern thread_local ThreadCtx tctx;
extern int g_sm_count;

inline unsigned char *dyn_smem() { return tctx.cta->smem; }

template <class T>
inline T exchange(unsigned mask, T v, int src_lane, bool valid_src) {
  static_assert(sizeof(T) <= 8, "shuffle payload");
  WarpSlot &s = tctx.cta->warps[tctx.warp].get(mask);
  const unsigned n = (unsigned)__builtin_popcount(mask);
  uint64_t raw = 0;
  memcpy(&raw, &v, sizeof(T));
  s.val[tctx.lane] = raw;
  s.bar.wait(n);
  T out = v;
  if (valid_src && ((mask >> src_lane) & 1u)) { uint64_t r = s.val[src_lane]; memcpy(&out, &r, sizeof(T)); }
  s.bar.wait(n);
  return out;
}

template <class F>
void launch(dim3 grid, dim3 block, size_t smem_bytes, F body);

}  // namespace cuemu

extern thread_local uint3 threadIdx, blockIdx;
extern thread_local dim3 blockDim, gridDim;

// ---- synchronisation and warp collectives -------------------------------------------------
static inline void __syncthreads() { cuemu::tctx.cta->bar.wait(cuemu::tctx.cta->nthreads); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) {
  cuemu::WarpSlot &s = cuemu::tctx.cta->warps[cuemu::tctx.warp].get(mask);
  s.bar.wait((unsigned)__builtin_popcount(mask));
}
static inline void cuemu_named_barrier(int id, int nthreads) { cuemu::tctx.cta->named[id & 15].wait((unsigned)nthreads); }

template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  const int lane = (int)cuemu::tctx.lane;
  const int base = lane & ~(width - 1);
  return cuemu::exchange(mask, v, base + (src & (width - 1)), true);
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned d, int width = 32) {
  const int lane = (int)cuemu::tctx.lane;
  const int base = lane & ~(width - 1);
  const int src = lane - (int)d;
  return cuemu::exchange(mask, v, src, src >= base);
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned d, int width = 32) {
  const int lane = (int)cuemu::tctx.lane;
  const int base = lane & ~(width - 1);
  const int src = lane + (int)d;
  return cuemu::exchange(mask, v, src, src < base + width);
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int x, int width = 32) {
  const int lane = (int)cuemu::tctx.lane;
  const int src = lane ^ x;
  return cuemu::exchange(mask, v, src, (src & ~(width - 1)) == (lane & ~(width - 1)));
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
  cuemu::WarpSlot &s = cuemu::tctx.cta->warps[cuemu::tctx.warp].get(mask);
  const unsigned n = (unsigned)__builtin_popcount(mask);
  s.val[cuemu::tctx.lane] = pred ? 1u : 0u;
  s.bar.wait(n);
  unsigned r = 0;
  for (int l = 0; l < 32; l++) if (((mask >> l) & 1u) && s.val[l]) r |= 1u << l;
  s.bar.wait(n);
  return r;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) == mask; }
template <class T, class Op> static inline T cuemu_reduce(unsigned mask, T v, Op op) {
  cuemu::WarpSlot &s = cuemu::tctx.cta->warps[cuemu::tctx.warp].get(mask);
  const unsigned n = (unsigned)__builtin_popcount(mask);
  uint64_t raw = 0; memcpy(&raw, &v, sizeof(T));
  s.val[cuemu::tctx.lane] = raw;
  s.bar.wait(n);
  bool first = true; T acc = v;
  for (int l = 0; l < 32; l++) if ((mask >> l) & 1u) {
    T x; uint64_t r = s.val[l]; memcpy(&x, &r, sizeof(T));
    acc = first ? x : op(acc, x); first = false;
  }
  s.bar.wait(n);
  return acc;
}
static inline int __reduce_add_sync(unsigned m, int v) { return cuemu_reduce(m, v, [](int a, int b) { return a + b; }); }
static inline unsigned __reduce_add_sync(unsigned m, unsigned v) { return cuemu_reduce(m, v, [](unsigned a, unsigned b) { return a + b; }); }
static inline unsigned __reduce_or_sync(unsigned m, unsigned v) { return cuemu_reduce(m, v, [](unsigned a, unsigned b) { return a | b; }); }
static inline int __reduce_or_sync(unsigned m, int v) { return (int)__reduce_or_sync(m, (unsigned)v); }
static inline int __reduce_max_sync(unsigned m, int v) { return cuemu_reduce(m, v, [](int a, int b) { return a > b ? a : b; }); }
static inline int __reduce_min_sync(unsigned m, int v) { return cuemu_reduce(m, v, [](int a, int b) { return a < b ? a : b; }); }

// ---- memory helpers -----------------------------------------------------------------------
template <class T> static inline T __ldg(const T *p) { return *p; }
template <class T> static inline T __ldcs(const T *p) { return *p; }
template <class T> static inline T __ldcg(const T *p) { return *p; }
template <class T> static inline T __ldca(const T *p) { return *p; }
template <class T> static inline void __stcs(T *p, T v) { *p = v; }
template <class T> static inline void __stcg(T *p, T v) { *p = v; }
template <class T> static inline void __stwt(T *p, T v) { *p = v; }
static inline size_t __cvta_generic_to_shared(const void *p) { return (size_t)((const unsigned char *)p - (const unsigned char *)nullptr); }
template <class T> static inline T atomicAdd(T *p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int atomicAnd(int *p, int v) { return __atomic_fetch_and(p, v, __ATOMIC_RELAXED); }
static inline unsigned atomicOr(unsigned *p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
static inline int atomicOr(int *p, int v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
static inline int atomicMax(int *p, int v) { int o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o < v && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
static inline int atomicMin(int *p, int v) { int o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o > v && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
static inline unsigned long long atomicCAS(unsigned long long *p, unsigned long long cmp, unsigned long long v) { __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED); return cmp; }
static inline long long clock64() { return 0; }

// ---- arithmetic intrinsics ----------------------------------------------------------------
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline unsigned __float_as_uint(float f) { unsigned i; memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline float __uint_as_float(unsigned i) { float f; memcpy(&f, &i, 4); return f; }
static inline float __uint2float_rn(unsigned u) { return (float)u; }
static inline float __int2float_rn(int u) { return (float)u; }
static inline int __float2int_rz(float f) { return (int)f; }
static inline int __double2int_rz(double f) { return (int)f; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __clz(int v) { return v == 0 ? 32 : __builtin_clz((unsigned)v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline unsigned __brev(unsigned v) { unsigned r = 0; for (int i = 0; i < 32; i++) if (v >> i & 1u) r |= 1u << (31 - i); return r; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fdividef(float a, float b) { return a / b; }
static inline float __fsqrt_rn(float a) { return sqrtf(a); }
using std::max;
using std::min;

// ---- a minimal CUDA runtime (host memory is device memory) ---------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 };
typedef struct cuemu_stream *cudaStream_t;
typedef struct cuemu_event *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaEventDefault = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
struct cudaDeviceProp { int multiProcessorCount; char name[64]; size_t sharedMemPerBlockOptin; };
static inline const char *cudaGetErrorString(cudaError_t e) { return e ? "cuemu error" : "no error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
  memset(p, 0, sizeof(*p)); p->multiProcessorCount = cuemu::g_sm_count; strcpy(p->name, "cuemu"); p->sharedMemPerBlockOptin = 227 * 1024;
  return cudaSuccess;
}
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) { *p = (T *)aligned_alloc(256, (n + 255) & ~(size_t)255); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
template <class T> static inline cudaError_t cudaMallocHost(T **p, size_t n) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h,
                                            cudaMemcpyKind, cudaStream_t = nullptr) {
  for (size_t r = 0; r < h; r++) memmove((char *)d + r * dp, (const char *)s + r * sp, w);
  return cudaSuccess;
}
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t *s) { return cudaStreamCreateWithFlags(s, 0); }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = (cudaEvent_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { return cudaEventCreateWithFlags(e, 0); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
template <class K> static inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int) { return cudaSuccess; }
enum { cudaSharedmemCarveoutMaxShared = 100 };
template <class K> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, K, int, size_t) { *n = 1; return cudaSuccess; }

// ---- launch --------------------------------------------------------------------------------
namespace cuemu {
template <class F>
void launch(dim3 grid, dim3 block, size_t smem_bytes, F body) {
  const unsigned nt = block.x * block.y * block.z;
  const unsigned nctas = grid.x * grid.y * grid.z;
  if (nt == 0 || nctas == 0) return;
  Cta cta;
  cta.nthreads = nt;
  cta.warps = std::vector<Warp>((nt + 31) / 32);
  cta.smem = (unsigned char *)aligned_alloc(128, ((smem_bytes + 127) & ~(size_t)127) + 128);
  Barrier edge;
  std::vector<std::thread> th;
  th.reserve(nt);
  for (unsigned t = 0; t < nt; t++) {
    th.emplace_back([&, t]() {
      tctx.cta = &cta;
      tctx.lane = t & 31; tctx.warp = t >> 5;
      threadIdx = uint3{t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
      blockDim = block; gridDim = grid;
      for (unsigned b = 0; b < nctas; b++) {
        blockIdx = uint3{b % grid.x, (b / grid.x) % grid.y, b / (grid.x * grid.y)};
        body();
        edge.wait(nt);                  // the next CTA reuses the shared memory
      }
    });
  }
  for (auto &x : th) x.join();
  free(cta.smem);
}
}  // namespace cuemu
