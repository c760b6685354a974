// Shared device/host helpers: error reporting across the C ABI, the split-bf16 activation format,
// the counter-hash dropout generator, warp reductions.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace dsvg {

// ----------------------------------------------------------------------------------------------
// Error handling: no C++ exception crosses the ABI. Entry points return 0 or a non-zero code and leave a
// thread-local message that dsvg_last_error() hands to the host language.
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* last_error();

#define DSVG_CHECK(cond, ...)          \
  do {                                 \
    if (!(cond)) {                     \
      ::dsvg::set_error(__VA_ARGS__);  \
      return 1;                        \
    }                                  \
  } while (0)

#define DSVG_CUDA(expr)                                                                       \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::dsvg::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 2;                                                                               \
    }                                                                                         \
  } while (0)

#define DSVG_LAUNCH_CHECK() DSVG_CUDA(cudaGetLastError())

// ----------------------------------------------------------------------------------------------
// Activation format.  An activation tensor is one bf16 plane ("hi") in fast mode, or two planes in parity mode:
// plane 0 = hi = bf16(v), plane 1 = lo = bf16(v - hi), the second plane `lo_off` elements after the first.
// hi+lo carries ~16 mantissa bits, and the tensor-core GEMMs consume the planes as three products
// (hi*hi + hi*lo + lo*hi) -- "bf16x3".  lo_off == 0 means fast mode.
// ----------------------------------------------------------------------------------------------
using bf16 = __nv_bfloat16;

struct Act {
  bf16* p;
  size_t lo_off;  // 0 => single plane
};
struct CAct {
  const bf16* p;
  size_t lo_off;
};

__device__ __forceinline__ float act_load(const bf16* p, size_t lo_off, size_t i) {
  float v = __bfloat162float(p[i]);
  if (lo_off) v += __bfloat162float(p[i + lo_off]);
  return v;
}
__device__ __forceinline__ void act_store(bf16* p, size_t lo_off, size_t i, float v) {
  bf16 h = __float2bfloat16_rn(v);
  p[i] = h;
  if (lo_off) p[i + lo_off] = __float2bfloat16_rn(v - __bfloat162float(h));
}
// two adjacent elements (i even, pointers 4-byte aligned)
__device__ __forceinline__ float2 act_load2(const bf16* p, size_t lo_off, size_t i) {
  __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(p + i);
  float2 v = __bfloat1622float2(h);
  if (lo_off) {
    __nv_bfloat162 l = *reinterpret_cast<const __nv_bfloat162*>(p + i + lo_off);
    float2 w = __bfloat1622float2(l);
    v.x += w.x;
    v.y += w.y;
  }
  return v;
}
__device__ __forceinline__ void act_store2(bf16* p, size_t lo_off, size_t i, float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  *reinterpret_cast<__nv_bfloat162*>(p + i) = h;
  if (lo_off) {
    float2 hf = __bfloat1622float2(h);
    *reinterpret_cast<__nv_bfloat162*>(p + i + lo_off) = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  }
}

// ----------------------------------------------------------------------------------------------
// Dropout masks: stateless counter-based generator.  A dropout call site is (seed, site id).  Elements are numbered
// i = 0, 1, 2, ... inside the site's tensor; the four elements of "quad" q = i >> 2 share one first mixing stage
//     s = xs15( xs16( q * 0x9E3779B1 ^ key' ) * 0x7feb352d )           key' = key(seed, site) ^ (q >> 32) * 0x85EBCA77
// (the first half of the "lowbias32" integer finaliser) and two finalisers
//     a = xs16( s * 0x846ca68b )   -> elements 4q (low 16 bits) and 4q + 1 (high 16 bits)
//     b = xs16( s * 0xC2B2AE35 )   -> elements 4q + 2 and 4q + 3
// An element is kept iff its 16-bit draw >= thr16; survivors are scaled by the exact complement of thr16 / 65536.
// Cost: 13 integer instructions per four draws.  The masks are generated inside the GEMM epilogues, where every
// instruction counts: ncu showed the previous one-hash-per-two-elements version at 62 % of the FFN1 epilogue's
// instructions (and a Philox4x32-10 version before it at 2 k instructions per 32x32 chunk).  Marginal keep rates,
// pairwise joint rates inside a quad and at lags 1..1024, and byte histograms of the draws were checked against
// their binomial / chi-square expectations on 2^24 quads for several keys (tools/check_dropout_hash.py).
// The backward pass regenerates the same draws from (seed, site, index).
// ----------------------------------------------------------------------------------------------
struct Dropout {
  float p;             // requested drop probability; 0 disables
  uint32_t thr16;      // keep iff 16-bit draw >= thr16
  float scale;         // 1 / (1 - thr16 / 65536)
  uint32_t key;        // mixes seed and call-site id (host-computed, or resolved in the kernel from *seed_dev)
  const unsigned long long* seed_dev;  // non-null: the seed lives in device memory (CUDA-graph replays draw new masks)
  uint32_t site;
};
__host__ __device__ inline uint32_t host_mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__host__ __device__ inline uint32_t drop_key_of(unsigned long long seed, uint32_t site) {
  return host_mix32(uint32_t(seed) ^ host_mix32(uint32_t(seed >> 32) + 0x9E3779B9u * (site + 1u)));
}
// C ABI convention (include/dsvg_b200.h): bit 31 of `drop_site` set => `seed` is a DEVICE POINTER to the uint64 seed,
// read by the kernel at run time (so a captured CUDA graph draws fresh masks on every replay).
constexpr uint32_t kSeedIsDevicePtr = 0x80000000u;
inline Dropout make_dropout(float p, uint32_t site, unsigned long long seed) {
  Dropout d;
  d.p = p;
  double t = double(p) * 65536.0 + 0.5;
  d.thr16 = t >= 65535.0 ? 65535u : (t <= 0.0 ? 0u : uint32_t(t));
  d.scale = 1.f / (1.f - float(d.thr16) / 65536.f);
  d.site = site & ~kSeedIsDevicePtr;
  if (site & kSeedIsDevicePtr) {
    d.seed_dev = reinterpret_cast<const unsigned long long*>(static_cast<uintptr_t>(seed));
    d.key = 0;
  } else {
    d.seed_dev = nullptr;
    d.key = drop_key_of(seed, d.site);
  }
  return d;
}
// every kernel that draws dropout masks calls this once (after pdl_wait: the seed may be written by a preceding kernel)
__device__ __forceinline__ void drop_resolve(Dropout& d) {
  if (d.p > 0.f && d.seed_dev != nullptr) d.key = drop_key_of(__ldg(d.seed_dev), d.site);
}
// key' for a quad index (the high word is zero for every tensor below 2^34 elements, but stays part of the definition)
__device__ __forceinline__ uint32_t drop_hikey(const Dropout& d, unsigned long long quad) {
  return (uint32_t(quad >> 32) * 0x85EBCA77u) ^ d.key;
}
__device__ __forceinline__ uint32_t drop_stage1(uint32_t quad_lo, uint32_t hikey) {
  uint32_t x = (quad_lo * 0x9E3779B1u) ^ hikey;
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15;
  return x;
}
__device__ __forceinline__ uint32_t drop_fin_a(uint32_t s) { s *= 0x846ca68bu; return s ^ (s >> 16); }
__device__ __forceinline__ uint32_t drop_fin_b(uint32_t s) { s *= 0xC2B2AE35u; return s ^ (s >> 16); }
// keep tests on the two halves of a 32-bit word of draws.  thr_hi = thr16 << 16: (h >> 16) >= thr16 <=> h >= thr_hi.
__device__ __forceinline__ bool drop_keep_lo(uint32_t h, uint32_t thr16) { return (h & 0xFFFFu) >= thr16; }
__device__ __forceinline__ bool drop_keep_hi(uint32_t h, uint32_t thr16) { return h >= (thr16 << 16); }
// 32 random bits shared by elements 2*pair and 2*pair + 1 (low / high half)
__device__ __forceinline__ uint32_t dropout_bits(const Dropout& d, unsigned long long pair) {
  const unsigned long long quad = pair >> 1;
  const uint32_t s = drop_stage1(uint32_t(quad), drop_hikey(d, quad));
  return (pair & 1) ? drop_fin_b(s) : drop_fin_a(s);
}
// multiplier (0 or scale) for a single element
__device__ __forceinline__ float dropout_mult(const Dropout& d, unsigned long long idx) {
  if (d.p <= 0.f) return 1.f;
  const uint32_t h = dropout_bits(d, idx >> 1);
  const bool keep = (idx & 1) ? drop_keep_hi(h, d.thr16) : drop_keep_lo(h, d.thr16);
  return keep ? d.scale : 0.f;
}
// multipliers for the 4 elements of quad `quad` (elements 4*quad .. 4*quad + 3)
__device__ __forceinline__ float4 dropout_quad_mult(const Dropout& d, uint32_t quad_lo, uint32_t hikey) {
  const uint32_t s = drop_stage1(quad_lo, hikey);
  const uint32_t a = drop_fin_a(s), b = drop_fin_b(s);
  const float sc = d.scale;
  return make_float4(drop_keep_lo(a, d.thr16) ? sc : 0.f, drop_keep_hi(a, d.thr16) ? sc : 0.f,
                     drop_keep_lo(b, d.thr16) ? sc : 0.f, drop_keep_hi(b, d.thr16) ? sc : 0.f);
}
// multipliers for 4 consecutive elements starting at idx (idx % 4 == 0)
__device__ __forceinline__ float4 dropout_mult4(const Dropout& d, unsigned long long idx) {
  if (d.p <= 0.f) return make_float4(1.f, 1.f, 1.f, 1.f);
  const unsigned long long quad = idx >> 2;
  return dropout_quad_mult(d, uint32_t(quad), drop_hikey(d, quad));
}

// ----------------------------------------------------------------------------------------------
// warp reductions
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

inline int ceil_div(long long a, long long b) { return int((a + b - 1) / b); }

// Function attributes (cudaFuncSetAttribute) are PER DEVICE: a process that drives several GPUs (nn.DataParallel threads)
// must configure every kernel once on each of them.  `flags` is a function-local static array, one entry per device.
constexpr int kMaxDevices = 64;
inline bool first_use_on_device(bool (&flags)[kMaxDevices]) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) return true;
  if (flags[dev]) return false;
  flags[dev] = true;
  return true;
}

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch.  Kernels launched through launch_k() may start while their predecessor in the stream
// is still draining: they run their prologue (barrier init, descriptor prefetch ...) and then block in
// pdl_wait() until the predecessor has completed and its memory is visible.  EVERY kernel launched with launch_k() must
// call pdl_wait() before its first access to global memory.  ~400 dependent launches per train step: this hides the
// launch gap and the prologues of the many small group-level kernels.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(static_cast<Args&&>(args))...);
}

}  // namespace dsvg
