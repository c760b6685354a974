// wgmma / TMA contractions for sm_90a.
//
//   dsvg_linear : Y[M,N] = epilogue(X[M,K] . W[N,K]^T)     both operands K-major   (forward + dgrad)
//   dsvg_outer  : C[P,Q] += alpha * A[M,P]^T . B[M,Q]      both operands MN-major  (wgrad, contraction over rows)
//
// Both are warp-specialised: the last warp is the TMA producer (one elected lane); the consumer warpgroups before it
// issue wgmma into fp32 register accumulators and then run the epilogue (accumulator fragments -> per-warp shared-memory
// transpose -> registers -> bf16 staging tile + bulk tensor store, or coalesced global accesses / vector reductions).
// Operands land in shared memory through TMA with the 128-byte swizzle that the wgmma shared-memory descriptors
// name.  dsvg_linear is persistent (static round-robin tile schedule): the producer streams the next tile's operands
// while the consumers run the epilogue of the current one.
//
// Parity mode ("bf16x3"): operands carry a second bf16 plane (lo = v - bf16(v)); the consumers run three products
// per K step (hi*hi + hi*lo + lo*hi) into the same accumulator.  Same kernel, NPLANES = 2.
#include <cstdarg>
#include <cstring>
#include <mutex>
#include <unordered_map>

#include "../../include/dsvg_b200.h"
#include "common.cuh"
#include "ptx.cuh"

namespace dsvg {

// ------------------------------------------------------------------------------------------------
// error string + launch counter (shared by every translation unit)
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = {0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }
unsigned long long g_launches = 0;

// ------------------------------------------------------------------------------------------------
// TMA tensor maps (host).  cuTensorMapEncodeTiled is fetched through the runtime so libcuda is not a link-time
// dependency (the library must load on a CPU-only box for the symbol test).
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct MapKey {
  const void* ptr;
  uint64_t d0, d1, stride;
  uint32_t b0, b1;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && stride == o.stride && b0 == o.b0 && b1 == o.b1;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h ^= k.d0 * 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    h ^= k.d1 * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2);
    h ^= k.stride * 0x165667B19E3779F9ull + (h << 6) + (h >> 2);
    h ^= (uint64_t(k.b0) << 32 | k.b1) + (h << 6) + (h >> 2);
    return h;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
static std::mutex g_maps_mu;

// 2-D bf16 tensor, dim0 = contiguous (d0 elements), dim1 rows (d1) with `stride` elements between rows;
// box = b0 x b1 elements, 128-byte swizzle (b0 * 2 bytes must be 128).
static int make_map(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t stride, uint32_t b0,
                    uint32_t b1) {
  MapKey key{ptr, d0, d1, stride, b0, b1};
  {
    std::lock_guard<std::mutex> g(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) {
      *out = it->second;
      return 0;
    }
  }
  EncodeTiledFn enc = get_encode();
  DSVG_CHECK(enc != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  DSVG_CHECK((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA operand not 16-byte aligned");
  DSVG_CHECK((stride * 2) % 16 == 0, "TMA operand row stride must be a multiple of 8 elements (got %llu)",
             (unsigned long long)stride);
  cuuint64_t dims[2] = {d0, d1};
  cuuint64_t strides[1] = {stride * 2};
  cuuint32_t box[2] = {b0, b1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DSVG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (dims %llu x %llu, stride %llu)",
             int(r), (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)stride);
  {
    std::lock_guard<std::mutex> g(g_maps_mu);
    if (g_maps.size() > 4096) g_maps.clear();
    g_maps.emplace(key, *out);
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// shared epilogue
// ------------------------------------------------------------------------------------------------
struct Epi {
  const float* acc_scale_dev;  // optional device scalar multiplying the accumulator first
  const float* bias;
  int scale_cols;
  float scale;
  int relu;
  Dropout drop;
  const float* rowvec;
  int rowvec_ld;
  int rows_per_group;
  uint32_t rpg_magic;  // ceil(2^32 / rows_per_group): row / rows_per_group == __umulhi(row, magic) while row * rpg < 2^32
  const bf16* mask;
  size_t mask_lo_off;
  int mask_ld;
  float mask_scale;
  const float* residual;
  int res_ld;
  float* out_f32;
  int out_f32_ld;
  bf16* out_act;
  size_t out_lo_off;
  int out_act_ld;
  int vec;   // 1: every pointer/stride satisfies the 4-wide vector path
  int mode;  // 0: generic run-time epilogue; k > 0: lean epilogue kLeanFeat[k - 1]; 8: fused LayerNorm (see below)
  // ---- mode 8, fused LayerNorm (N == BN == 256: a CTA tile owns whole rows) ----
  // x1 = residual epilogue of mode 4 -> out_f32;  ln_out = bf16(LN(x1) * gamma + beta); mean / rstd saved
  const float* ln_gamma;
  const float* ln_beta;
  bf16* ln_out;         // [M, 256]
  float* ln_mean;
  float* ln_rstd;
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;         // 64 bf16 = 128 bytes = one swizzle span
constexpr int kStageRow = 36;       // fp32 staging row stride in words: 16-byte aligned rows, conflict-free v4 access
constexpr int kStageWarpBytes = 32 * kStageRow * 4;

__device__ __forceinline__ void st_shared_v4(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr)
               : "memory");
  return v;
}
__device__ __forceinline__ float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// scalar epilogue of one element (row, col): everything after the accumulator
__device__ __forceinline__ void epi_scalar(float x, long long row, int col, int N, const Epi& ep, float acc_scale) {
  x *= acc_scale;
  if (ep.bias != nullptr) x += __ldg(ep.bias + col);
  if (col < ep.scale_cols) x *= ep.scale;
  if (ep.relu) x = fmaxf(x, 0.f);
  if (ep.drop.p > 0.f) x *= dropout_mult(ep.drop, (unsigned long long)row * (unsigned long long)N + col);
  if (ep.rowvec != nullptr) x += __ldg(ep.rowvec + (long long)(int(row) / ep.rows_per_group) * ep.rowvec_ld + col);
  if (ep.mask != nullptr) {
    float m = act_load(ep.mask, ep.mask_lo_off, size_t(row) * ep.mask_ld + col);
    x = (m != 0.f) ? x * ep.mask_scale : 0.f;
  }
  if (ep.residual != nullptr) x += ep.residual[row * (long long)ep.res_ld + col];
  if (ep.out_f32 != nullptr) ep.out_f32[row * (long long)ep.out_f32_ld + col] = x;
  if (ep.out_act != nullptr) act_store(ep.out_act, ep.out_lo_off, size_t(row) * ep.out_act_ld + col, x);
}

__device__ __forceinline__ float4 ld_bf16x4(const bf16* p) {
  uint2 u = *reinterpret_cast<const uint2*>(p);
  float2 a = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u.x));
  float2 b = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void st_act4(bf16* p, size_t lo_off, size_t i, float4 x) {
  __nv_bfloat162 h0 = __floats2bfloat162_rn(x.x, x.y), h1 = __floats2bfloat162_rn(x.z, x.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&h0);
  u.y = *reinterpret_cast<uint32_t*>(&h1);
  *reinterpret_cast<uint2*>(p + i) = u;
  if (lo_off) {
    float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
    __nv_bfloat162 l0 = __floats2bfloat162_rn(x.x - f0.x, x.y - f0.y), l1 = __floats2bfloat162_rn(x.z - f1.x, x.w - f1.y);
    u.x = *reinterpret_cast<uint32_t*>(&l0);
    u.y = *reinterpret_cast<uint32_t*>(&l1);
    *reinterpret_cast<uint2*>(p + i + lo_off) = u;
  }
}

// Operands of the vector epilogue that come from global memory; loaded for all 8 row-iterations of a chunk BEFORE any
// store is issued, so the (up to three) DRAM round trips of a chunk overlap instead of serialising per iteration.
struct EpiLoads {
  float4 res, rv;
  uint2 mhi, mlo;
};
__device__ __forceinline__ float4 bf16x4_to_f4(uint2 u) {
  float2 a = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u.x));
  float2 b = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void epi_vec4_load(EpiLoads& l, long long row, int col, const Epi& ep) {
  if (ep.rowvec != nullptr)
    l.rv = __ldg(reinterpret_cast<const float4*>(ep.rowvec + (long long)(int(row) / ep.rows_per_group) * ep.rowvec_ld + col));
  if (ep.mask != nullptr) {
    const size_t mi = size_t(row) * ep.mask_ld + col;
    l.mhi = *reinterpret_cast<const uint2*>(ep.mask + mi);
    if (ep.mask_lo_off) l.mlo = *reinterpret_cast<const uint2*>(ep.mask + mi + ep.mask_lo_off);
  }
  if (ep.residual != nullptr) l.res = *reinterpret_cast<const float4*>(ep.residual + row * (long long)ep.res_ld + col);
}
// 4 consecutive columns of one row, all vector accesses aligned (host guarantees ep.vec preconditions)
__device__ __forceinline__ void epi_vec4(float4 x, long long row, int col, int N, const Epi& ep, const float4& bias4,
                                         float acc_scale, const EpiLoads& l) {
  x.x *= acc_scale; x.y *= acc_scale; x.z *= acc_scale; x.w *= acc_scale;
  x.x += bias4.x; x.y += bias4.y; x.z += bias4.z; x.w += bias4.w;
  if (ep.scale_cols > 0) {
    if (col + 0 < ep.scale_cols) x.x *= ep.scale;
    if (col + 1 < ep.scale_cols) x.y *= ep.scale;
    if (col + 2 < ep.scale_cols) x.z *= ep.scale;
    if (col + 3 < ep.scale_cols) x.w *= ep.scale;
  }
  if (ep.relu) {
    x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f);
  }
  if (ep.drop.p > 0.f) {
    float4 m = dropout_mult4(ep.drop, (unsigned long long)row * (unsigned long long)N + col);
    x.x *= m.x; x.y *= m.y; x.z *= m.z; x.w *= m.w;
  }
  if (ep.rowvec != nullptr) {
    x.x += l.rv.x; x.y += l.rv.y; x.z += l.rv.z; x.w += l.rv.w;
  }
  if (ep.mask != nullptr) {
    float4 m = bf16x4_to_f4(l.mhi);
    if (ep.mask_lo_off) {
      float4 lo = bf16x4_to_f4(l.mlo);
      m.x += lo.x; m.y += lo.y; m.z += lo.z; m.w += lo.w;
    }
    x.x = m.x != 0.f ? x.x * ep.mask_scale : 0.f;
    x.y = m.y != 0.f ? x.y * ep.mask_scale : 0.f;
    x.z = m.z != 0.f ? x.z * ep.mask_scale : 0.f;
    x.w = m.w != 0.f ? x.w * ep.mask_scale : 0.f;
  }
  if (ep.residual != nullptr) {
    x.x += l.res.x; x.y += l.res.y; x.z += l.res.z; x.w += l.res.w;
  }
  if (ep.out_f32 != nullptr) *reinterpret_cast<float4*>(ep.out_f32 + row * (long long)ep.out_f32_ld + col) = x;
  if (ep.out_act != nullptr) st_act4(ep.out_act, ep.out_lo_off, size_t(row) * ep.out_act_ld + col, x);
}

// Processes 32 accumulator columns held one-row-per-thread (as acc_to_rows leaves them), transposing them through
// this warp's private shared-memory tile so that every global access is a coalesced row segment.
//   v[j]       : accumulator of row (row0 + lane), column (col0 + j)
//   stage_addr : shared-space byte address of this warp's [32][36] fp32 staging tile
__device__ __forceinline__ void epilogue_chunk(uint32_t (&v)[32], uint32_t stage_addr, int lane, long long row0, int col0,
                                               int M, int N, const Epi& ep) {
  const float acc_scale = ep.acc_scale_dev != nullptr ? __ldg(ep.acc_scale_dev) : 1.f;
  {
    const uint32_t my = stage_addr + lane * (kStageRow * 4);
#pragma unroll
    for (int q = 0; q < 8; ++q)
      st_shared_v4(my + q * 16, __uint_as_float(v[4 * q]), __uint_as_float(v[4 * q + 1]), __uint_as_float(v[4 * q + 2]),
                   __uint_as_float(v[4 * q + 3]));
  }
  __syncwarp();
  if (ep.vec) {
    const int cg = lane & 7, rsub = lane >> 3;
    const int col = col0 + 4 * cg;
    const bool col_ok = col < N;
    float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ep.bias != nullptr && col_ok) bias4 = __ldg(reinterpret_cast<const float4*>(ep.bias + col));
#pragma unroll
    for (int h = 0; h < 2; ++h) {   // two groups of four rows: 4 x (residual, mask, rowvec) loads in flight per group
      EpiLoads ld[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const long long row = row0 + 4 * (4 * h + i) + rsub;
        if (row < M && col_ok) epi_vec4_load(ld[i], row, col, ep);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int rl = 4 * (4 * h + i) + rsub;
        float4 x = ld_shared_v4(stage_addr + (rl * kStageRow + 4 * cg) * 4);
        const long long row = row0 + rl;
        if (row < M && col_ok) epi_vec4(x, row, col, N, ep, bias4, acc_scale, ld[i]);
      }
    }
  } else {
    // scalar path (row stride not 16-byte friendly: the fp32 logits).  Lane = column; the column's bias is loaded once.
    const int col = col0 + lane;
    const bool col_ok = col < N;
    const bool simple = ep.rowvec == nullptr && ep.mask == nullptr && ep.residual == nullptr && ep.drop.p <= 0.f &&
                        ep.out_act == nullptr && ep.scale_cols == 0;
    if (simple) {
      const float b = (ep.bias != nullptr && col_ok) ? __ldg(ep.bias + col) : 0.f;
#pragma unroll 8
      for (int r = 0; r < 32; ++r) {
        const long long row = row0 + r;
        float x = ld_shared_f32(stage_addr + (r * kStageRow + lane) * 4) * acc_scale + b;
        if (ep.relu) x = fmaxf(x, 0.f);
        if (row < M && col_ok) ep.out_f32[row * (long long)ep.out_f32_ld + col] = x;
      }
    } else {
#pragma unroll 4
      for (int r = 0; r < 32; ++r) {
        const long long row = row0 + r;
        float x = ld_shared_f32(stage_addr + (r * kStageRow + lane) * 4);
        if (row < M && col_ok) epi_scalar(x, row, col, N, ep, acc_scale);
      }
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// Lean epilogues.  The generic path above decides every step at run time (~100 instructions per 4 outputs, which makes
// the epilogue warps issue-bound).  The model's
// fast-mode GEMMs use only a handful of step combinations; each is compiled with its steps fixed (FEAT bit mask) and
// pointer arithmetic hoisted out of the row loop.  All of them require the aligned vector layout (ep.vec != 0) and
// single-plane act tensors.
// ------------------------------------------------------------------------------------------------
enum : uint32_t { F_BIAS = 1, F_SCALE = 2, F_RELU = 4, F_DROP = 8, F_ROWVEC = 16, F_MASK = 32, F_RES = 64,
                  F_OUTF = 128, F_OUTA = 256, F_ACCS = 512 };

// global-memory operands of one 32x32 chunk (8 row-iterations of this lane), fetched one chunk ahead of their use
template <uint32_t FEAT>
struct LeanPre {
  float4 res[(FEAT & F_RES) ? 8 : 1];
  uint2 msk[(FEAT & F_MASK) ? 8 : 1];
};
template <uint32_t FEAT>
__device__ __forceinline__ void lean_prefetch(LeanPre<FEAT>& p, int lane, int row0, int col0, int M, int N, const Epi& ep) {
  if constexpr ((FEAT & (F_RES | F_MASK)) != 0) {
    const int cg = lane & 7, rsub = lane >> 3;
    const int col = col0 + 4 * cg;
    if (col < N) {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int row = row0 + rsub + 4 * it;
        if (row < M) {
          if constexpr (FEAT & F_RES)
            p.res[it] = ep.residual != nullptr ? *reinterpret_cast<const float4*>(ep.residual + size_t(row) * ep.res_ld + col)
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
          if constexpr (FEAT & F_MASK) p.msk[it] = *reinterpret_cast<const uint2*>(ep.mask + size_t(row) * ep.mask_ld + col);
        }
      }
    }
  }
}

template <uint32_t FEAT>
__device__ __forceinline__ void epilogue_chunk_lean(uint32_t (&v)[32], uint32_t stage_addr, int lane, int row0, int col0,
                                                    int M, int N, const Epi& ep, const LeanPre<FEAT>& pre,
                                                    const float4& bias_in) {
  {
    const uint32_t my = stage_addr + lane * (kStageRow * 4);
#pragma unroll
    for (int q = 0; q < 8; ++q)
      st_shared_v4(my + q * 16, __uint_as_float(v[4 * q]), __uint_as_float(v[4 * q + 1]), __uint_as_float(v[4 * q + 2]),
                   __uint_as_float(v[4 * q + 3]));
  }
  __syncwarp();
  const int cg = lane & 7, rsub = lane >> 3;
  const int col = col0 + 4 * cg;
  if (col < N) {
    const float4 bias4 = bias_in;   // fetched by the caller at the top of the tile (off the chunk's critical path)
    float accs = 1.f;
    if constexpr (FEAT & F_ACCS) accs = __ldg(ep.acc_scale_dev);
    const int r_first = row0 + rsub;
    float* outf_p = nullptr;
    bf16* outa_p = nullptr;
    if constexpr (FEAT & F_OUTF) outf_p = ep.out_f32 + size_t(r_first) * ep.out_f32_ld + col;
    if constexpr (FEAT & F_OUTA) outa_p = ep.out_act + size_t(r_first) * ep.out_act_ld + col;
    const bool has_rv = (FEAT & F_ROWVEC) && ep.rowvec != nullptr;
    const bool has_drop = (FEAT & F_DROP) && ep.drop.p > 0.f;
    const uint32_t lds_base = stage_addr + (rsub * kStageRow + 4 * cg) * 4;
    // dropout quad index of (r_first, col); N % 4 == 0 and col % 4 == 0 on this path
    const unsigned long long quad0 = ((unsigned long long)r_first * (unsigned long long)N + (unsigned long long)col) >> 2;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = r_first + 4 * it;
      float4 x = ld_shared_v4(lds_base + it * (4 * kStageRow * 4));
      if (row < M) {
        if constexpr (FEAT & F_ACCS) { x.x *= accs; x.y *= accs; x.z *= accs; x.w *= accs; }
        if constexpr (FEAT & F_BIAS) { x.x += bias4.x; x.y += bias4.y; x.z += bias4.z; x.w += bias4.w; }
        if constexpr (FEAT & F_SCALE) {
          if (col < ep.scale_cols) { x.x *= ep.scale; x.y *= ep.scale; x.z *= ep.scale; x.w *= ep.scale; }  // scale_cols % 4 == 0
        }
        if constexpr (FEAT & F_RELU) {
          x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f);
        }
        if constexpr (FEAT & F_DROP) {
          if (has_drop) {
            const unsigned long long quad = quad0 + (unsigned long long)it * (unsigned long long)N;   // row advances by 4
            const float4 m = dropout_quad_mult(ep.drop, uint32_t(quad), drop_hikey(ep.drop, quad));
            x.x *= m.x; x.y *= m.y; x.z *= m.z; x.w *= m.w;
          }
        }
        if constexpr (FEAT & F_ROWVEC) {
          if (has_rv) {
            const uint32_t grp = ep.rpg_magic ? __umulhi(uint32_t(row), ep.rpg_magic) : uint32_t(row / ep.rows_per_group);
            float4 rv = __ldg(reinterpret_cast<const float4*>(ep.rowvec + size_t(grp) * ep.rowvec_ld + col));
            x.x += rv.x; x.y += rv.y; x.z += rv.z; x.w += rv.w;
          }
        }
        if constexpr (FEAT & F_MASK) {
          float4 m = bf16x4_to_f4(pre.msk[it]);
          x.x = m.x != 0.f ? x.x * ep.mask_scale : 0.f;
          x.y = m.y != 0.f ? x.y * ep.mask_scale : 0.f;
          x.z = m.z != 0.f ? x.z * ep.mask_scale : 0.f;
          x.w = m.w != 0.f ? x.w * ep.mask_scale : 0.f;
        }
        if constexpr (FEAT & F_RES) {
          x.x += pre.res[it].x; x.y += pre.res[it].y; x.z += pre.res[it].z; x.w += pre.res[it].w;
        }
        if constexpr (FEAT & F_OUTF) *reinterpret_cast<float4*>(outf_p + size_t(4 * it) * ep.out_f32_ld) = x;
        if constexpr (FEAT & F_OUTA) {
          __nv_bfloat162 h0 = __floats2bfloat162_rn(x.x, x.y), h1 = __floats2bfloat162_rn(x.z, x.w);
          uint2 u;
          u.x = *reinterpret_cast<uint32_t*>(&h0);
          u.y = *reinterpret_cast<uint32_t*>(&h1);
          *reinterpret_cast<uint2*>(outa_p + size_t(4 * it) * ep.out_act_ld) = u;
          if (ep.out_lo_off != 0) {   // parity mode: lo plane = bf16(v - hi)  (warp-uniform branch)
            const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
            h0 = __floats2bfloat162_rn(x.x - f0.x, x.y - f0.y);
            h1 = __floats2bfloat162_rn(x.z - f1.x, x.w - f1.y);
            u.x = *reinterpret_cast<uint32_t*>(&h0);
            u.y = *reinterpret_cast<uint32_t*>(&h1);
            *reinterpret_cast<uint2*>(outa_p + ep.out_lo_off + size_t(4 * it) * ep.out_act_ld) = u;
          }
        }
      }
    }
  }
  __syncwarp();
}


// feature sets with a compiled lean epilogue (index = Epi::mode - 1)
constexpr uint32_t kLeanFeat[] = {
    F_OUTA,                                   // 1: plain dgrad
    F_BIAS | F_SCALE | F_OUTA,                // 2: QKV projection
    F_BIAS | F_RELU | F_DROP | F_OUTA,        // 3: FFN first linear
    F_BIAS | F_DROP | F_ROWVEC | F_RES | F_OUTF,  // 4: out-proj / FFN second linear into the fp32 residual stream
    F_MASK | F_OUTA,                          // 5: dgrad through ReLU (+dropout) mask
    F_ACCS | F_RES | F_OUTF,                  // 6: head dgrads accumulated in fp32
    F_BIAS | F_OUTF,                          // 7: fp32 rows of ANY alignment (the 2827-wide logits, N = 7 / 2 heads);
                                              //    chosen by pick_mode for ep.vec == 0, never by the feature search
};
constexpr int kNumLean = 6;                   // modes found by the feature search in pick_mode

// mode 7: one 32 x 32 chunk -> out_f32[row, col] = acc + bias[col]; lane = column, so every store instruction writes one
// 128-byte row segment whatever the row stride (no 16-byte alignment needed).
__device__ __forceinline__ void plain_rows_chunk(uint32_t (&v)[32], uint32_t stage_addr, int lane, long long row0, int col0,
                                                 int M, int N, const Epi& ep) {
  const uint32_t my = stage_addr + lane * (kStageRow * 4);
#pragma unroll
  for (int q = 0; q < 8; ++q)
    st_shared_v4(my + q * 16, __uint_as_float(v[4 * q]), __uint_as_float(v[4 * q + 1]), __uint_as_float(v[4 * q + 2]),
                 __uint_as_float(v[4 * q + 3]));
  __syncwarp();
  const int col = col0 + lane;
  if (col < N) {
    const float b = ep.bias != nullptr ? __ldg(ep.bias + col) : 0.f;
    float* out = ep.out_f32 + row0 * (long long)ep.out_f32_ld + col;
    const int rows = (M - row0) < 32 ? int(M - row0) : 32;
    if (rows == 32) {
#pragma unroll
      for (int r = 0; r < 32; ++r) out[(long long)r * ep.out_f32_ld] = ld_shared_f32(stage_addr + (r * kStageRow + lane) * 4) + b;
    } else {
      for (int r = 0; r < rows; ++r) out[(long long)r * ep.out_f32_ld] = ld_shared_f32(stage_addr + (r * kStageRow + lane) * 4) + b;
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// TMA-store epilogue (act outputs): thread = accumulator row, 32 columns in registers; every step runs in
// registers, the bf16 result goes into a 128-byte-swizzled [128 x BN] tile in shared memory and leaves the SM as one
// bulk tensor store per 64-column box.  No shared-memory read-back, no per-thread global stores.
// ------------------------------------------------------------------------------------------------
template <uint32_t FEAT>
__device__ __forceinline__ void tma_out_chunk(uint32_t (&v)[32], uint8_t* out_tile, int r, long long grow, int gc0, int c,
                                              int M, int N, const Epi& ep, const uint4 (&mk)[4], uint32_t bias_sm) {
  float x[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) x[j] = __uint_as_float(v[j]);
  if constexpr (FEAT & F_BIAS) {
    // bias_sm holds bias[n0 .. n0 + BN) (zero past N), staged once per n-tile by the epilogue warps: broadcast LDS.128
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 b = ld_shared_v4(bias_sm + (c + 4 * q) * 4);
      x[4 * q] += b.x; x[4 * q + 1] += b.y; x[4 * q + 2] += b.z; x[4 * q + 3] += b.w;
    }
  }
  if constexpr (FEAT & F_SCALE) {
    if (gc0 < ep.scale_cols) {   // scale_cols % 32 == 0 (pick_mode): the whole chunk is scaled or none of it
#pragma unroll
      for (int j = 0; j < 32; ++j) x[j] *= ep.scale;
    }
  }
  if constexpr (FEAT & F_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] = fmaxf(x[j], 0.f);
  }
  if constexpr (FEAT & F_DROP) {
    if (ep.drop.p > 0.f) {
      // 32 consecutive elements starting at a multiple of 8 (N % 8 == 0, gc0 % 32 == 0): 8 quads whose low index
      // word cannot carry, so key' is computed once
      const unsigned long long qb = ((unsigned long long)grow * (unsigned long long)N + (unsigned long long)gc0) >> 2;
      const uint32_t hk = drop_hikey(ep.drop, qb), q0 = uint32_t(qb), thr = ep.drop.thr16;
      const float sc = ep.drop.scale;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const uint32_t s1 = drop_stage1(q0 + q, hk);
        const uint32_t a = drop_fin_a(s1), b = drop_fin_b(s1);
        x[4 * q] = drop_keep_lo(a, thr) ? x[4 * q] * sc : 0.f;
        x[4 * q + 1] = drop_keep_hi(a, thr) ? x[4 * q + 1] * sc : 0.f;
        x[4 * q + 2] = drop_keep_lo(b, thr) ? x[4 * q + 2] * sc : 0.f;
        x[4 * q + 3] = drop_keep_hi(b, thr) ? x[4 * q + 3] * sc : 0.f;
      }
    }
  }
  if constexpr (FEAT & F_MASK) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t w[4] = {mk[q].x, mk[q].y, mk[q].z, mk[q].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        // a bf16 is non-zero iff any of its 15 magnitude bits is set
        x[8 * q + 2 * e] = (w[e] & 0x7FFFu) ? x[8 * q + 2 * e] * ep.mask_scale : 0.f;
        x[8 * q + 2 * e + 1] = (w[e] & 0x7FFF0000u) ? x[8 * q + 2 * e + 1] * ep.mask_scale : 0.f;
      }
    }
  }
  // pack and store: 4 x 16 bytes at swizzled positions of row r in the 64-column box (c / 64)
  uint8_t* box = out_tile + (c >> 6) * (kBlockM * 128) + r * 128;
  const int j0 = (c & 63) >> 3;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 u;
    __nv_bfloat162 t;
    t = __floats2bfloat162_rn(x[8 * q], x[8 * q + 1]); u.x = *reinterpret_cast<uint32_t*>(&t);
    t = __floats2bfloat162_rn(x[8 * q + 2], x[8 * q + 3]); u.y = *reinterpret_cast<uint32_t*>(&t);
    t = __floats2bfloat162_rn(x[8 * q + 4], x[8 * q + 5]); u.z = *reinterpret_cast<uint32_t*>(&t);
    t = __floats2bfloat162_rn(x[8 * q + 6], x[8 * q + 7]); u.w = *reinterpret_cast<uint32_t*>(&t);
    *reinterpret_cast<uint4*>(box + (((j0 + q) ^ (r & 7)) << 4)) = u;
  }
}
template <uint32_t FEAT>
__device__ __forceinline__ void tma_out_load_mask(uint4 (&mk)[4], long long grow, int gc0, int M, int N, const Epi& ep) {
  if constexpr (FEAT & F_MASK) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      mk[q] = make_uint4(0, 0, 0, 0);
      if (grow < M && gc0 + 8 * q < N)
        mk[q] = *reinterpret_cast<const uint4*>(ep.mask + size_t(grow) * ep.mask_ld + gc0 + 8 * q);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// dsvg_linear kernel
// ------------------------------------------------------------------------------------------------
// act-output lean modes write their bf16 tile through shared memory with one TMA store per 64-column box
// (single-plane tensors only: the two-plane parity mode sends the same feature sets through the per-warp staged epilogue,
// which writes the hi and lo planes with plain vector stores)
__host__ __device__ constexpr bool lin_tma_out(int mode, int nplanes = 1) {
  return nplanes == 1 && (mode == 1 || mode == 2 || mode == 3 || mode == 5);
}
// E consumer warps (E / 4 warpgroups issue the wgmma and then run the epilogue) + one TMA producer warp.
__host__ __device__ constexpr int lin_epi_warps(int mode, int bn) {
  // mode 7 (fp32 rows of any alignment) runs 16 warps wide on the 256-wide tile: each thread then holds 64 accumulator
  // registers.  Mode 6 (head dgrads, K = 2827, light epilogue) keeps 8 warps.
  return (mode == 7 && bn == 256) ? 16 : 8;
}
// The 256-wide single-plane kernels of the path-level GEMM roles (modes 1-5 and the fused LayerNorm 8) run the
// full-width kernel below (linear_wide): two consumer warpgroups with one m64n256 wgmma per k16 step each, and the
// epilogue applied to the accumulator fragments.
__host__ __device__ constexpr bool lin_wide(int mode, int bn, int nplanes) {
  return bn == 256 && nplanes == 1 && ((mode >= 1 && mode <= 5) || mode == 8);
}

template <int MODE>
struct WideCfg {
  static constexpr int kThreads = 384;                   // consumer warpgroups 0 and 1, producer warpgroup 2
  static constexpr int kStages = 4;
  static constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KB: warpgroup g reads rows [64 g, 64 g + 64)
  static constexpr int kBBytes = 256 * kBlockK * 2;      // 32 KB, read by both warpgroups
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBoxBytes = 64 * 128;             // one [64 rows][64 bf16 columns] output box, 128-byte swizzle
  // bf16 outputs (mode 8: the LayerNorm output) leave through a two-box ring per consumer warpgroup
  static constexpr int kStagingBytes = MODE == 4 ? 0 : 2 * 2 * kBoxBytes;
  static constexpr int kSmemBytes = 1024 /*align slack*/ + kStages * kStageBytes + kStagingBytes + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "linear_wide: shared memory over the per-block limit of sm_90");
};

template <int BN, int NPLANES, int MODE = 0>
struct LinearCfg {
  static constexpr bool kWide = lin_wide(MODE, BN, NPLANES);
  static constexpr int kEpiWarps = lin_epi_warps(MODE, BN);
  // staged kernel: the producer is the last warp (consumers stay warpgroup-aligned)
  static constexpr int kThreads = kWide ? WideCfg<MODE>::kThreads : 32 * kEpiWarps + 32;
  static constexpr int kChunks = BN / (8 * kEpiWarps);    // 32-column accumulator chunks per consumer warp
  static constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KB
  static constexpr int kBBytes = BN * kBlockK * 2;       // 16/32 KB
  static constexpr int kStageBytes = NPLANES * (kABytes + kBBytes);
  static constexpr int kStagingBytes = lin_tma_out(MODE, NPLANES) ? BN * kBlockM * 2 : kEpiWarps * kStageWarpBytes;
  // per-warp fragment transposition tiles; the staged epilogues use their staging tiles for it
  static constexpr int kXposeBytes = lin_tma_out(MODE, NPLANES) ? kEpiWarps * kStageWarpBytes : 0;
  static constexpr int kBiasBytes = BN * 4;   // bias slice of the current n-tile (TMA-out epilogues)
  static constexpr int kFixedBytes = 1024 /*align slack*/ + kStagingBytes + kXposeBytes + 256 + kBiasBytes;
  static constexpr int kMaxSmem = 227 * 1024;   // per-block dynamic shared memory limit of sm_90
  static constexpr int kStages = (kMaxSmem - kFixedBytes) / kStageBytes > 4 ? 4 : (kMaxSmem - kFixedBytes) / kStageBytes;
  static_assert(kStages >= 2, "linear: at least two pipeline stages must fit");
  static constexpr int kSmemBytes = kWide ? WideCfg<MODE>::kSmemBytes : kFixedBytes + kStages * kStageBytes;
};

// One 32 x 32 chunk of a consumer warp's accumulators, a[h] = fragment of the m64 half h (local rows [16 h, 16 h + 16)),
// -> v[j] = accumulator (local row = lane, column j): the row-per-thread form the epilogues consume.  Transposed through
// the warp's private [32][kStageRow] staging tile.
__device__ __forceinline__ void acc_to_rows(const float (&a)[2][16], uint32_t stage_addr, int lane, uint32_t (&v)[32]) {
  __syncwarp();
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int lr = 16 * h + 8 * i + (lane >> 2), col = 8 * j + 2 * (lane & 3);
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stage_addr + (lr * kStageRow + col) * 4),
                     "f"(a[h][4 * j + 2 * i]), "f"(a[h][4 * j + 2 * i + 1]) : "memory");
      }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 x = ld_shared_v4(stage_addr + (lane * kStageRow + 4 * q) * 4);
    v[4 * q] = __float_as_uint(x.x); v[4 * q + 1] = __float_as_uint(x.y);
    v[4 * q + 2] = __float_as_uint(x.z); v[4 * q + 3] = __float_as_uint(x.w);
  }
  __syncwarp();
}

// Staged kernel (every linear_kernel instantiation but the full-width ones): consumer warps issue n32 wgmmas and
// drain the accumulators 32 x 32 chunks at a time through per-warp transposition tiles.  The tensor maps are the
// kernel's __grid_constant__ parameters.
template <int BN, int NPLANES, int MODE>
__device__ __forceinline__ void linear_staged(const CUtensorMap& tmA, const CUtensorMap& tmAlo, const CUtensorMap& tmB,
                                              const CUtensorMap& tmBlo, const CUtensorMap& tmC, const CUtensorMap& tmM,
                                              int M, int N, int K, Epi ep) {
  using Cfg = LinearCfg<BN, NPLANES, MODE>;
  constexpr int kCols = Cfg::kEpiWarps * 8;   // accumulator columns drained per pass of all epilogue warps (64 or 128)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* tiles = smem;
  float* staging = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint8_t* xpose = smem + Cfg::kStages * Cfg::kStageBytes + Cfg::kStagingBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(xpose + Cfg::kXposeBytes);
  uint64_t* full_bar = bars;                       // [kStages]
  uint64_t* empty_bar = bars + Cfg::kStages;       // [kStages]
  uint64_t* mfull_bar = bars + 2 * Cfg::kStages;   // [2] mask boxes of pass 0 / 1 have landed (mode 5)
  float* bias_sm = reinterpret_cast<float*>(xpose + Cfg::kXposeBytes + 256);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kProducer = Cfg::kEpiWarps;

  if (warp == kProducer && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (NPLANES == 2) {
      tma_prefetch_desc(&tmAlo);
      tma_prefetch_desc(&tmBlo);
    }
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], Cfg::kEpiWarps);
    }
    for (int a = 0; a < 2; ++a) mbar_init(&mfull_bar[a], 1);
    fence_barrier_init();
  }
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();   // everything above touched only this CTA's shared memory

  const int m_tiles = (M + kBlockM - 1) / kBlockM;
  const int n_tiles = (N + BN - 1) / BN;
  const int num_tiles = m_tiles * n_tiles;
  const int num_kb = (K + kBlockK - 1) / kBlockK;

  if (warp == kProducer) {
    // =================== TMA producer (warp-uniform control flow, one elected lane issues) ===================
    // A arrives in 16-row boxes: tile rows [32 w + 16 h, +16) go to shared rows [64 h + 16 w, +16), so that warp w of a
    // consumer warpgroup, which owns rows [16 w, 16 w + 16) of each m64 half h, holds tile rows [32 w, 32 w + 32).
    int stage = 0;
    uint32_t phase = 0;
    int pit = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++pit) {
      const int m0 = (tile / n_tiles) * kBlockM;
      const int n0 = (tile % n_tiles) * BN;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* st = tiles + stage * Cfg::kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
#pragma unroll
          for (int w = 0; w < 4; ++w)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int srow = 64 * h + 16 * w;
              tma_load_2d(st + srow * 128, &tmA, &full_bar[stage], kb * kBlockK, m0 + 32 * w + 16 * h);
              if (NPLANES == 2)
                tma_load_2d(st + Cfg::kABytes + Cfg::kBBytes + srow * 128, &tmAlo, &full_bar[stage], kb * kBlockK,
                            m0 + 32 * w + 16 * h);
            }
          tma_load_2d(st + Cfg::kABytes, &tmB, &full_bar[stage], kb * kBlockK, n0);
          if (NPLANES == 2) tma_load_2d(st + 2 * Cfg::kABytes + Cfg::kBBytes, &tmBlo, &full_bar[stage], kb * kBlockK, n0);
        }
        __syncwarp();
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // =================== consumer warpgroups: wgmma main loop, then the epilogue ===================
    drop_resolve(ep.drop);
    const int quarter = warp & 3;   // warp within its warpgroup: accumulator rows [32 quarter, 32 quarter + 32)
    const int half = warp >> 2;     // warpgroup: accumulator column chunks half * 32 + kCols * ci
    const uint32_t stage_buf = smem_u32(lin_tma_out(MODE, NPLANES) ? static_cast<void*>(xpose) : static_cast<void*>(staging)) +
                               warp * kStageWarpBytes;
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    int bias_n0 = -1;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int m0 = (tile / n_tiles) * kBlockM;
      const int n0 = (tile % n_tiles) * BN;
      const long long row0 = (long long)m0 + quarter * 32;
      // accumulators of this warp: chunk ci, m64 half h (operand columns past N are zero-filled by TMA)
      float accum[Cfg::kChunks][2][16];
#pragma unroll
      for (int ci = 0; ci < Cfg::kChunks; ++ci)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 16; ++j) accum[ci][h][j] = 0.f;
      int prev_stage = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        const uint32_t a_hi = smem_u32(tiles + stage * Cfg::kStageBytes);
        const uint32_t b_hi = a_hi + Cfg::kABytes;
        const uint32_t a_lo = b_hi + Cfg::kBBytes;
        const uint32_t b_lo = a_lo + Cfg::kABytes;
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)
#pragma unroll
          for (int ci = 0; ci < Cfg::kChunks; ++ci) {
            const uint32_t boff = uint32_t(half * 32 + kCols * ci) * 128u + k * 32;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t aoff = h * 8192 + k * 32;
              wgmma_m64n32_kk(accum[ci][h], gmma_smem_desc(a_hi + aoff, 16, 1024), gmma_smem_desc(b_hi + boff, 16, 1024));
              if (NPLANES == 2) {
                wgmma_m64n32_kk(accum[ci][h], gmma_smem_desc(a_hi + aoff, 16, 1024), gmma_smem_desc(b_lo + boff, 16, 1024));
                wgmma_m64n32_kk(accum[ci][h], gmma_smem_desc(a_lo + aoff, 16, 1024), gmma_smem_desc(b_hi + boff, 16, 1024));
              }
            }
          }
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();                                    // the previous k-block's MMAs have read their stage
          if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        }
        prev_stage = stage;
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int ci = 0; ci < Cfg::kChunks; ++ci)
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma_fence_regs(accum[ci][h]);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      if constexpr (MODE == 0) {
#pragma unroll
        for (int ci = 0; ci < Cfg::kChunks; ++ci) {
          const int c = half * 32 + kCols * ci;
          if (n0 + c >= N) break;
          uint32_t v[32];
          acc_to_rows(accum[ci], stage_buf, lane, v);
          epilogue_chunk(v, stage_buf, lane, row0, n0 + c, M, N, ep);
        }
      } else if constexpr (MODE == 7) {
#pragma unroll
        for (int ci = 0; ci < Cfg::kChunks; ++ci) {
          const int c = half * 32 + kCols * ci;
          if (n0 + c >= N) break;
          uint32_t v[32];
          acc_to_rows(accum[ci], stage_buf, lane, v);
          plain_rows_chunk(v, stage_buf, lane, row0, n0 + c, M, N, ep);
        }
      } else if constexpr (lin_tma_out(MODE, NPLANES)) {
        // Streamed TMA-store epilogue.  A "pass" = all epilogue warps draining kCols accumulator columns into their
        // 64-column boxes of the staging tile; each pass ends with ONE named barrier after which an elected thread
        // bulk-stores the pass's boxes as one group.  Box reuse: the boxes of pass ci were last stored kPasses groups
        // ago, so before the barrier of pass ci - 1 the storing thread waits until at most kPasses - 2 groups are still
        // reading shared memory; the TMA engine therefore streams tile t's boxes out while tile t + 1 is drained.
        constexpr uint32_t FEAT = kLeanFeat[MODE > 0 ? MODE - 1 : 0];
        constexpr int kPasses = BN / kCols;
        static_assert(kPasses >= 2, "streamed TMA-store epilogue needs at least two passes per tile");
        uint8_t* out_tile = reinterpret_cast<uint8_t*>(staging);
        const int r = quarter * 32 + lane;
        const long long grow = (long long)m0 + r;
        // Mask dgrad: the ReLU/dropout mask tile arrives by TMA INTO the staging boxes the output is about to overwrite
        // (same 128-byte swizzle, so a thread finds its row's mask at the very positions it will write).  The per-thread
        // global loads it replaces read 64 bytes per lane from 32 different rows: latency-bound at 19 % issue / 40 % DRAM.
        constexpr bool kTmaMask = (FEAT & F_MASK) != 0 && kPasses == 2;
        constexpr int kBoxesPerPass = kCols / 64;
        auto issue_mask = [&](int tile_, int pass) {           // storing thread only
          const int mm0 = (tile_ / n_tiles) * kBlockM, nn0 = (tile_ % n_tiles) * BN;
          uint32_t bytes = 0;
#pragma unroll
          for (int bx = pass * kBoxesPerPass; bx < (pass + 1) * kBoxesPerPass; ++bx)
            if (nn0 + 64 * bx < N) bytes += kBlockM * 128;
          mbar_arrive_expect_tx(&mfull_bar[pass], bytes);
#pragma unroll
          for (int bx = pass * kBoxesPerPass; bx < (pass + 1) * kBoxesPerPass; ++bx)
            if (nn0 + 64 * bx < N) tma_load_2d(out_tile + bx * (kBlockM * 128), &tmM, &mfull_bar[pass], nn0 + 64 * bx, mm0);
        };
        if constexpr (kTmaMask) {
          if (warp == 0 && lane == 0) {
            if (it == 0) {
              issue_mask(tile, 0);                              // nothing has used the staging tile yet
              issue_mask(tile, 1);
            } else {
              tma_store_wait_read_n<0>();                       // the previous tile's last store has drained its boxes
              issue_mask(tile, 1);                              // (pass 0 of this tile was requested during the previous tile)
            }
          }
        }
        uint4 mk[2][4];
        if constexpr (!kTmaMask) tma_out_load_mask<FEAT>(mk[0], grow, n0 + half * 32, M, N, ep);
        if constexpr (FEAT & F_BIAS) {
          if (n0 != bias_n0) {   // same decision in every epilogue warp (they walk the same tile sequence)
            const int et = threadIdx.x;
            named_bar_sync(2, Cfg::kEpiWarps * 32);        // nobody still reads the previous slice
            for (int j = et; j < BN; j += Cfg::kEpiWarps * 32) bias_sm[j] = (n0 + j < N) ? __ldg(ep.bias + n0 + j) : 0.f;
            named_bar_sync(2, Cfg::kEpiWarps * 32);
            bias_n0 = n0;
          }
        }
#pragma unroll
        for (int ci = 0; ci < kPasses; ++ci) {
          const int c = half * 32 + kCols * ci;
          if (n0 + c < N) {
            uint32_t v[32];
            acc_to_rows(accum[ci], stage_buf, lane, v);
            if constexpr (kTmaMask) {
              mbar_wait(&mfull_bar[ci], uint32_t(it & 1));
              const uint8_t* box = out_tile + (c >> 6) * (kBlockM * 128) + r * 128;
              const int j0 = (c & 63) >> 3;
#pragma unroll
              for (int q = 0; q < 4; ++q) mk[ci & 1][q] = *reinterpret_cast<const uint4*>(box + (((j0 + q) ^ (r & 7)) << 4));
            } else {
              if (ci + 1 < kPasses) tma_out_load_mask<FEAT>(mk[(ci + 1) & 1], grow, n0 + c + kCols, M, N, ep);
            }
            tma_out_chunk<FEAT>(v, out_tile, r, grow, n0 + c, c, M, N, ep, mk[ci & 1], smem_u32(bias_sm));
          }
          fence_proxy_async_smem();                          // generic-proxy smem writes -> visible to the TMA engine
          if (warp == 0 && lane == 0) {
            tma_store_wait_read_n<(kPasses - 2)>();   // next pass's boxes are free again
            if constexpr (kTmaMask) {
              // pass 0's store of this tile has drained: request the next tile's pass-0 mask into those boxes now, a whole
              // pass ahead of its use
              if (ci == 1 && tile + int(gridDim.x) < num_tiles) issue_mask(tile + int(gridDim.x), 0);
            }
          }
          named_bar_sync(1, Cfg::kEpiWarps * 32);
          if (warp == 0 && lane == 0) {
#pragma unroll
            for (int bx = ci * (kCols / 64); bx < (ci + 1) * (kCols / 64); ++bx)
              if (n0 + 64 * bx < N) tma_store_2d(&tmC, out_tile + bx * (kBlockM * 128), n0 + 64 * bx, m0);
            tma_store_commit();
          }
        }
        continue;
      } else {
        constexpr uint32_t FEAT = kLeanFeat[MODE > 0 ? MODE - 1 : 0];
        // residual / mask operands are fetched one chunk ahead: the first chunk's loads fly while the MMAs of this
        // tile are still running, the others while the previous chunk is being written out
        // (the 16-warp configuration has 96 registers per thread: one prefetch buffer, refilled right after its last
        // use; its four warps per scheduler cover the shorter prefetch distance)
        constexpr int kPre = Cfg::kEpiWarps > 8 ? 1 : 2;
        LeanPre<FEAT> pre[kPre];
        lean_prefetch<FEAT>(pre[0], lane, int(row0), n0 + half * 32, M, N, ep);
        // this lane's bias columns of every chunk of the tile: the shared-memory carve-out leaves L1 too small to keep
        // the bias vector resident next to the residual stream, so a per-chunk load paid L2 latency on the critical path
        float4 bias_pre[BN / kCols];
#pragma unroll
        for (int ci = 0; ci < BN / kCols; ++ci) {
          bias_pre[ci] = make_float4(0.f, 0.f, 0.f, 0.f);
          if constexpr (FEAT & F_BIAS) {
            const int bc = n0 + half * 32 + kCols * ci + 4 * (lane & 7);
            if (bc < N && ep.bias != nullptr) bias_pre[ci] = __ldg(reinterpret_cast<const float4*>(ep.bias + bc));
          }
        }
#pragma unroll
        for (int ci = 0; ci < BN / kCols; ++ci) {
          const int c = half * 32 + kCols * ci;
          if (n0 + c < N) {
            if (kPre == 2 && ci + 1 < BN / kCols)
              lean_prefetch<FEAT>(pre[(ci + 1) & 1], lane, int(row0), n0 + c + kCols, M, N, ep);
            uint32_t v[32];
            acc_to_rows(accum[ci], stage_buf, lane, v);
            epilogue_chunk_lean<FEAT>(v, stage_buf, lane, int(row0), n0 + c, M, N, ep, pre[ci & (kPre - 1)], bias_pre[ci]);
            if (kPre == 1 && ci + 1 < BN / kCols) lean_prefetch<FEAT>(pre[0], lane, int(row0), n0 + c + kCols, M, N, ep);
          }
        }
      }
    }
    if constexpr (lin_tma_out(MODE, NPLANES)) {
      if (warp == 0 && lane == 0) tma_store_wait_all();   // bulk stores must complete before the CTA's smem goes away
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Full-width kernel (lin_wide): persistent over 128 x 256 CTA tiles in the staged kernel's round-robin order.
// Warpgroup 2 produces: one elected lane streams the A [128 x 64] and B [256 x 64] k-blocks of each tile through four
// stages, so B is loaded once per 128 output rows.  Consumer warpgroup g accumulates rows [64 g, 64 g + 64) of the tile
// with one m64n256k16 wgmma per k16 step and runs the epilogue on the accumulator fragments, in which thread (w, lane)
// of the warpgroup holds
//   acc[4 j + 2 i + e] = D[16 w + lane / 4 + 8 i][8 j + 2 (lane % 4) + e]
// i.e. column pairs of two rows; the four lanes of a quad cover 8 contiguous columns of a row.  bf16 outputs go through
// a swizzled two-box ring and leave by TMA store; fp32 outputs and the residual / mask operands are accessed in the
// fragment layout directly.
// ------------------------------------------------------------------------------------------------
template <uint32_t FEAT>
struct WidePre {   // global operands of one 64-column box, [i][jj] = rows (i), column pairs 8 jj + 2 (lane % 4)
  float2 res[(FEAT & F_RES) ? 16 : 1];
  uint32_t mk[(FEAT & F_MASK) ? 16 : 1];
};
template <uint32_t FEAT>
__device__ __forceinline__ void wide_prefetch(WidePre<FEAT>& p, int row0, int col0, int M, int N, const Epi& ep) {
  if constexpr ((FEAT & (F_RES | F_MASK)) != 0) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int row = row0 + 8 * i, col = col0 + 8 * jj;
        const bool ok = row < M && col < N;
        if constexpr (FEAT & F_RES)
          p.res[8 * i + jj] = (ok && ep.residual != nullptr)
                                  ? *reinterpret_cast<const float2*>(ep.residual + size_t(row) * ep.res_ld + col)
                                  : make_float2(0.f, 0.f);
        if constexpr (FEAT & F_MASK)
          p.mk[8 * i + jj] = ok ? *reinterpret_cast<const uint32_t*>(ep.mask + size_t(row) * ep.mask_ld + col) : 0u;
      }
  }
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
// One [64 x 64] bf16 box of a consumer warpgroup's tile -> ring buffer -> TMA store at (c0, r0).  word(i, jj) is this
// thread's column pair jj of row i.  The warpgroup's leader thread issues the stores, so it alone tracks their groups.
template <class Word>
__device__ __forceinline__ void wide_box_out(uint8_t* ring, int& nbox, int bar_id, bool leader, int w, int lane,
                                             const CUtensorMap* tm, int c0, int r0, Word word) {
  if (leader) tma_store_wait_read_n<1>();   // the box stored from this buffer two boxes ago has been read out
  named_bar_sync(bar_id, 128);
  uint8_t* box = ring + (nbox & 1) * WideCfg<0>::kBoxBytes;
  const int rq = lane >> 2;                 // == row & 7: the row's 16-byte chunk swizzle
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    uint8_t* rowp = box + (16 * w + 8 * i + rq) * 128 + 4 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) *reinterpret_cast<uint32_t*>(rowp + ((jj ^ rq) << 4)) = word(i, jj);
  }
  fence_proxy_async_smem();                 // generic-proxy smem writes -> visible to the TMA engine
  named_bar_sync(bar_id, 128);
  if (leader) {
    tma_store_2d(tm, box, c0, r0);
    tma_store_commit();
  }
  ++nbox;
}

template <int MODE>
__device__ __forceinline__ void linear_wide(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, int M,
                                            int N, int K, Epi ep) {
  using Cfg = WideCfg<MODE>;
  // mode 8 is the residual epilogue of mode 4 followed by the LayerNorm of the finished rows (N == 256)
  constexpr uint32_t FEAT = kLeanFeat[(MODE == 8 ? 4 : MODE) - 1];
  constexpr bool kBoxOut = (FEAT & F_OUTA) != 0 || MODE == 8;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* tiles = smem;
  uint8_t* rings = smem + Cfg::kStages * Cfg::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(rings + Cfg::kStagingBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 256) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();   // everything above touched only this CTA's shared memory

  const int n_tiles = (N + 255) / 256;
  const int num_tiles = ((M + kBlockM - 1) / kBlockM) * n_tiles;
  const int num_kb = (K + kBlockK - 1) / kBlockK;

  if (wg == 2) {
    // =================== producer warpgroup: registers go to the consumers, one warp issues ===================
    setmaxnreg_dec<40>();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles && warp == 8; tile += gridDim.x) {
      const int m0 = (tile / n_tiles) * kBlockM;
      const int n0 = (tile % n_tiles) * 256;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* st = tiles + stage * Cfg::kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
#pragma unroll
          for (int r = 0; r < kBlockM; r += 16) tma_load_2d(st + r * 128, &tmA, &full_bar[stage], kb * kBlockK, m0 + r);
          tma_load_2d(st + Cfg::kABytes, &tmB, &full_bar[stage], kb * kBlockK, n0);
        }
        __syncwarp();
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
  // =================== consumer warpgroups ===================
  // 40 (producer) x 128 + 232 x 256 = 64512 registers = 168 (the launch-bounds count) x 384
  setmaxnreg_inc<232>();
  drop_resolve(ep.drop);
  const int w = warp & 3, q = lane & 3;
  const int rloc = 16 * w + (lane >> 2);    // warpgroup-local row of acc[4 j + e]; acc[4 j + 2 + e] is 8 rows further
  const bool leader = (threadIdx.x & 127) == 0;
  uint8_t* ring = rings + wg * 2 * Cfg::kBoxBytes;
  const bool has_bias = (FEAT & F_BIAS) && ep.bias != nullptr;
  const bool has_drop = (FEAT & F_DROP) && ep.drop.p > 0.f;
  const bool has_rv = (FEAT & F_ROWVEC) && ep.rowvec != nullptr;
  int stage = 0;
  uint32_t phase = 0;
  int nbox = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = (tile / n_tiles) * kBlockM;
    const int n0 = (tile % n_tiles) * 256;
    const int row0 = m0 + 64 * wg + rloc;
    float acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0.f;
    int prev_stage = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
      const uint32_t a = smem_u32(tiles + stage * Cfg::kStageBytes) + wg * 8192;
      const uint32_t b = smem_u32(tiles + stage * Cfg::kStageBytes) + Cfg::kABytes;
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)
        wgmma_m64n256_kk(acc, gmma_smem_desc(a + k * 32, 16, 1024), gmma_smem_desc(b + k * 32, 16, 1024));
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();                                    // the previous k-block's MMAs have read their stage
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      }
      prev_stage = stage;
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    // the first box's residual / mask loads fly while the last MMAs finish.  The fp32 residual boxes (32 registers
    // each) are single-buffered, refilled right after their last use, to stay within the register budget.
    constexpr int kPre = (FEAT & F_RES) ? 1 : 2;
    WidePre<FEAT> pre[kPre];
    wide_prefetch<FEAT>(pre[0], row0, n0 + 2 * q, M, N, ep);
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
    if (m0 + 64 * wg < M) {                 // warpgroup-uniform: otherwise all of its rows are past the matrix

      unsigned long long rowq[2];               // dropout quad index of (row, 0); N % 4 == 0 on every lean mode
      uint32_t grp[2];
      float s[2] = {0.f, 0.f}, ss[2] = {0.f, 0.f};   // mode 8: row sums of x1 and x1^2 (this thread's columns)
  #pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = row0 + 8 * i;
        rowq[i] = (unsigned long long)row * (unsigned long long)(N >> 2);
        grp[i] = (has_rv && row < M) ? (ep.rpg_magic ? __umulhi(uint32_t(row), ep.rpg_magic) : uint32_t(row / ep.rows_per_group)) : 0u;
      }
  #pragma unroll
      for (int bx = 0; bx < 4; ++bx) {
        const int c0 = n0 + 64 * bx;            // first column of the box
        if (c0 >= N) break;                     // CTA-uniform
        if (kPre == 2 && bx < 3) wide_prefetch<FEAT>(pre[(bx + 1) & 1], row0, c0 + 64 + 2 * q, M, N, ep);
        const WidePre<FEAT>& p = pre[bx & (kPre - 1)];
  #pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int col = c0 + 8 * jj + 2 * q;  // even; col < N covers col + 1 as N % 4 == 0
          float2 bias = make_float2(0.f, 0.f);
          if (has_bias && col < N) bias = __ldg(reinterpret_cast<const float2*>(ep.bias + col));
  #pragma unroll
          for (int i = 0; i < 2; ++i) {
            float& x0 = acc[4 * (8 * bx + jj) + 2 * i];
            float& x1 = acc[4 * (8 * bx + jj) + 2 * i + 1];
            const int row = row0 + 8 * i;
            if constexpr (FEAT & F_BIAS) { x0 += bias.x; x1 += bias.y; }
            if constexpr (FEAT & F_SCALE) {
              if (col < ep.scale_cols) { x0 *= ep.scale; x1 *= ep.scale; }
            }
            if constexpr (FEAT & F_RELU) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            if constexpr (FEAT & F_DROP) {
              if (has_drop) {   // this pair is half (lane % 2) of quad (row N + col) / 4, as dropout_quad_mult draws it
                const unsigned long long quad = rowq[i] + uint32_t(col >> 2);
                const uint32_t s1 = drop_stage1(uint32_t(quad), drop_hikey(ep.drop, quad));
                const uint32_t h = (q & 1) ? drop_fin_b(s1) : drop_fin_a(s1);
                x0 = drop_keep_lo(h, ep.drop.thr16) ? x0 * ep.drop.scale : 0.f;
                x1 = drop_keep_hi(h, ep.drop.thr16) ? x1 * ep.drop.scale : 0.f;
              }
            }
            if constexpr (FEAT & F_ROWVEC) {
              if (has_rv && row < M && col < N) {
                const float2 rv = __ldg(reinterpret_cast<const float2*>(ep.rowvec + size_t(grp[i]) * ep.rowvec_ld + col));
                x0 += rv.x; x1 += rv.y;
              }
            }
            if constexpr (FEAT & F_MASK) {   // a bf16 is non-zero iff any of its 15 magnitude bits is set
              const uint32_t m = p.mk[8 * i + jj];
              x0 = (m & 0x7FFFu) ? x0 * ep.mask_scale : 0.f;
              x1 = (m & 0x7FFF0000u) ? x1 * ep.mask_scale : 0.f;
            }
            if constexpr (FEAT & F_RES) { x0 += p.res[8 * i + jj].x; x1 += p.res[8 * i + jj].y; }
            if constexpr (FEAT & F_OUTF) {
              if (row < M && col < N) *reinterpret_cast<float2*>(ep.out_f32 + size_t(row) * ep.out_f32_ld + col) = make_float2(x0, x1);
            }
            if constexpr (MODE == 8) {
              s[i] += x0 + x1;
              ss[i] += x0 * x0 + x1 * x1;
            }
          }
        }
        if (kPre == 1 && bx < 3) wide_prefetch<FEAT>(pre[0], row0, c0 + 64 + 2 * q, M, N, ep);
        if constexpr ((FEAT & F_OUTA) != 0) {
          wide_box_out(ring, nbox, 1 + wg, leader, w, lane, &tmC, c0, m0 + 64 * wg, [&](int i, int jj) {
            return pack_bf16x2(acc[4 * (8 * bx + jj) + 2 * i], acc[4 * (8 * bx + jj) + 2 * i + 1]);
          });
        }
      }
      if constexpr (MODE == 8) {
        // a quad holds whole rows: its four lanes' partial sums make the row's
        float sc[2], sh[2];
  #pragma unroll
        for (int i = 0; i < 2; ++i) {
          s[i] += __shfl_xor_sync(0xffffffffu, s[i], 1);
          s[i] += __shfl_xor_sync(0xffffffffu, s[i], 2);
          ss[i] += __shfl_xor_sync(0xffffffffu, ss[i], 1);
          ss[i] += __shfl_xor_sync(0xffffffffu, ss[i], 2);
          const float mean = s[i] * (1.f / 256.f);
          const float rstd = rsqrtf(fmaxf(ss[i] * (1.f / 256.f) - mean * mean, 0.f) + 1e-5f);
          sc[i] = rstd;                          // (x - mean) rstd = x sc + sh
          sh[i] = -mean * rstd;
          const int row = row0 + 8 * i;
          if (q == 0 && row < M) {
            ep.ln_mean[row] = mean;
            ep.ln_rstd[row] = rstd;
          }
        }
  #pragma unroll
        for (int bx = 0; bx < 4; ++bx) {
          wide_box_out(ring, nbox, 1 + wg, leader, w, lane, &tmC, 64 * bx, m0 + 64 * wg, [&](int i, int jj) {
            const int col = 64 * bx + 8 * jj + 2 * q;
            const float2 g = __ldg(reinterpret_cast<const float2*>(ep.ln_gamma + col));
            const float2 be = __ldg(reinterpret_cast<const float2*>(ep.ln_beta + col));
            const float x0 = acc[4 * (8 * bx + jj) + 2 * i], x1 = acc[4 * (8 * bx + jj) + 2 * i + 1];
            return pack_bf16x2((x0 * sc[i] + sh[i]) * g.x + be.x, (x1 * sc[i] + sh[i]) * g.y + be.y);
          });
        }
      }
    }
    // bulk stores must complete before the CTA's smem goes away.  Waited for inside the tile loop: after the loop, the
    // wait costs the consumer warpgroups their setmaxnreg budget (ptxas then allocates 168 registers).
    if (kBoxOut && w == 0 && tile + int(gridDim.x) >= num_tiles) tma_store_wait_all();
  }
  }
}

template <int BN, int NPLANES, int MODE>
__global__ void __launch_bounds__((LinearCfg<BN, NPLANES, MODE>::kThreads), 1)
linear_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmAlo,
              const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmBlo,
              const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmM, int M, int N, int K,
              Epi ep) {
  if constexpr (lin_wide(MODE, BN, NPLANES))
    linear_wide<MODE>(tmA, tmB, tmC, M, N, K, ep);
  else
    linear_staged<BN, NPLANES, MODE>(tmA, tmAlo, tmB, tmBlo, tmC, tmM, M, N, K, ep);
}

// 16-byte vector reduction (REDG.E.ADD.F32x4): four consecutive fp32 gradient entries per instruction
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// One 32 x 32 accumulator chunk of an outer-product consumer warp -> C[p, col0 + j] += alpha * chunk.
// a[h] = fragment of the m64 half h: local row 16 h + r (r < 16) of the chunk is P row prow0 + 64 h + r.
// Transposed through the warp's staging tile so that 8 lanes cover one 128-byte row segment; the vector path needs
// ldc % 4 == 0, Q % 4 == 0 and a 16-byte aligned C.
__device__ __forceinline__ void outer_chunk(const float (&a)[2][16], uint32_t stage_addr, int lane, int prow0, int col0,
                                            int P, int Q, float alpha, float* C, int ldc, int vec) {
  __syncwarp();
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int lr = 16 * h + 8 * i + (lane >> 2), col = 8 * j + 2 * (lane & 3);
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stage_addr + (lr * kStageRow + col) * 4),
                     "f"(a[h][4 * j + 2 * i]), "f"(a[h][4 * j + 2 * i + 1]) : "memory");
      }
  __syncwarp();
  if (vec) {
    const int cg = lane & 7, rsub = lane >> 3;
    const int col = col0 + 4 * cg;
    if (col < Q) {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int lr = rsub + 4 * it;
        const int prow = prow0 + 64 * (lr >> 4) + (lr & 15);
        const float4 x = ld_shared_v4(stage_addr + (lr * kStageRow + 4 * cg) * 4);
        if (prow < P) red_add_v4(C + size_t(prow) * ldc + col, x.x * alpha, x.y * alpha, x.z * alpha, x.w * alpha);
      }
    }
  } else {
    const int col = col0 + lane;
#pragma unroll 4
    for (int lr = 0; lr < 32; ++lr) {
      const int prow = prow0 + 64 * (lr >> 4) + (lr & 15);
      const float x = ld_shared_f32(stage_addr + (lr * kStageRow + lane) * 4);
      if (prow < P && col < Q) atomicAdd(C + size_t(prow) * ldc + col, x * alpha);
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// dsvg_outer kernel (MN-major operands): output tiles [128 x BQ], each a sum of contractions over row ranges (chunks)
// ------------------------------------------------------------------------------------------------
// Warpgroup g (warps 4 g .. 4 g + 3) accumulates all 128 P rows (two m64 halves) against Q columns
// [g BQ / 2, (g + 1) BQ / 2) in registers; warpgroup 0 also sums the A columns (bias gradient) with an n8 wgmma
// against an all-ones operand.  The last warp is the TMA producer.  Single-plane operands run persistent CTAs over
// (tile, chunk) work items (outer_persistent); two-plane operands one (tile, chunk) per CTA (outer_body).
template <int BQ, int NPLANES>
struct OuterCfg {
  static constexpr int kBoxBytes = 64 * 64 * 2;                 // [64 rows(m) x 64 cols] = 8 KB
  static constexpr int kABytes = 2 * kBoxBytes;                 // 128 P columns
  static constexpr int kBBytes = (BQ / 64) * kBoxBytes;         // BQ Q columns
  static constexpr int kStageBytes = NPLANES * (kABytes + kBBytes);
  static constexpr int kStages = (NPLANES == 1) ? 4 : 2;
  static constexpr int kOnesBytes = 1024;   // [8 x 64] bf16 1.0, K-major B operand of the column-sum wgmma
  // 8 consumer warps.  In the two-plane kernel their transposition buffers alias the operand stages: the epilogue starts
  // once every consumer warp has retired its last wgmma, and by then every TMA load has landed.
  static constexpr int kEpiWarps = 8;
  // one producer warp; the persistent single-plane kernel gives it a whole warpgroup, to hand the consumers its registers
  static constexpr int kThreads = 32 * kEpiWarps + (NPLANES == 1 ? 128 : 32);
  static constexpr int kNW = BQ / 2;   // Q columns per warpgroup
  static_assert(kEpiWarps * kStageWarpBytes <= kStages * kStageBytes, "outer: staging must fit in the operand stages");
  // + the persistent kernel's 16-row staging tile per consumer warp
  static constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kOnesBytes + 256 +
                                    (NPLANES == 1 ? kEpiWarps * kStageWarpBytes / 2 : 0);
  static_assert(kSmemBytes <= 227 * 1024, "outer: shared memory over the per-block limit of sm_90");
};

// The whole CTA program of the two-plane kernel; `tile_id` / `split_id` (the block indices) select the output tile and the
// M range.  The tensor maps live in kernel-parameter space (__grid_constant__) of the caller.
template <int BQ, int NPLANES>
__device__ __forceinline__ void outer_body(const CUtensorMap* tmA_p, const CUtensorMap* tmAlo_p, const CUtensorMap* tmB_p,
                                           const CUtensorMap* tmBlo_p, int M, int P, int Q, int mblk_per_split, float alpha,
                                           const float* alpha_dev, float* C, int ldc, float* colsum_out, uint32_t lbo,
                                           uint32_t sbo, int vec, int tile_id, int split_id) {
  using Cfg = OuterCfg<BQ, NPLANES>;
  constexpr int kNW = Cfg::kNW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* tiles = smem;
  uint8_t* ones = smem + Cfg::kStages * Cfg::kStageBytes;  // 1024-aligned
  const int q_tiles = (Q + BQ - 1) / BQ;
  const bool do_colsum = colsum_out != nullptr && (tile_id % q_tiles) == 0;
  float* staging = reinterpret_cast<float*>(tiles);   // epilogue only, after the main loop (see OuterCfg)
  uint64_t* bars = reinterpret_cast<uint64_t*>(ones + Cfg::kOnesBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kProducer = Cfg::kEpiWarps;

  if (warp == kProducer && lane == 0) {
    tma_prefetch_desc(tmA_p);
    tma_prefetch_desc(tmB_p);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], Cfg::kEpiWarps);
    }
    fence_barrier_init();
  }
  // bf16 1.0 everywhere: the layout of an all-ones operand is irrelevant, only the descriptor must be valid
  for (int i = threadIdx.x; i < Cfg::kOnesBytes / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(ones)[i] = 0x3F803F80u;
  fence_proxy_async_smem();
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();   // everything above touched only this CTA's shared memory

  const int p0 = (tile_id / q_tiles) * 128;
  const int q0 = (tile_id % q_tiles) * BQ;
  const int total_mblk = (M + 63) / 64;
  const int mb_begin = split_id * mblk_per_split;
  const int mb_end = min(total_mblk, mb_begin + mblk_per_split);
  const int num_mb = mb_end - mb_begin;  // >= 1 by construction of the grid

  if (warp == kProducer) {
    int stage = 0;
    uint32_t phase = 0;
    for (int mb = mb_begin; mb < mb_end; ++mb) {
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (elect_one()) {
        uint8_t* st = tiles + stage * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
#pragma unroll
        for (int i = 0; i < 2; ++i) tma_load_2d(st + i * Cfg::kBoxBytes, tmA_p, &full_bar[stage], p0 + 64 * i, mb * 64);
#pragma unroll
        for (int j = 0; j < BQ / 64; ++j)
          tma_load_2d(st + Cfg::kABytes + j * Cfg::kBoxBytes, tmB_p, &full_bar[stage], q0 + 64 * j, mb * 64);
        if (NPLANES == 2) {
          uint8_t* lo = st + Cfg::kABytes + Cfg::kBBytes;
#pragma unroll
          for (int i = 0; i < 2; ++i)
            tma_load_2d(lo + i * Cfg::kBoxBytes, tmAlo_p, &full_bar[stage], p0 + 64 * i, mb * 64);
#pragma unroll
          for (int j = 0; j < BQ / 64; ++j)
            tma_load_2d(lo + Cfg::kABytes + j * Cfg::kBoxBytes, tmBlo_p, &full_bar[stage], q0 + 64 * j, mb * 64);
        }
      }
      __syncwarp();
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    return;
  }

  const int quarter = warp & 3;   // warp within its warpgroup: P rows [16 quarter, +16) of each m64 half
  const int half = warp >> 2;     // warpgroup: Q columns [half * kNW, (half + 1) * kNW)
  float acc[2][kNW / 2];
  float cs[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int j = 0; j < kNW / 2; ++j) acc[h][j] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) cs[h][j] = 0.f;
  }
  const uint64_t ones_desc = gmma_smem_desc(smem_u32(ones), 16, 1024);
  int stage = 0, prev_stage = 0;
  uint32_t phase = 0;
  for (int i = 0; i < num_mb; ++i) {
    mbar_wait(&full_bar[stage], phase);
    wgmma_fence();
    const uint32_t a_hi = smem_u32(tiles + stage * Cfg::kStageBytes);
    const uint32_t b_hi = a_hi + Cfg::kABytes + half * (kNW / 64) * Cfg::kBoxBytes;
    const uint32_t a_lo = a_hi + Cfg::kABytes + Cfg::kBBytes;
    const uint32_t b_lo = a_lo + Cfg::kABytes + half * (kNW / 64) * Cfg::kBoxBytes;
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // 16 rows (= 2 KB) of the 64-row block per k16 step
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t ao = h * Cfg::kBoxBytes + k * 2048, bo = k * 2048;
        wgmma_m64_tt<kNW>(acc[h], gmma_smem_desc(a_hi + ao, lbo, sbo), gmma_smem_desc(b_hi + bo, lbo, sbo));
        if (NPLANES == 2) {
          wgmma_m64_tt<kNW>(acc[h], gmma_smem_desc(a_hi + ao, lbo, sbo), gmma_smem_desc(b_lo + bo, lbo, sbo));
          wgmma_m64_tt<kNW>(acc[h], gmma_smem_desc(a_lo + ao, lbo, sbo), gmma_smem_desc(b_hi + bo, lbo, sbo));
        }
        // issued unconditionally (a wgmma under a run-time branch makes ptxas serialise all of them, C7520); only
        // warpgroup 0 of a CTA that owns the first Q tile writes the sums out
        wgmma_m64n8_tk(cs[h], gmma_smem_desc(a_hi + ao, lbo, sbo), ones_desc);
        if (NPLANES == 2) wgmma_m64n8_tk(cs[h], gmma_smem_desc(a_lo + ao, lbo, sbo), ones_desc);
      }
    }
    wgmma_commit();
    if (i > 0) {
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
    }
    prev_stage = stage;
    if (++stage == Cfg::kStages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    wgmma_fence_regs(acc[h]);
    wgmma_fence_regs(cs[h]);
  }
  // the transposition buffers alias the operand stages: every consumer warp must be done reading them
  named_bar_sync(1, Cfg::kEpiWarps * 32);
  if (alpha_dev != nullptr) alpha *= __ldg(alpha_dev);
  const uint32_t stage_buf = smem_u32(staging) + warp * kStageWarpBytes;
  const int prow0 = p0 + 16 * quarter;
#pragma unroll
  for (int cc = 0; cc < kNW / 32; ++cc) {
    const int col0 = q0 + half * kNW + 32 * cc;
    if (col0 >= Q) break;
    float a2[2][16];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 16; ++j) a2[h][j] = acc[h][16 * cc + j];
    outer_chunk(a2, stage_buf, lane, prow0, col0, P, Q, alpha, C, ldc, vec);
  }
  if (do_colsum && half == 0 && (lane & 3) == 0) {   // column 0 of the [128 x 8] column-sum tile = sum over this CTA's rows of A[:, p]
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int prow = prow0 + 64 * h + 8 * i + (lane >> 2);
        if (prow < P) atomicAdd(colsum_out + prow, cs[h][2 * i] * alpha);
      }
  }
}

// The problems of one launch: a single dsvg_outer call, or the weight gradients of one transformer block (QKV, out-proj,
// FFN1, FFN2: same row count M, different operands) from dsvg_outer_group, which then share one persistent grid instead of
// paying a pipeline ramp and a ragged last wave per launch.  Work item w of the single-plane kernel is (chunk w / T,
// tile w % T), T = tile_begin[n] output tiles of 128 x BQ over all problems, a chunk = mblk_per_chunk row blocks of 64 rows.
constexpr int kMaxGroup = 4;
struct OuterGroup {
  CUtensorMap a[kMaxGroup];
  CUtensorMap b[kMaxGroup];
  CUtensorMap alo, blo;            // two-plane launches (always one problem): the low planes of a[0] / b[0]
  float* C[kMaxGroup];
  float* colsum[kMaxGroup];
  const float* alpha_dev[kMaxGroup];
  float alpha[kMaxGroup];
  int P[kMaxGroup], Q[kMaxGroup], ldc[kMaxGroup], vec[kMaxGroup];
  int tile_begin[kMaxGroup + 1];   // first output tile of each problem; tile_begin[n] = T
  int n, M, chunks, mblk_per_chunk;
};

// One 64-row half of a consumer warp's accumulators (P rows prow + [0, 16)) -> C[row, col0 + ...] += alpha * acc, in
// 32-column chunks through the warp's 16-row staging tile: eight lanes then cover one 128-byte row segment with 16-byte
// reductions (ldc % 4 == 0, Q % 4 == 0 and a 16-byte aligned C), or 32 lanes one with scalar ones (gradient slices at odd
// offsets of a flat bucket).  Straight from the fragments, a reduction instruction would touch 16 rows (measured slower
// where the reductions are not hidden behind long row chunks: 4096-row weight gradients).
template <int NV>
__device__ __forceinline__ void outer_red_half(const float (&acc)[NV], uint32_t stage_addr, int lane, int prow, int col0, int P,
                                               int Q, float alpha, float* C, int ldc, int vec) {
#pragma unroll
  for (int cc = 0; cc < NV / 16; ++cc) {
    if (col0 + 32 * cc >= Q) break;   // warp-uniform
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int lr = 8 * i + (lane >> 2), col = 8 * j + 2 * (lane & 3);
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stage_addr + (lr * kStageRow + col) * 4),
                     "f"(acc[16 * cc + 4 * j + 2 * i]), "f"(acc[16 * cc + 4 * j + 2 * i + 1]) : "memory");
      }
    __syncwarp();
    if (vec) {
      const int cg = lane & 7, col = col0 + 32 * cc + 4 * cg;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int lr = (lane >> 3) + 4 * it;
        const float4 x = ld_shared_v4(stage_addr + (lr * kStageRow + 4 * cg) * 4);
        if (prow + lr < P && col < Q)
          red_add_v4(C + size_t(prow + lr) * ldc + col, x.x * alpha, x.y * alpha, x.z * alpha, x.w * alpha);
      }
    } else {
      const int col = col0 + 32 * cc + lane;
#pragma unroll 4
      for (int lr = 0; lr < 16; ++lr) {
        const float x = ld_shared_f32(stage_addr + (lr * kStageRow + lane) * 4);
        if (prow + lr < P && col < Q) atomicAdd(C + size_t(prow + lr) * ldc + col, x * alpha);
      }
    }
  }
  __syncwarp();
}

// Single-plane operands: a persistent grid (at most one CTA per SM) walks the launch's work items in chunk-major order, so
// the CTAs that read the same rows of a shared operand (the same A for the Q tiles of one P range, the same B for the P
// tiles) stream them at about the same time and L2 serves all but the first read.  Each output element is still the sum of
// per-chunk fp32 wgmma chains of at most kMaxSplitBlocks row blocks, added with red.add.  The producer warp runs ahead into
// the next item's row blocks while the consumer warps reduce the current one from their registers.
template <int BQ>
__device__ __forceinline__ void outer_persistent(const OuterGroup& g, uint32_t lbo, uint32_t sbo) {
  using Cfg = OuterCfg<BQ, 1>;
  constexpr int kNW = Cfg::kNW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* tiles = smem;
  uint8_t* ones = smem + Cfg::kStages * Cfg::kStageBytes;  // 1024-aligned
  uint64_t* bars = reinterpret_cast<uint64_t*>(ones + Cfg::kOnesBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;
  uint8_t* staging = reinterpret_cast<uint8_t*>(bars) + 256;   // the consumer warps' own, the stages stay in flight

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kProducer = Cfg::kEpiWarps;

  if (warp == kProducer && lane == 0) {
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], Cfg::kEpiWarps);
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < Cfg::kOnesBytes / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(ones)[i] = 0x3F803F80u;
  fence_proxy_async_smem();
  __syncthreads();
  pdl_wait();   // everything above touched only this CTA's shared memory

  const int T = g.tile_begin[g.n];
  const int items = T * g.chunks;
  const int total_mblk = (g.M + 63) / 64;
  // work item -> problem p, output tile origin (p0, q0), row blocks [mb_begin, mb_end)
  auto decode = [&](int w, int& p, int& p0, int& q0, int& mb_begin, int& mb_end) {
    const int chunk = w / T;
    int t = w - chunk * T;
    p = 0;
    while (p + 1 < g.n && t >= g.tile_begin[p + 1]) ++p;
    t -= g.tile_begin[p];
    const int q_tiles = (g.Q[p] + BQ - 1) / BQ;
    p0 = (t / q_tiles) * 128;
    q0 = (t % q_tiles) * BQ;
    mb_begin = chunk * g.mblk_per_chunk;
    mb_end = min(total_mblk, mb_begin + g.mblk_per_chunk);
  };

  if (warp >= kProducer) {
    // producer warpgroup: registers go to the consumers (40 x 128 + 232 x 256 = 64512), one warp issues
    setmaxnreg_dec<40>();
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < items && warp == kProducer; w += gridDim.x) {
      // the next kernel may launch once every CTA is on its last item: earlier, its CTAs would only wait for SMs
      if (w + int(gridDim.x) >= items) pdl_launch_dependents();
      int p, p0, q0, mb_begin, mb_end;
      decode(w, p, p0, q0, mb_begin, mb_end);
      for (int mb = mb_begin; mb < mb_end; ++mb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          uint8_t* st = tiles + stage * Cfg::kStageBytes;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
#pragma unroll
          for (int i = 0; i < 2; ++i) tma_load_2d(st + i * Cfg::kBoxBytes, &g.a[p], &full_bar[stage], p0 + 64 * i, mb * 64);
#pragma unroll
          for (int j = 0; j < BQ / 64; ++j)
            tma_load_2d(st + Cfg::kABytes + j * Cfg::kBoxBytes, &g.b[p], &full_bar[stage], q0 + 64 * j, mb * 64);
        }
        __syncwarp();
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const uint32_t stage_buf = smem_u32(staging) + warp * (kStageWarpBytes / 2);
  const int quarter = warp & 3;   // warp within its warpgroup: P rows [16 quarter, +16) of each m64 half
  const int half = warp >> 2;     // warpgroup: Q columns [half * kNW, (half + 1) * kNW)
  const uint64_t ones_desc = gmma_smem_desc(smem_u32(ones), 16, 1024);
  int stage = 0;
  uint32_t phase = 0;
  for (int w = blockIdx.x; w < items; w += gridDim.x) {
    if (w + int(gridDim.x) >= items) pdl_launch_dependents();
    int p, p0, q0, mb_begin, mb_end;
    decode(w, p, p0, q0, mb_begin, mb_end);
    float acc[2][kNW / 2];
    float cs[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < kNW / 2; ++j) acc[h][j] = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) cs[h][j] = 0.f;
    }
    int prev_stage = 0;
    for (int mb = mb_begin; mb < mb_end; ++mb) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
      const uint32_t a_hi = smem_u32(tiles + stage * Cfg::kStageBytes);
      const uint32_t b_hi = a_hi + Cfg::kABytes + half * (kNW / 64) * Cfg::kBoxBytes;
#pragma unroll
      for (int k = 0; k < 4; ++k) {  // 16 rows (= 2 KB) of the 64-row block per k16 step
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t ao = h * Cfg::kBoxBytes + k * 2048;
          wgmma_m64_tt<kNW>(acc[h], gmma_smem_desc(a_hi + ao, lbo, sbo), gmma_smem_desc(b_hi + k * 2048, lbo, sbo));
          // issued unconditionally (a wgmma under a run-time branch makes ptxas serialise all of them, C7520); only
          // warpgroup 0 of an item on the first Q tile writes the sums out
          wgmma_m64n8_tk(cs[h], gmma_smem_desc(a_hi + ao, lbo, sbo), ones_desc);
        }
      }
      wgmma_commit();
      if (mb > mb_begin) {
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      }
      prev_stage = stage;
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      wgmma_fence_regs(acc[h]);
      wgmma_fence_regs(cs[h]);
    }
    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);   // the producer refills it for the next item during the reduction

    const int P = g.P[p], Q = g.Q[p];
    float alpha = g.alpha[p];
    if (g.alpha_dev[p] != nullptr) alpha *= __ldg(g.alpha_dev[p]);
    const int prow0 = p0 + 16 * quarter;
    const int col0 = q0 + half * kNW;
    if (col0 < Q) {   // warp-uniform
#pragma unroll
      for (int h = 0; h < 2; ++h)
        outer_red_half(acc[h], stage_buf, lane, prow0 + 64 * h, col0, P, Q, alpha, g.C[p], g.ldc[p], g.vec[p]);
    }
    if (g.colsum[p] != nullptr && q0 == 0 && half == 0 && (lane & 3) == 0) {
      // column 0 of the [128 x 8] column-sum tile = sum over this chunk's rows of A[:, p]
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int prow = prow0 + 64 * h + 8 * i + (lane >> 2);
          if (prow < P) atomicAdd(g.colsum[p] + prow, cs[h][2 * i] * alpha);
        }
    }
  }
}

template <int BQ, int NPLANES>
__global__ void __launch_bounds__((OuterCfg<BQ, NPLANES>::kThreads), 1)
outer_kernel(const __grid_constant__ OuterGroup g, uint32_t lbo, uint32_t sbo) {
  if constexpr (NPLANES == 1)
    outer_persistent<BQ>(g, lbo, sbo);
  else
    outer_body<BQ, NPLANES>(&g.a[0], &g.alo, &g.b[0], &g.blo, g.M, g.P[0], g.Q[0], g.mblk_per_chunk, g.alpha[0],
                            g.alpha_dev[0], g.C[0], g.ldc[0], g.colsum[0], lbo, sbo, g.vec[0], int(blockIdx.x),
                            int(blockIdx.y));
}

static int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int BN, int NPLANES, int MODE>
static int launch_linear_mode(const CUtensorMap& a, const CUtensorMap& alo, const CUtensorMap& b, const CUtensorMap& blo,
                              int M, int N, int K, const Epi& ep, cudaStream_t st) {
  CUtensorMap c = a, mk = a;
  if (lin_wide(MODE, BN, NPLANES)) {   // 64 x 64 output boxes, one consumer warpgroup's rows each
    if (MODE == 8) {
      if (make_map(&c, ep.ln_out, 256, M, 256, 64, 64)) return 1;
    } else if (lin_tma_out(MODE, NPLANES)) {
      if (make_map(&c, ep.out_act, N, M, ep.out_act_ld, 64, 64)) return 1;
    }
  } else if (lin_tma_out(MODE, NPLANES)) {
    if (make_map(&c, ep.out_act, N, M, ep.out_act_ld, 64, 128)) return 1;
    if (ep.mask != nullptr && make_map(&mk, ep.mask, N, M, ep.mask_ld, 64, 128)) return 1;
  }
  using Cfg = LinearCfg<BN, NPLANES, MODE>;
  static bool configured[kMaxDevices] = {};
  if (first_use_on_device(configured)) {
    DSVG_CUDA(cudaFuncSetAttribute(linear_kernel<BN, NPLANES, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   Cfg::kSmemBytes));
  }
  const int tiles = ceil_div(M, kBlockM) * ceil_div(N, BN);
  const int slots = sm_count();
  const int grid = tiles < slots ? tiles : slots;
  DSVG_CUDA(launch_k(linear_kernel<BN, NPLANES, MODE>, dim3(grid), dim3(Cfg::kThreads), Cfg::kSmemBytes, st, a, alo, b, blo, c, mk,
                     M, N, K, ep));
  ++g_launches;
  return 0;
}
template <int BN>
static int launch_linear_fast(const CUtensorMap& a, const CUtensorMap& b, int M, int N, int K, const Epi& ep,
                              cudaStream_t st) {
  switch (ep.mode) {
    case 1: return launch_linear_mode<BN, 1, 1>(a, a, b, b, M, N, K, ep, st);
    case 2: return launch_linear_mode<BN, 1, 2>(a, a, b, b, M, N, K, ep, st);
    case 3: return launch_linear_mode<BN, 1, 3>(a, a, b, b, M, N, K, ep, st);
    case 4: return launch_linear_mode<BN, 1, 4>(a, a, b, b, M, N, K, ep, st);
    case 5: return launch_linear_mode<BN, 1, 5>(a, a, b, b, M, N, K, ep, st);
    case 6: return launch_linear_mode<BN, 1, 6>(a, a, b, b, M, N, K, ep, st);
    case 7: return launch_linear_mode<BN, 1, 7>(a, a, b, b, M, N, K, ep, st);
    default: return launch_linear_mode<BN, 1, 0>(a, a, b, b, M, N, K, ep, st);
  }
}

// parity mode (two bf16 planes per operand, 128-wide tiles): the same lean feature sets, staged per-warp epilogue
static int launch_linear_split(const CUtensorMap& a, const CUtensorMap& alo, const CUtensorMap& b, const CUtensorMap& blo, int M,
                               int N, int K, const Epi& ep, cudaStream_t st) {
  switch (ep.mode) {
    case 1: return launch_linear_mode<128, 2, 1>(a, alo, b, blo, M, N, K, ep, st);
    case 2: return launch_linear_mode<128, 2, 2>(a, alo, b, blo, M, N, K, ep, st);
    case 3: return launch_linear_mode<128, 2, 3>(a, alo, b, blo, M, N, K, ep, st);
    case 4: return launch_linear_mode<128, 2, 4>(a, alo, b, blo, M, N, K, ep, st);
    case 5: return launch_linear_mode<128, 2, 5>(a, alo, b, blo, M, N, K, ep, st);
    case 6: return launch_linear_mode<128, 2, 6>(a, alo, b, blo, M, N, K, ep, st);
    case 7: return launch_linear_mode<128, 2, 7>(a, alo, b, blo, M, N, K, ep, st);
    default: return launch_linear_mode<128, 2, 0>(a, alo, b, blo, M, N, K, ep, st);
  }
}

// which lean epilogue (if any) covers exactly the requested steps
static int pick_mode(const Epi& ep, bool split, int N) {
  if (ep.vec == 0) {   // unaligned rows: only the plain "acc + bias -> fp32" head epilogue has a lean version
    const bool plain = ep.out_f32 && !ep.out_act && !ep.acc_scale_dev && ep.scale_cols == 0 && !ep.relu &&
                       !(ep.drop.p > 0.f) && !ep.rowvec && !ep.mask && !ep.residual;
    return plain ? 7 : 0;
  }
  if (!split && (ep.mask_lo_off != 0 || ep.out_lo_off != 0)) return 0;   // single-plane operands with two-plane outputs: generic
  uint32_t f = 0;
  if (ep.acc_scale_dev) f |= F_ACCS;
  if (ep.bias) f |= F_BIAS;
  if (ep.scale_cols > 0) f |= F_SCALE;
  if (ep.relu) f |= F_RELU;
  if (ep.drop.p > 0.f) f |= F_DROP;
  if (ep.rowvec) f |= F_ROWVEC;
  if (ep.mask) f |= F_MASK;
  if (ep.residual) f |= F_RES;
  if (ep.out_f32) f |= F_OUTF;
  if (ep.out_act) f |= F_OUTA;
  if ((f & F_SCALE) && ep.scale_cols % 4 != 0) return 0;
  for (int k = 0; k < kNumLean; ++k) {
    const uint32_t have = kLeanFeat[k];
    // steps that the lean code checks at run time (warp-uniform branches): dropout, row vector; and for the fp32 output
    // mode 4 also bias and residual, so that it covers the latent / group-level "global" linears and their dgrads
    const uint32_t optional = have & (F_DROP | F_ROWVEC | ((have & F_OUTF) && !(have & F_ACCS) ? (F_BIAS | F_RES) : 0u));
    if ((f & ~optional) == (have & ~optional) && (f & ~have) == 0) {
      if (lin_tma_out(k + 1, split ? 2 : 1)) {
        const bool ok = N % 8 == 0 && ep.out_act_ld % 8 == 0 && ep.scale_cols % 32 == 0 && (reinterpret_cast<uintptr_t>(ep.out_act) & 15) == 0 &&
                        (!ep.mask || (ep.mask_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(ep.mask) & 15) == 0)) &&
                        (!ep.bias || (reinterpret_cast<uintptr_t>(ep.bias) & 15) == 0);
        if (!ok) return 0;
      }
      return k + 1;
    }
  }
  return 0;
}

// At most this many 64-row blocks per split of the contraction: the wgmma accumulates a split's rows in fp32 inside the
// tensor core, and shorter chains keep the weight gradients of long row ranges (M ~ 131072) within 2e-5 of an fp64 sum.
constexpr int kMaxSplitBlocks = 48;

// Fills g.chunks / g.mblk_per_chunk and launches.  Two-plane: one CTA per (tile, chunk), as many chunks as fill one wave.
// Single-plane (persistent): the chunk count that minimises the launch's makespan, counted in row blocks per CTA plus one
// per work item for its reduction, e.g. the hier block's 16 tiles at M = 131072 in 49 chunks of 42 row blocks (784 items,
// 5.94 per SM) rather than 43 of 48 (688 items, 5.2 per SM: a last round on a fifth of the machine).
template <int BQ, int NPLANES>
static int launch_outer(OuterGroup& g, cudaStream_t st) {
  using Cfg = OuterCfg<BQ, NPLANES>;
  static bool configured[kMaxDevices] = {};
  if (first_use_on_device(configured)) {
    DSVG_CUDA((cudaFuncSetAttribute(outer_kernel<BQ, NPLANES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    Cfg::kSmemBytes)));
  }
  const int tiles = g.tile_begin[g.n];
  const int total_mblk = ceil_div(g.M, 64);
  const int min_chunks = ceil_div(total_mblk, kMaxSplitBlocks);
  const int max_chunks = total_mblk / 4 > min_chunks ? total_mblk / 4 : min_chunks;   // >= 4 blocks of 64 rows per chunk
  dim3 grid;
  if (NPLANES == 2) {
    int splits = sm_count() / tiles;  // one CTA per SM fits (shared memory): fill exactly one wave, no ragged tail
    if (splits < min_chunks) splits = min_chunks;
    if (splits > max_chunks) splits = max_chunks;
    g.mblk_per_chunk = ceil_div(total_mblk, splits);
    g.chunks = ceil_div(total_mblk, g.mblk_per_chunk);
    grid = dim3(tiles, g.chunks);
  } else {
    long long best = -1;
    for (int c = min_chunks; c <= max_chunks; ++c) {
      const int per = ceil_div(total_mblk, c), chunks = ceil_div(total_mblk, per);
      const long long span = (long long)ceil_div(tiles * chunks, sm_count()) * (per + 1);
      if (best < 0 || span < best) {
        best = span;
        g.mblk_per_chunk = per;
        g.chunks = chunks;
      }
    }
    const int items = tiles * g.chunks;
    grid = dim3(items < sm_count() ? items : sm_count());
  }
  DSVG_CUDA(launch_k(outer_kernel<BQ, NPLANES>, grid, dim3(Cfg::kThreads), Cfg::kSmemBytes, st, g,
                     uint32_t(Cfg::kBoxBytes), 1024u));
  ++g_launches;
  return 0;
}

static void outer_problem(OuterGroup& g, int i, const float* alpha_dev, float alpha, float* C, int ldc, float* colsum,
                          int P, int Q, int BQ) {
  g.C[i] = C; g.colsum[i] = colsum; g.alpha_dev[i] = alpha_dev; g.alpha[i] = alpha;
  g.P[i] = P; g.Q[i] = Q; g.ldc[i] = ldc;
  g.vec[i] = int(ldc % 4 == 0 && Q % 4 == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0);
  g.tile_begin[i + 1] = g.tile_begin[i] + ceil_div(P, 128) * ceil_div(Q, BQ);
}

}  // namespace dsvg

using namespace dsvg;

extern "C" const char* dsvg_last_error(void) { return dsvg::last_error(); }
extern "C" int dsvg_abi_version(void) { return 6; }
extern "C" unsigned long long dsvg_launch_count(void) { return dsvg::g_launches; }

static int fill_epi(Epi& ep, const dsvg_epilogue* e, int M, int N) {
  ep.acc_scale_dev = e->acc_scale_dev;
  ep.bias = e->bias;
  ep.scale_cols = e->scale_cols;
  ep.scale = e->scale;
  ep.relu = e->relu;
  ep.drop = make_dropout(e->drop_p, e->drop_site, e->seed);
  ep.rowvec = e->rowvec;
  ep.rowvec_ld = e->rowvec_ld;
  ep.rows_per_group = e->rows_per_group > 0 ? e->rows_per_group : 1;
  ep.rpg_magic = 0;
  if (ep.rows_per_group > 1 && (unsigned long long)M * ep.rows_per_group < (1ull << 32))
    ep.rpg_magic = uint32_t(((1ull << 32) + ep.rows_per_group - 1) / ep.rows_per_group);
  ep.mask = reinterpret_cast<const bf16*>(e->mask);
  ep.mask_lo_off = e->mask_lo_off;
  ep.mask_ld = e->mask_ld;
  ep.mask_scale = e->mask_scale;
  ep.residual = e->residual;
  ep.res_ld = e->res_ld;
  ep.out_f32 = e->out_f32;
  ep.out_f32_ld = e->out_f32_ld;
  ep.out_act = reinterpret_cast<bf16*>(e->out_act);
  ep.out_lo_off = e->out_lo_off;
  ep.out_act_ld = e->out_act_ld;
  {
    auto al = [](const void* p, size_t a) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) % a) == 0; };
    bool v = (N % 4 == 0) && al(ep.bias, 16) && al(ep.rowvec, 16) && al(ep.residual, 16) && al(ep.out_f32, 16) &&
             al(ep.mask, 8) && al(ep.out_act, 8);
    v = v && (!ep.rowvec || ep.rowvec_ld % 4 == 0) && (!ep.residual || ep.res_ld % 4 == 0) &&
        (!ep.out_f32 || ep.out_f32_ld % 4 == 0) && (!ep.mask || (ep.mask_ld % 4 == 0 && ep.mask_lo_off % 4 == 0)) &&
        (!ep.out_act || (ep.out_act_ld % 4 == 0 && ep.out_lo_off % 4 == 0));
    ep.vec = v ? 1 : 0;
  }
  return 0;
}

extern "C" int dsvg_linear(const dsvg_bf16* X, size_t x_lo_off, int lda, const dsvg_bf16* W, size_t w_lo_off, int ldb,
                           int M, int N, int K, const dsvg_epilogue* e, void* stream) {
  DSVG_CHECK(X && W && e, "dsvg_linear: null pointer");
  DSVG_CHECK(M > 0 && N > 0 && K > 0, "dsvg_linear: bad shape %d x %d x %d", M, N, K);
  DSVG_CHECK(lda % 8 == 0 && ldb % 8 == 0, "dsvg_linear: lda/ldb must be multiples of 8 elements (TMA row stride)");
  DSVG_CHECK((x_lo_off == 0) == (w_lo_off == 0), "dsvg_linear: both operands must have the same number of planes");
  Epi ep{};
  if (fill_epi(ep, e, M, N)) return 1;
  DSVG_CHECK(ep.out_f32 || ep.out_act, "dsvg_linear: no output requested");
  const bool split = x_lo_off != 0;
  // 256-wide tiles for the big path-level GEMMs; the group-level ones (M = N_icons * 8 rows, a few dozen tiles) run the
  // 128-wide kernel: twice the CTAs and two CTAs per SM shorten their latency-bound critical path.  Parity mode always
  // uses the 128-wide tile (shared-memory budget of the split planes).
  const bool wide = (N > 128) && !split && M > 16384;
  const uint32_t bn = wide ? 256 : 128;
  CUtensorMap a, alo, b, blo;
  const bf16* Xb = reinterpret_cast<const bf16*>(X);
  const bf16* Wb = reinterpret_cast<const bf16*>(W);
  if (make_map(&a, Xb, K, M, lda, 64, 16)) return 1;
  if (make_map(&b, Wb, K, N, ldb, 64, bn)) return 1;
  alo = a;
  blo = b;
  if (split) {
    if (make_map(&alo, Xb + x_lo_off, K, M, lda, 64, 16)) return 1;
    if (make_map(&blo, Wb + w_lo_off, K, N, ldb, 64, bn)) return 1;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ep.mode = pick_mode(ep, split, N);
  if (split) return launch_linear_split(a, alo, b, blo, M, N, K, ep, st);
  return wide ? launch_linear_fast<256>(a, b, M, N, K, ep, st) : launch_linear_fast<128>(a, b, M, N, K, ep, st);
}

// ---------------------------------------------------------------------------------------------------------------
// GEMM + LayerNorm in one kernel (fast mode, d_model = 256 rows owned by one CTA tile, path-level row counts)
// ---------------------------------------------------------------------------------------------------------------
extern "C" int dsvg_linear_ln_fusable(int M, int N, int n_planes) {
  return (n_planes == 1 && N == 256 && M > 16384) ? 1 : 0;
}

extern "C" int dsvg_linear_ln_fwd(const dsvg_bf16* X, size_t x_lo_off, int lda, const dsvg_bf16* W, size_t w_lo_off, int ldb,
                                  int M, int N, int K, const dsvg_epilogue* e, const float* gamma, const float* beta,
                                  dsvg_bf16* y, float* mean, float* rstd, void* stream) {
  DSVG_CHECK(X && W && e && gamma && beta && y && mean && rstd, "dsvg_linear_ln_fwd: null pointer");
  DSVG_CHECK(M > 0 && K > 0, "dsvg_linear_ln_fwd: bad shape");
  DSVG_CHECK(lda % 8 == 0 && ldb % 8 == 0, "dsvg_linear_ln_fwd: lda/ldb must be multiples of 8 elements");
  DSVG_CHECK(x_lo_off == 0 && w_lo_off == 0 && dsvg_linear_ln_fusable(M, N, 1),
             "dsvg_linear_ln_fwd: shape / mode not fusable (ask dsvg_linear_ln_fusable first)");
  Epi ep{};
  if (fill_epi(ep, e, M, N)) return 1;
  DSVG_CHECK(ep.out_f32 && !ep.out_act && !ep.mask && !ep.relu && ep.scale_cols == 0 && !ep.acc_scale_dev && ep.vec == 1,
             "dsvg_linear_ln_fwd: the epilogue must be the residual-stream form (bias, dropout, row vector, residual -> fp32)");
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  DSVG_CHECK(al16(gamma) && al16(beta) && al16(y), "dsvg_linear_ln_fwd: gamma / beta / y must be 16-byte aligned");
  ep.ln_gamma = gamma; ep.ln_beta = beta; ep.ln_out = reinterpret_cast<bf16*>(y); ep.ln_mean = mean; ep.ln_rstd = rstd;
  ep.mode = 8;
  CUtensorMap a, b;
  if (make_map(&a, reinterpret_cast<const bf16*>(X), K, M, lda, 64, 16)) return 1;
  if (make_map(&b, reinterpret_cast<const bf16*>(W), K, N, ldb, 64, 256)) return 1;
  return launch_linear_mode<256, 1, 8>(a, a, b, b, M, N, K, ep, static_cast<cudaStream_t>(stream));
}

extern "C" int dsvg_outer_group(int n, const dsvg_outer_problem* pr, int M, void* stream) {
  DSVG_CHECK(n >= 1 && n <= kMaxGroup && pr != nullptr && M > 0, "dsvg_outer_group: 1..%d problems", kMaxGroup);
  OuterGroup g{};
  g.n = n;
  g.M = M;
  for (int i = 0; i < n; ++i) {
    const dsvg_outer_problem& q = pr[i];
    DSVG_CHECK(q.A && q.B && q.C && q.P > 0 && q.Q > 0, "dsvg_outer_group: bad problem %d", i);
    DSVG_CHECK(q.lda % 8 == 0 && q.ldb % 8 == 0, "dsvg_outer_group: lda/ldb must be multiples of 8");
    if (make_map(&g.a[i], reinterpret_cast<const bf16*>(q.A), q.P, M, q.lda, 64, 64)) return 1;
    if (make_map(&g.b[i], reinterpret_cast<const bf16*>(q.B), q.Q, M, q.ldb, 64, 64)) return 1;
    outer_problem(g, i, q.alpha_dev, q.alpha, q.C, q.ldc, q.colsum_out, q.P, q.Q, 256);
  }
  return launch_outer<256, 1>(g, static_cast<cudaStream_t>(stream));
}

extern "C" int dsvg_outer(const dsvg_bf16* A, size_t a_lo_off, int lda, const dsvg_bf16* B, size_t b_lo_off, int ldb,
                          int M, int P, int Q, float alpha, const float* alpha_dev, float* C, int ldc, float* colsum_out,
                          void* stream) {
  DSVG_CHECK(A && B && C, "dsvg_outer: null pointer");
  DSVG_CHECK(M > 0 && P > 0 && Q > 0, "dsvg_outer: bad shape");
  DSVG_CHECK(lda % 8 == 0 && ldb % 8 == 0, "dsvg_outer: lda/ldb must be multiples of 8");
  DSVG_CHECK((a_lo_off == 0) == (b_lo_off == 0), "dsvg_outer: both operands must have the same number of planes");
  const bool wide = (Q > 128);
  OuterGroup g{};
  g.n = 1;
  g.M = M;
  const bf16* Ab = reinterpret_cast<const bf16*>(A);
  const bf16* Bb = reinterpret_cast<const bf16*>(B);
  // dim0 = feature columns (contiguous), dim1 = M rows; the tensor extents clip (zero-fill) ragged edges
  if (make_map(&g.a[0], Ab, P, M, lda, 64, 64)) return 1;
  if (make_map(&g.b[0], Bb, Q, M, ldb, 64, 64)) return 1;
  const bool split = a_lo_off != 0;
  if (split) {
    if (make_map(&g.alo, Ab + a_lo_off, P, M, lda, 64, 64)) return 1;
    if (make_map(&g.blo, Bb + b_lo_off, Q, M, ldb, 64, 64)) return 1;
  }
  outer_problem(g, 0, alpha_dev, alpha, C, ldc, colsum_out, P, Q, wide ? 256 : 128);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (wide) return split ? launch_outer<256, 2>(g, st) : launch_outer<256, 1>(g, st);
  return split ? launch_outer<128, 2>(g, st) : launch_outer<128, 1>(g, st);
}
