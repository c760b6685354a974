// Short-sequence multi-head self-attention, forward and backward, fp32 SIMT.
//
//   reference: multi_head_attention_forward, model/layers/functional.py:168-248 -- per (sequence, head):
//              softmax(q k^T, keys masked by key_padding_mask -> -inf) -> dropout(P) -> P v
//   q arrives pre-scaled by head_dim^-0.5 (folded into the QKV GEMM epilogue, functional.py:168).
//
// DeepSVG's sequences are tiny (L = 8, 31, 32, <= 66; head_dim 32/64): one warp owns one (sequence, head) pair, lane i
// owns query row i, K/V (and Q/dO in the backward) of the pair are staged in shared memory as fp32 and read as
// warp-broadcast float4s; the L x L probability tile never leaves shared memory.  Attention is 2.4 % of the step's
// FLOPs (SURVEY.md 8d).  This file also holds the dispatcher of dsvg_attn_fwd / dsvg_attn_bwd: the tensor-core kernels of
// attention_mma.cu take every shape of the BASELINE configs in both precision modes (one plane: attn_mma / attn_gmma,
// two planes: attn_x3 / attn_gx3); the SIMT kernels below remain for head_dim 16 and L > 80.
#include "../../include/dsvg_b200.h"

#include "common.cuh"

namespace dsvg {
extern unsigned long long g_launches;

struct AttnArgs {
  const bf16* qkv;
  size_t qkv_lo;
  const uint8_t* valid;  // [nseq * L] 1 = key usable, or nullptr
  bf16* out;             // fwd: [nseq*L, d]
  size_t out_lo;
  const bf16* dout;      // bwd: [nseq*L, d]
  size_t dout_lo;
  bf16* dqkv;            // bwd: [nseq*L, 3d]
  size_t dqkv_lo;
  int nseq, L, H;
  float scale;           // bwd: dq is multiplied by this (the folded q scaling)
  Dropout drop;
  int causal;            // 1: query i sees keys j <= i only (square_subsequent_mask, model/utils.py:69-72)
};

template <int HD>
__device__ __forceinline__ void load_row_regs(const bf16* p, size_t lo, size_t base, float (&r)[HD]) {
#pragma unroll
  for (int c = 0; c < HD; c += 2) {
    float2 t = act_load2(p, lo, base + c);
    r[c] = t.x;
    r[c + 1] = t.y;
  }
}
template <int HD>
__device__ __forceinline__ void store_row_regs(bf16* p, size_t lo, size_t base, const float (&r)[HD], float mul) {
#pragma unroll
  for (int c = 0; c < HD; c += 2) act_store2(p, lo, base + c, r[c] * mul, r[c + 1] * mul);
}
template <int HD>
__device__ __forceinline__ float dot_smem(const float (&q)[HD], const float* row) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < HD; c += 4) {
    float4 k = *reinterpret_cast<const float4*>(row + c);
    s = fmaf(q[c], k.x, s);
    s = fmaf(q[c + 1], k.y, s);
    s = fmaf(q[c + 2], k.z, s);
    s = fmaf(q[c + 3], k.w, s);
  }
  return s;
}
template <int HD>
__device__ __forceinline__ void axpy_smem(float (&o)[HD], float a, const float* row) {
#pragma unroll
  for (int c = 0; c < HD; c += 4) {
    float4 v = *reinterpret_cast<const float4*>(row + c);
    o[c] = fmaf(a, v.x, o[c]);
    o[c + 1] = fmaf(a, v.y, o[c + 1]);
    o[c + 2] = fmaf(a, v.z, o[c + 2]);
    o[c + 3] = fmaf(a, v.w, o[c + 3]);
  }
}
// stage `rows` rows of HD channels (one head slice of a [.., ld] act tensor) into shared fp32
template <int HD>
__device__ __forceinline__ void stage_rows(float* dst, const bf16* p, size_t lo, size_t base, int ld, int rows,
                                           int lane) {
  for (int e = lane; e < rows * (HD / 2); e += 32) {
    int j = e / (HD / 2), c = 2 * (e % (HD / 2));
    float2 t = act_load2(p, lo, base + size_t(j) * ld + c);
    dst[j * HD + c] = t.x;
    dst[j * HD + c + 1] = t.y;
  }
}

template <int HD>
__global__ void __launch_bounds__(128) attn_fwd_kernel(AttnArgs a) {
  drop_resolve(a.drop);
  extern __shared__ __align__(16) float smem[];
  const int wpb = blockDim.x >> 5, wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = a.L, Lp = L | 1, d = a.H * HD, ld = 3 * d;
  float* Ks = smem + size_t(wib) * (2 * L * HD + 32 * Lp);
  float* Vs = Ks + L * HD;
  float* Ps = Vs + L * HD;
  const long long npairs = (long long)a.nseq * a.H;
  for (long long pair = (long long)blockIdx.x * wpb + wib; pair < npairs; pair += (long long)gridDim.x * wpb) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    stage_rows<HD>(Ks, a.qkv, a.qkv_lo, row0 * ld + d + h * HD, ld, L, lane);
    stage_rows<HD>(Vs, a.qkv, a.qkv_lo, row0 * ld + 2 * d + h * HD, ld, L, lane);
    __syncwarp();
    for (int i0 = 0; i0 < L; i0 += 32) {
      const int i = i0 + lane;
      if (i < L) {
        float q[HD];
        load_row_regs<HD>(a.qkv, a.qkv_lo, (row0 + i) * ld + h * HD, q);
        float* prow = Ps + lane * Lp;
        float m = -INFINITY;
        for (int j = 0; j < L; ++j) {
          float s = dot_smem<HD>(q, Ks + j * HD);
          if ((a.valid != nullptr && !a.valid[row0 + j]) || (a.causal && j > i)) s = -INFINITY;
          prow[j] = s;
          m = fmaxf(m, s);
        }
        float sum = 0.f;
        for (int j = 0; j < L; ++j) {
          float e = expf(prow[j] - m);
          prow[j] = e;
          sum += e;
        }
        const float inv = 1.f / sum;
        float o[HD];
#pragma unroll
        for (int c = 0; c < HD; ++c) o[c] = 0.f;
        const unsigned long long pbase = ((unsigned long long)pair * L + i) * L;
        for (int j = 0; j < L; ++j) {
          float p = prow[j] * inv;
          if (a.drop.p > 0.f) p *= dropout_mult(a.drop, pbase + j);
          axpy_smem<HD>(o, p, Vs + j * HD);
        }
        store_row_regs<HD>(a.out, a.out_lo, (row0 + i) * d + h * HD, o, 1.f);
      }
    }
    __syncwarp();
  }
}

template <int HD>
__global__ void __launch_bounds__(128) attn_bwd_kernel(AttnArgs a) {
  drop_resolve(a.drop);
  extern __shared__ __align__(16) float smem[];
  const int wpb = blockDim.x >> 5, wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = a.L, Lp = L | 1, d = a.H * HD, ld = 3 * d;
  float* Qs = smem + size_t(wib) * ((size_t(4) * L * HD + size_t(2) * L * Lp + 3) & ~size_t(3));
  float* Ks = Qs + L * HD;
  float* Vs = Ks + L * HD;
  float* Gs = Vs + L * HD;   // dO
  float* Ps = Gs + L * HD;   // dropout-scaled probabilities  [L][Lp]
  float* Ds = Ps + L * Lp;   // dS                             [L][Lp]
  const long long npairs = (long long)a.nseq * a.H;
  for (long long pair = (long long)blockIdx.x * wpb + wib; pair < npairs; pair += (long long)gridDim.x * wpb) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    stage_rows<HD>(Qs, a.qkv, a.qkv_lo, row0 * ld + h * HD, ld, L, lane);
    stage_rows<HD>(Ks, a.qkv, a.qkv_lo, row0 * ld + d + h * HD, ld, L, lane);
    stage_rows<HD>(Vs, a.qkv, a.qkv_lo, row0 * ld + 2 * d + h * HD, ld, L, lane);
    stage_rows<HD>(Gs, a.dout, a.dout_lo, row0 * d + h * HD, d, L, lane);
    __syncwarp();
    // ---- rows: lane i owns query i ----
    for (int i0 = 0; i0 < L; i0 += 32) {
      const int i = i0 + lane;
      if (i < L) {
        float q[HD], g[HD];
        load_row_regs<HD>(a.qkv, a.qkv_lo, (row0 + i) * ld + h * HD, q);
        load_row_regs<HD>(a.dout, a.dout_lo, (row0 + i) * d + h * HD, g);
        float* prow = Ps + i * Lp;
        float* drow = Ds + i * Lp;
        float m = -INFINITY;
        for (int j = 0; j < L; ++j) {
          float s = dot_smem<HD>(q, Ks + j * HD);
          if ((a.valid != nullptr && !a.valid[row0 + j]) || (a.causal && j > i)) s = -INFINITY;
          prow[j] = s;
          m = fmaxf(m, s);
        }
        float sum = 0.f;
        for (int j = 0; j < L; ++j) {
          float e = expf(prow[j] - m);
          prow[j] = e;
          sum += e;
        }
        const float inv = 1.f / sum;
        const unsigned long long pbase = ((unsigned long long)pair * L + i) * L;
        float delta = 0.f;
        for (int j = 0; j < L; ++j) {
          float p = prow[j] * inv;
          float mult = a.drop.p > 0.f ? dropout_mult(a.drop, pbase + j) : 1.f;
          float dp = dot_smem<HD>(g, Vs + j * HD) * mult;  // d loss / d p_ij
          delta = fmaf(dp, p, delta);
          drow[j] = dp;
          prow[j] = p;
        }
        float dq[HD];
#pragma unroll
        for (int c = 0; c < HD; ++c) dq[c] = 0.f;
        for (int j = 0; j < L; ++j) {
          float p = prow[j];
          float ds = p * (drow[j] - delta);
          float mult = a.drop.p > 0.f ? dropout_mult(a.drop, pbase + j) : 1.f;
          drow[j] = ds;
          prow[j] = p * mult;
          axpy_smem<HD>(dq, ds, Ks + j * HD);
        }
        store_row_regs<HD>(a.dqkv, a.dqkv_lo, (row0 + i) * ld + h * HD, dq, a.scale);
      }
    }
    __syncwarp();
    // ---- columns: lane j owns key/value j ----
    for (int j0 = 0; j0 < L; j0 += 32) {
      const int j = j0 + lane;
      if (j < L) {
        float dk[HD], dv[HD];
#pragma unroll
        for (int c = 0; c < HD; ++c) dk[c] = dv[c] = 0.f;
        for (int i = 0; i < L; ++i) {
          axpy_smem<HD>(dk, Ds[i * Lp + j], Qs + i * HD);
          axpy_smem<HD>(dv, Ps[i * Lp + j], Gs + i * HD);
        }
        store_row_regs<HD>(a.dqkv, a.dqkv_lo, (row0 + j) * ld + d + h * HD, dk, 1.f);
        store_row_regs<HD>(a.dqkv, a.dqkv_lo, (row0 + j) * ld + 2 * d + h * HD, dv, 1.f);
      }
    }
    __syncwarp();
  }
}

static int pick_wpb(size_t per_warp_bytes) {
  int wpb = 4;
  while (wpb > 1 && per_warp_bytes * wpb > 200 * 1024) wpb >>= 1;
  return wpb;
}

template <int HD>
static int launch_attn(bool bwd, const AttnArgs& a, cudaStream_t st) {
  const int L = a.L, Lp = L | 1;
  const size_t per_warp = bwd ? sizeof(float) * ((size_t(4) * L * HD + size_t(2) * L * Lp + 3) & ~size_t(3))
                              : sizeof(float) * (size_t(2) * L * HD + size_t(32) * Lp);
  const int wpb = pick_wpb(per_warp);
  const size_t smem = per_warp * wpb;
  DSVG_CHECK(smem <= 227 * 1024, "attention: sequence length %d too long for shared memory", L);
  auto kern = bwd ? attn_bwd_kernel<HD> : attn_fwd_kernel<HD>;
  DSVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  const long long npairs = (long long)a.nseq * a.H;
  long long blocks = (npairs + wpb - 1) / wpb;
  const long long cap = 132LL * 16;
  if (blocks > cap) blocks = cap;
  kern<<<int(blocks), wpb * 32, smem, st>>>(a);
  ++g_launches;
  DSVG_LAUNCH_CHECK();
  return 0;
}

}  // namespace dsvg
using namespace dsvg;

// tensor-core (mma.sync) fast path, attention_mma.cu
int dsvg_attn_mma_fwd(const bf16* qkv, const uint8_t* valid, bf16* out, int nseq, int L, int H, Dropout drop, int causal,
                      cudaStream_t st);
int dsvg_attn_mma_bwd(const bf16* qkv, const uint8_t* valid, const bf16* dout, bf16* dqkv, int nseq, int L, int H,
                      float q_scale, Dropout drop, int causal, cudaStream_t st);
int dsvg_attn_gmma(bool bwd, const bf16* qkv, const uint8_t* valid, bf16* out, const bf16* dout, bf16* dqkv, int nseq, int L,
                   int H, int head_dim, float q_scale, Dropout drop, int causal, cudaStream_t st);
int dsvg_attn_x3(bool bwd, const bf16* qkv, size_t qkv_lo, const uint8_t* valid, bf16* out, size_t out_lo, const bf16* dout,
                 size_t dout_lo, bf16* dqkv, size_t dqkv_lo, int nseq, int L, int H, float q_scale, Dropout drop, int causal,
                 cudaStream_t st);
int dsvg_attn_gx3(bool bwd, const bf16* qkv, size_t qkv_lo, const uint8_t* valid, bf16* out, size_t out_lo, const bf16* dout,
                  size_t dout_lo, bf16* dqkv, size_t dqkv_lo, int nseq, int L, int H, int head_dim, float q_scale, Dropout drop,
                  int causal, cudaStream_t st);
static bool use_mma(bool single_plane, int L, int head_dim) {
  return single_plane && head_dim == 32 && L <= 32;
}
// parity mode (two planes everywhere) on the same 32 x 32 tiles: three bf16 products per contraction step
static bool use_x3(bool two_planes, int L, int head_dim) {
  return two_planes && head_dim == 32 && L <= 32;
}
static bool use_gx3(bool two_planes, int L, int head_dim) {
  return two_planes && (head_dim == 32 || head_dim == 64) && L <= 80;
}
// general tensor-core kernel (attention_mma.cu): every other fast-mode shape of the BASELINE configs
static bool use_gmma(bool single_plane, int L, int head_dim) {
  return single_plane && (head_dim == 32 || head_dim == 64) && L <= 80;
}

extern "C" int dsvg_attn_fwd(const dsvg_bf16* qkv, size_t qkv_lo_off, const uint8_t* key_valid, dsvg_bf16* out,
                             size_t out_lo_off, int nseq, int L, int H, int head_dim, int causal, float drop_p,
                             uint32_t drop_site, uint64_t seed, void* stream) {
  DSVG_CHECK(qkv && out && nseq > 0 && L > 0 && H > 0, "dsvg_attn_fwd: bad arguments");
  AttnArgs a{};
  a.qkv = reinterpret_cast<const bf16*>(qkv); a.qkv_lo = qkv_lo_off; a.valid = key_valid;
  a.out = reinterpret_cast<bf16*>(out); a.out_lo = out_lo_off;
  a.nseq = nseq; a.L = L; a.H = H; a.scale = 1.f; a.causal = causal ? 1 : 0;
  a.drop = make_dropout(drop_p, drop_site, seed);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (use_mma(qkv_lo_off == 0 && out_lo_off == 0, L, head_dim))
    return dsvg_attn_mma_fwd(a.qkv, key_valid, a.out, nseq, L, H, a.drop, a.causal, st);
  if (use_x3(qkv_lo_off != 0 && out_lo_off != 0, L, head_dim))
    return dsvg_attn_x3(false, a.qkv, qkv_lo_off, key_valid, a.out, out_lo_off, nullptr, 0, nullptr, 0, nseq, L, H, 1.f,
                        a.drop, a.causal, st);
  if (use_gx3(qkv_lo_off != 0 && out_lo_off != 0, L, head_dim))
    return dsvg_attn_gx3(false, a.qkv, qkv_lo_off, key_valid, a.out, out_lo_off, nullptr, 0, nullptr, 0, nseq, L, H, head_dim,
                         1.f, a.drop, a.causal, st);
  if (use_gmma(qkv_lo_off == 0 && out_lo_off == 0, L, head_dim))
    return dsvg_attn_gmma(false, a.qkv, key_valid, a.out, nullptr, nullptr, nseq, L, H, head_dim, 1.f, a.drop, a.causal, st);
  if (head_dim == 32) return launch_attn<32>(false, a, st);
  if (head_dim == 64) return launch_attn<64>(false, a, st);
  if (head_dim == 16) return launch_attn<16>(false, a, st);
  DSVG_CHECK(false, "dsvg_attn_fwd: head_dim %d unsupported (16, 32, 64)", head_dim);
}

extern "C" int dsvg_attn_bwd(const dsvg_bf16* qkv, size_t qkv_lo_off, const uint8_t* key_valid, const dsvg_bf16* dout,
                             size_t dout_lo_off, dsvg_bf16* dqkv, size_t dqkv_lo_off, int nseq, int L, int H,
                             int head_dim, int causal, float q_scale, float drop_p, uint32_t drop_site, uint64_t seed,
                             void* stream) {
  DSVG_CHECK(qkv && dout && dqkv && nseq > 0 && L > 0 && H > 0, "dsvg_attn_bwd: bad arguments");
  AttnArgs a{};
  a.qkv = reinterpret_cast<const bf16*>(qkv); a.qkv_lo = qkv_lo_off; a.valid = key_valid;
  a.dout = reinterpret_cast<const bf16*>(dout); a.dout_lo = dout_lo_off;
  a.dqkv = reinterpret_cast<bf16*>(dqkv); a.dqkv_lo = dqkv_lo_off;
  a.nseq = nseq; a.L = L; a.H = H; a.scale = q_scale; a.causal = causal ? 1 : 0;
  a.drop = make_dropout(drop_p, drop_site, seed);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (use_mma(qkv_lo_off == 0 && dout_lo_off == 0 && dqkv_lo_off == 0, L, head_dim))
    return dsvg_attn_mma_bwd(a.qkv, key_valid, a.dout, a.dqkv, nseq, L, H, q_scale, a.drop, a.causal, st);
  if (use_x3(qkv_lo_off != 0 && dout_lo_off != 0 && dqkv_lo_off != 0, L, head_dim))
    return dsvg_attn_x3(true, a.qkv, qkv_lo_off, key_valid, nullptr, 0, a.dout, dout_lo_off, a.dqkv, dqkv_lo_off, nseq, L, H,
                        q_scale, a.drop, a.causal, st);
  if (use_gx3(qkv_lo_off != 0 && dout_lo_off != 0 && dqkv_lo_off != 0, L, head_dim))
    return dsvg_attn_gx3(true, a.qkv, qkv_lo_off, key_valid, nullptr, 0, a.dout, dout_lo_off, a.dqkv, dqkv_lo_off, nseq, L, H,
                         head_dim, q_scale, a.drop, a.causal, st);
  if (use_gmma(qkv_lo_off == 0 && dout_lo_off == 0 && dqkv_lo_off == 0, L, head_dim))
    return dsvg_attn_gmma(true, a.qkv, key_valid, nullptr, a.dout, a.dqkv, nseq, L, H, head_dim, q_scale, a.drop, a.causal, st);
  if (head_dim == 32) return launch_attn<32>(true, a, st);
  if (head_dim == 64) return launch_attn<64>(true, a, st);
  if (head_dim == 16) return launch_attn<16>(true, a, st);
  DSVG_CHECK(false, "dsvg_attn_bwd: head_dim %d unsupported (16, 32, 64)", head_dim);
}
