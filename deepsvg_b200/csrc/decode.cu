// Incremental autoregressive decoding: one new row per sequence per step, over per-layer key/value caches.
//
//   reference: SVGTransformer._greedy_sample / greedy_sample, model/model.py:428-448 -- every step re-runs the causal decoder
//              on the whole prefix and keeps the last position.  The causal mask (model/utils.py:69-72) makes position t's
//              output depend on tokens <= t only, so keeping each layer's keys and values and pushing only row t through
//              the stack computes the same function with N rows per step instead of N (t + 1).
//
// Every kernel here reads the step index t from device memory (`step[0]`), so one captured CUDA graph of a decode step
// replays unchanged for every t; decode_sample_kernel advances it.  `step[1]` is a block ticket used for that.
//   decode_embed_kernel   SVGEmbedding (model.py:46-57, use_group=True) of the token at position t, plus the per-sequence
//                         state seq_prep derives from a whole prefix, carried over from step t - 1: group index (number
//                         of "m" so far, model/utils.py:35-42) and key validity (no EOS at or before t, model/utils.py:7-17)
//   decode_attn_kernel    appends row t's K and V to the layer's cache, then attends row t's query over cached keys 0..t
//   decode_sample_kernel  argmax (temperature < 1e-3) or Gumbel-max sampling of the head logits, CMD_ARGS_MASK
//                         (model.py:450-459), tokens out, t += 1
#include "../../include/dsvg_b200.h"
#include "common.cuh"

namespace dsvg {
extern unsigned long long g_launches;

namespace {
constexpr int kCmdM = 0, kCmdEos = 4, kCmdSos = 5;
constexpr int kMaxSteps = 256;     // cached positions per sequence (the attention tile limits max_total_len to 153)
constexpr int kMaxClasses = 1024;  // classes per slot in the sampler's noise counter
// CMD_ARGS_MASK (difflib/tensor.py:15-21) as one bit per argument slot
__constant__ uint16_t c_args_used[7] = {0x600, 0x600, 0x7E0, 0x61F, 0, 0, 0};
}  // namespace

// ---------------------------------------------------------------------------------------------------------
// embedding of the token at position t: one warp per sequence, lane owns channels {128 i + 4 lane .. +3}.
// The sum is formed in embed_fwd_kernel's order, so row t equals row t of dsvg_embed_fwd on the whole prefix bitwise.
// ---------------------------------------------------------------------------------------------------------
struct DecodeEmbedArgs {
  const int* step;
  const int* cmd_in;     // [N] token at position t (t > 0; position 0 is SOS)
  const int* args_in;    // [N, n_args]
  int* grp;              // [N] number of "m" among positions 0..t (read at t - 1, written at t)
  uint8_t* key_valid;    // [N, Tmax]
  const float* cmd_tab;  // [7, d]
  const float* D;        // [n_args*V, d] difference table (dsvg_embed_fold)
  const float* base;     // [d]
  const float* pos_tab;  // [>= Tmax, d]
  const float* grp_tab;  // [>= Tmax + 1, d]
  float* x;              // [N, d]
  int N, Tmax, V, n_args;
};

template <int NV>
__global__ void __launch_bounds__(256) decode_embed_kernel(DecodeEmbedArgs a) {
  constexpr int d = NV * 128;
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  pdl_wait();
  if (n >= a.N) return;
  const int t = a.step[0];
  float mine;
  int cmd;
  if (t == 0) {  // model.py:428: SOS with every argument PAD
    mine = -1.f;
    cmd = kCmdSos;
  } else {
    mine = lane < a.n_args ? float(a.args_in[size_t(n) * a.n_args + lane]) : 0.f;
    cmd = a.cmd_in[n];
  }
  const int g = (t == 0 ? 0 : a.grp[n]) + (cmd == kCmdM ? 1 : 0);
  const bool valid = (t == 0 || a.key_valid[size_t(n) * a.Tmax + t - 1] != 0) && cmd != kCmdEos;
  float4 acc[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 128 * i + 4 * lane;
    float4 b = *reinterpret_cast<const float4*>(a.base + c);
    float4 e = *reinterpret_cast<const float4*>(a.cmd_tab + size_t(cmd) * d + c);
    float4 p = *reinterpret_cast<const float4*>(a.pos_tab + size_t(t) * d + c);
    acc[i] = make_float4(b.x + e.x + p.x, b.y + e.y + p.y, b.z + e.z + p.z, b.w + e.w + p.w);
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float4 e = *reinterpret_cast<const float4*>(a.grp_tab + size_t(g) * d + 128 * i + 4 * lane);
    acc[i].x += e.x; acc[i].y += e.y; acc[i].z += e.z; acc[i].w += e.w;
  }
  for (int k = 0; k < a.n_args; ++k) {
    const int v = int(__shfl_sync(0xffffffffu, mine, k)) + 1;  // shift due to the -1 PAD value (model.py:50)
    if (v <= 0) continue;                                      // PAD: its row is part of base
    const float* row = a.D + (size_t(k) * a.V + v) * d;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float4 e = __ldg(reinterpret_cast<const float4*>(row + 128 * i + 4 * lane));
      acc[i].x += e.x; acc[i].y += e.y; acc[i].z += e.z; acc[i].w += e.w;
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i)
    *reinterpret_cast<float4*>(a.x + size_t(n) * d + 128 * i + 4 * lane) = acc[i];
  if (lane == 0) {
    a.grp[n] = g;
    a.key_valid[size_t(n) * a.Tmax + t] = valid ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------------------------------
// attention of one new query row over the cache.  One warp per (sequence, head) pair.
//
// A key row of HD bf16 is HD / 8 16-byte chunks; HD / 8 lanes share one key (lane `sub` holds channels 8 sub .. 8 sub + 7)
// and the warp covers 32 / (HD / 8) keys per iteration.  Scores are reduced inside each lane group and kept in shared
// memory; softmax and P.V run in fp32, P.V partial sums are reduced across the key groups at the end.  The cache layout
// [N, H, Tmax, HD] (one plane after the other) keeps one pair's keys contiguous, so a warp streams 512 contiguous bytes
// per iteration.  Keys after a sequence's first EOS are never read.
//
// One query row per pair gives a 1 x t x HD product: there is no tile to feed the tensor cores, and every key byte is used
// once, so the kernel is bound by HBM (or L2) bandwidth over the cached K and V, not by arithmetic.
// ---------------------------------------------------------------------------------------------------------
struct DecodeAttnArgs {
  const int* step;
  const bf16* qkv;  // [N, 3d]: q (pre-scaled by the QKV epilogue) | k | v
  size_t qkv_lo;
  bf16* kc;         // [planes][N, H, Tmax, HD]
  bf16* vc;
  size_t cache_lo;
  const uint8_t* key_valid;  // [N, Tmax]
  bf16* out;                 // [N, d]
  size_t out_lo;
  int N, H, Tmax;
};

template <int PL>
__device__ __forceinline__ void load_chunk(const bf16* p, size_t lo, size_t i, float (&v)[8]) {
  const uint4 h = *reinterpret_cast<const uint4*>(p + i);
  const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&h);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float2 f = __bfloat1622float2(hp[c]);
    v[2 * c] = f.x;
    v[2 * c + 1] = f.y;
  }
  if (PL == 2) {
    const uint4 l = *reinterpret_cast<const uint4*>(p + i + lo);
    const __nv_bfloat162* lp = reinterpret_cast<const __nv_bfloat162*>(&l);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float2 f = __bfloat1622float2(lp[c]);
      v[2 * c] += f.x;
      v[2 * c + 1] += f.y;
    }
  }
}

template <int HD, int PL>
__global__ void __launch_bounds__(128, 8) decode_attn_kernel(DecodeAttnArgs a) {
  constexpr int LPK = HD / 8;    // lanes per key row
  constexpr int KPI = 32 / LPK;  // keys per warp iteration
  __shared__ float s_p[4][kMaxSteps];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane % LPK, kg = lane / LPK;
  const long long pair = (long long)blockIdx.x * 4 + wib;
  pdl_wait();
  if (pair >= (long long)a.N * a.H) return;
  const int n = int(pair / a.H), h = int(pair % a.H);
  const int d = a.H * HD;
  const int t = a.step[0];
  const size_t qrow = size_t(n) * 3 * d + size_t(h) * HD + 8 * sub;
  const size_t cbase = size_t(pair) * a.Tmax * HD + 8 * sub;
  // ---- 1. append row t's K and V (bitwise copies of the QKV output, every plane) ----
  if (kg == 0) {
#pragma unroll
    for (int p = 0; p < PL; ++p) {
      const size_t qo = p * a.qkv_lo, co = p * a.cache_lo;
      *reinterpret_cast<uint4*>(a.kc + co + cbase + size_t(t) * HD) = *reinterpret_cast<const uint4*>(a.qkv + qo + qrow + d);
      *reinterpret_cast<uint4*>(a.vc + co + cbase + size_t(t) * HD) =
          *reinterpret_cast<const uint4*>(a.qkv + qo + qrow + 2 * d);
    }
  }
  float q[8];
  load_chunk<PL>(a.qkv, a.qkv_lo, qrow, q);
  __syncwarp();
  // ---- 2. scores over keys 0..t ----
  float* sp = s_p[wib];
  const uint8_t* kv = a.key_valid + size_t(n) * a.Tmax;
  for (int j0 = 0; j0 <= t; j0 += KPI) {
    const int j = j0 + kg;
    const bool use = j <= t && kv[j] != 0;
    float s = 0.f;
    if (use) {
      float k[8];
      load_chunk<PL>(a.kc, a.cache_lo, cbase + size_t(j) * HD, k);
#pragma unroll
      for (int c = 0; c < 8; ++c) s = fmaf(q[c], k[c], s);
    }
#pragma unroll
    for (int o = 1; o < LPK; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (j <= t && sub == 0) sp[j] = use ? s : -INFINITY;
  }
  __syncwarp();
  float m = -INFINITY;
  for (int j = lane; j <= t; j += 32) m = fmaxf(m, sp[j]);
  m = warp_max(m);
  float sum = 0.f;
  for (int j = lane; j <= t; j += 32) {
    const float e = expf(sp[j] - m);  // key 0 (SOS) is always valid: m is finite
    sp[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  // ---- 3. P.V ----
  float o[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) o[c] = 0.f;
  for (int j0 = 0; j0 <= t; j0 += KPI) {
    const int j = j0 + kg;
    if (j <= t && kv[j] != 0) {
      const float p = sp[j];
      float v[8];
      load_chunk<PL>(a.vc, a.cache_lo, cbase + size_t(j) * HD, v);
#pragma unroll
      for (int c = 0; c < 8; ++c) o[c] = fmaf(p, v[c], o[c]);
    }
  }
#pragma unroll
  for (int off = LPK; off < 32; off <<= 1)
#pragma unroll
    for (int c = 0; c < 8; ++c) o[c] += __shfl_xor_sync(0xffffffffu, o[c], off);
  if (kg == 0) {
    const float inv = 1.f / sum;
    const size_t oi = size_t(n) * d + size_t(h) * HD + 8 * sub;
#pragma unroll
    for (int c = 0; c < 8; c += 2) act_store2(a.out, a.out_lo, oi + c, o[c] * inv, o[c + 1] * inv);
  }
}

// ---------------------------------------------------------------------------------------------------------
// token choice: one warp per sequence.  Slot 0 is the command (n_cmd classes), slots 1..n_args the argument slots.
// temperature < 1e-3: argmax, ties to the lowest index (torch.argmax).  Otherwise Gumbel-max: argmax_c(l_c / T + G_c),
// G = -log(-log(u)), u from 24 bits of a counter hash of (seed, t, sequence, slot, class) -- a draw from
// softmax(l / T), i.e. Categorical(logits = l / T).sample() of model.py:415-418.
// ---------------------------------------------------------------------------------------------------------
struct DecodeSampleArgs {
  int* step;                    // [2]: t, block ticket
  const float* cmd_logits;      // [N, ld_cmd]
  int ld_cmd;
  const float* args_logits;     // [N, ld_args], slot k at columns k*n_classes ..
  int ld_args;
  const float* temperature;     // device scalar
  const unsigned long long* seed;
  int* cmd_in;                  // [N]       next step's input
  int* args_in;                 // [N, n_args]
  long long* out_cmd;           // [N, Tmax]
  long long* out_args;          // [N, Tmax, n_args]
  int N, Tmax, n_cmd, n_args, n_classes;
};

__device__ __forceinline__ float gumbel_of(uint32_t key, uint32_t seq, uint32_t slot_class) {
  const uint32_t h = host_mix32(host_mix32(key ^ (seq * 0x9E3779B1u)) + slot_class * 0x85EBCA77u);
  // u = (k + 0.5) / 2^24 with 24 random bits k, strictly inside (0, 1).  -log(u) is formed from whichever of u and 1 - u
  // is exact in fp32: (k + 0.5) rounds to 2^24 (u = 1, an infinite draw) for k = 2^24 - 1.
  const uint32_t k = h >> 8;
  const float e = k < (1u << 23) ? -logf((float(k) + 0.5f) * (1.f / 16777216.f))
                                 : -log1pf(-(float((1u << 24) - 1u - k) + 0.5f) * (1.f / 16777216.f));
  return -logf(e);
}

__device__ __forceinline__ int warp_argmax(const float* row, int n, bool greedy, float inv_t, uint32_t key, uint32_t seq,
                                           uint32_t slot, int lane) {
  float best = -INFINITY;
  int bi = n;  // n = "none yet"
  for (int c = lane; c < n; c += 32) {  // ascending: a later equal value never replaces an earlier one
    float v = __ldg(row + c);
    if (!greedy) v = v * inv_t + gumbel_of(key, seq, slot * kMaxClasses + c);
    if (bi == n || v > best) {
      best = v;
      bi = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi < n && (bi == n || ov > best || (ov == best && oi < bi))) {
      best = ov;
      bi = oi;
    }
  }
  return bi;
}

__global__ void __launch_bounds__(256) decode_sample_kernel(DecodeSampleArgs a) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  pdl_wait();
  const int t = a.step[0];
  if (n < a.N) {
    const float T = *a.temperature;
    const bool greedy = T < 1e-3f;
    const float inv_t = greedy ? 1.f : 1.f / T;
    const uint32_t key = greedy ? 0u : drop_key_of(*a.seed, uint32_t(t));
    const int cmd = warp_argmax(a.cmd_logits + size_t(n) * a.ld_cmd, a.n_cmd, greedy, inv_t, key, n, 0, lane);
    const unsigned used = c_args_used[cmd];
    int mine = -1;
    for (int k = 0; k < a.n_args; ++k) {
      const int c = warp_argmax(a.args_logits + size_t(n) * a.ld_args + size_t(k) * a.n_classes, a.n_classes, greedy,
                                inv_t, key, n, k + 1, lane);
      if (lane == k) mine = ((used >> k) & 1u) ? c - 1 : -1;  // class 0 is the PAD value -1
    }
    if (lane == 0) {
      a.out_cmd[size_t(n) * a.Tmax + t] = cmd;
      a.cmd_in[n] = cmd;
    }
    if (lane < a.n_args) {
      a.out_args[(size_t(n) * a.Tmax + t) * a.n_args + lane] = mine;
      a.args_in[size_t(n) * a.n_args + lane] = mine;
    }
  }
  // t += 1 once every block has read t: the last block to take a ticket advances it and resets the ticket
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(reinterpret_cast<unsigned*>(a.step + 1), 1u);
    if (prev == gridDim.x - 1) {
      a.step[1] = 0;
      a.step[0] = t + 1;
      __threadfence();
    }
  }
}

template <int HD, int PL>
static cudaError_t launch_decode_attn(const DecodeAttnArgs& a, cudaStream_t st) {
  const long long pairs = (long long)a.N * a.H;
  return launch_k(decode_attn_kernel<HD, PL>, dim3(unsigned((pairs + 3) / 4)), dim3(128), 0, st, a);
}

}  // namespace dsvg
using namespace dsvg;

extern "C" int dsvg_decode_embed(const int* step, const int* cmd_in, const int* args_in, int* grp, uint8_t* key_valid,
                                 const float* cmd_tab, const float* table, const float* base, const float* pos_tab,
                                 const float* grp_tab, float* x, int N, int Tmax, int V, int n_args, int d,
                                 void* stream) {
  DSVG_CHECK(step && cmd_in && args_in && grp && key_valid && cmd_tab && table && base && pos_tab && grp_tab && x,
             "dsvg_decode_embed: null pointer");
  DSVG_CHECK(N > 0 && Tmax > 0 && V > 0, "dsvg_decode_embed: bad sizes");
  DSVG_CHECK(n_args >= 1 && n_args <= 30, "dsvg_decode_embed: n_args must be in [1, 30]");
  DSVG_CHECK(d == 128 || d == 256 || d == 512, "dsvg_decode_embed: d_model %d unsupported", d);
  DecodeEmbedArgs a{step, cmd_in, args_in, grp, key_valid, cmd_tab, table, base, pos_tab, grp_tab, x, N, Tmax, V, n_args};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(ceil_div(N, 8)), block(256);
  switch (d) {
    case 128: DSVG_CUDA(launch_k(decode_embed_kernel<1>, grid, block, 0, st, a)); break;
    case 256: DSVG_CUDA(launch_k(decode_embed_kernel<2>, grid, block, 0, st, a)); break;
    default: DSVG_CUDA(launch_k(decode_embed_kernel<4>, grid, block, 0, st, a)); break;
  }
  ++g_launches;
  return 0;
}

extern "C" int dsvg_decode_attn(const int* step, const dsvg_bf16* qkv, size_t qkv_lo_off, dsvg_bf16* k_cache,
                                dsvg_bf16* v_cache, size_t cache_lo_off, const uint8_t* key_valid, dsvg_bf16* out,
                                size_t out_lo_off, int N, int H, int head_dim, int Tmax, void* stream) {
  DSVG_CHECK(step && qkv && k_cache && v_cache && key_valid && out, "dsvg_decode_attn: null pointer");
  DSVG_CHECK(N > 0 && H > 0 && Tmax > 0, "dsvg_decode_attn: bad sizes");
  DSVG_CHECK(Tmax <= kMaxSteps, "dsvg_decode_attn: at most %d cached positions, got %d", kMaxSteps, Tmax);
  const bool two = qkv_lo_off != 0;
  DSVG_CHECK(two == (cache_lo_off != 0) && two == (out_lo_off != 0),
             "dsvg_decode_attn: qkv, cache and output must all have one plane or all two");
  DecodeAttnArgs a{};
  a.step = step;
  a.qkv = reinterpret_cast<const bf16*>(qkv); a.qkv_lo = qkv_lo_off;
  a.kc = reinterpret_cast<bf16*>(k_cache); a.vc = reinterpret_cast<bf16*>(v_cache); a.cache_lo = cache_lo_off;
  a.key_valid = key_valid;
  a.out = reinterpret_cast<bf16*>(out); a.out_lo = out_lo_off;
  a.N = N; a.H = H; a.Tmax = Tmax;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  switch (head_dim * 2 + (two ? 1 : 0)) {
    case 32: e = launch_decode_attn<16, 1>(a, st); break;
    case 33: e = launch_decode_attn<16, 2>(a, st); break;
    case 64: e = launch_decode_attn<32, 1>(a, st); break;
    case 65: e = launch_decode_attn<32, 2>(a, st); break;
    case 128: e = launch_decode_attn<64, 1>(a, st); break;
    case 129: e = launch_decode_attn<64, 2>(a, st); break;
    default: DSVG_CHECK(false, "dsvg_decode_attn: head_dim %d unsupported (16, 32, 64)", head_dim);
  }
  DSVG_CUDA(e);
  ++g_launches;
  return 0;
}

extern "C" int dsvg_decode_sample(int* step, const float* cmd_logits, int ld_cmd, const float* args_logits, int ld_args,
                                  const float* temperature, const unsigned long long* seed, int* cmd_in, int* args_in,
                                  long long* out_cmd, long long* out_args, int N, int Tmax, int n_cmd, int n_args,
                                  int n_classes, void* stream) {
  DSVG_CHECK(step && cmd_logits && args_logits && temperature && seed && cmd_in && args_in && out_cmd && out_args,
             "dsvg_decode_sample: null pointer");
  DSVG_CHECK(N > 0 && Tmax > 0 && n_cmd == 7, "dsvg_decode_sample: bad sizes (n_cmd must be 7)");
  DSVG_CHECK(n_args >= 1 && n_args <= 16 && n_classes >= 1 && n_classes <= kMaxClasses,
             "dsvg_decode_sample: n_args must be in [1, 16] and n_classes in [1, %d]", kMaxClasses);
  DSVG_CHECK(ld_cmd >= n_cmd && ld_args >= n_args * n_classes, "dsvg_decode_sample: bad leading dimensions");
  DecodeSampleArgs a{step, cmd_logits, ld_cmd, args_logits, ld_args, temperature, seed, cmd_in, args_in, out_cmd, out_args,
                     N, Tmax, n_cmd, n_args, n_classes};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DSVG_CUDA(launch_k(decode_sample_kernel, dim3(ceil_div(N, 8)), dim3(256), 0, st, a));
  ++g_launches;
  return 0;
}
