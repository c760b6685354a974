// Fast-mode attention for DeepSVG's tiny sequences on the warp-level tensor-core path (mma.sync m16n8k16, bf16 in,
// fp32 accumulate): one warp computes one (sequence, head) pair at a time, head_dim = 32, L <= 32 keys/queries padded
// to a 32 x 32 tile.  Whole sequences stream through shared memory (bulk copies into a ring of stages, see "sequence
// streaming" below) and are read with ldmatrix; scores, probabilities and all gradients of the pair stay in registers /
// shared memory, and the outputs leave through shared memory as whole-row bulk stores.
//
//   reference: functional.py:168-248 (attention.cu keeps the fp32 SIMT version for head_dim 16 / L > 80; the parity-mode
//   variants of these kernels -- two bf16 planes, three products -- follow further down in this file).  wgmma is not used here on purpose: a 32 x 32 x 32 problem fills a fraction of
//   the smallest warpgroup tile (m64; SURVEY.md section 7, hard part 2); attention is 2.4 % of the step's FLOPs.
//
// Dropout on the probabilities uses its own element numbering (8 consecutive draws per (row, lane-in-quad)),
// identical in forward and backward of THIS kernel.
#include "../../include/dsvg_b200.h"
#include "common.cuh"
#include "ptx.cuh"

namespace dsvg {
extern unsigned long long g_launches;

constexpr int kRow = 40;                   // smem row stride in bf16 (80 B: 16-byte aligned, conflict-free ldmatrix)
constexpr int kTile = 32 * kRow;           // one 32 x 32 tile

struct MmaAttnArgs {
  const bf16* qkv;      // [nseq*L, 3d]
  const uint8_t* valid; // [nseq*L] or null
  bf16* out;            // fwd  [nseq*L, d]
  const bf16* dout;     // bwd  [nseq*L, d]
  bf16* dqkv;           // bwd  [nseq*L, 3d]
  int nseq, L, H;
  float scale;
  Dropout drop;
  int causal;           // query i sees keys j <= i only
  int stages;           // attn_mma_fwd / bwd: shared-memory stages of the sequence ring (1 or 2)
};

__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }

// ---- fragment loaders (tile = 32 x 32 bf16, row stride kRow) -------------------------------------------
// A operand, rows [16*mt, +16), k columns [16*ks, +16): a0..a3 from one ldmatrix.x4
__device__ __forceinline__ void load_a(uint32_t (&a)[4], uint32_t tile, int mt, int ks, int lane, int st = kRow) {
  const int m = lane >> 3, r = lane & 7;
  ldsm_x4(a, tile + ((16 * mt + (m & 1) * 8 + r) * st + 16 * ks + (m >> 1) * 8) * 2);
}
// A operand taken TRANSPOSED from a row-major tile Z[k][m]: A[m][k] = Z[k][m]
__device__ __forceinline__ void load_a_t(uint32_t (&a)[4], uint32_t tile, int mt, int ks, int lane, int st = kRow) {
  const int m = lane >> 3, r = lane & 7;
  // matrices: (k0, m0) (k0, m0+8) (k0+8, m0) (k0+8, m0+8) -> a0 a1 a2 a3
  ldsm_x4_t(a, tile + ((16 * ks + (m >> 1) * 8 + r) * st + 16 * mt + (m & 1) * 8) * 2);
}
// B operand ("col") for two adjacent n-tiles from row-major X[n][k] (K for Q.K^T, V for dO.V^T):
// r0,r1 = b0,b1 of n-tile 2*np ; r2,r3 = b0,b1 of n-tile 2*np+1
__device__ __forceinline__ void load_b_nk(uint32_t (&b)[4], uint32_t tile, int np, int ks, int lane, int st = kRow) {
  const int m = lane >> 3, r = lane & 7;
  ldsm_x4(b, tile + ((16 * np + (m >> 1) * 8 + r) * st + 16 * ks + (m & 1) * 8) * 2);
}
// B operand for two adjacent n-tiles from row-major Y[k][n] (V for P.V, K for dS.K, Q / dO for the transposed products)
__device__ __forceinline__ void load_b_kn(uint32_t (&b)[4], uint32_t tile, int np, int ks, int lane, int st = kRow) {
  const int m = lane >> 3, r = lane & 7;
  ldsm_x4_t(b, tile + ((16 * ks + (m & 1) * 8 + r) * st + 16 * np + (m >> 1) * 8) * 2);
}

// stage a [L x 32] head slice (row stride ld elements) into a zero-padded 32 x 32 tile; 16-byte chunks
__device__ __forceinline__ void stage_tile(bf16* dst, const bf16* src, int ld, int L, int lane) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int chunk = lane + 32 * it, row = chunk >> 2, part = chunk & 3;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row < L) v = *reinterpret_cast<const uint4*>(src + size_t(row) * ld + part * 8);
    *reinterpret_cast<uint4*>(dst + row * kRow + part * 8) = v;
  }
}

// scores -> probabilities in the C-fragment layout.  s[mt][nt][e]: row 16*mt + g + 8*(e>>1), col 8*nt + 2*t + (e&1)
__device__ __forceinline__ void softmax_rows(float (&s)[2][4][4], uint32_t key_mask, int t, int g = 0, int causal = 0) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      float m = -INFINITY;
      // causal: row i = 16 mt + g + 8 hrow sees keys j <= i, i.e. the low i + 1 bits of the key mask
      const int i = 16 * mt + g + 8 * hrow;
      const uint32_t km = causal ? (key_mask & (0xFFFFFFFFu >> (31 - i))) : key_mask;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = 8 * nt + 2 * t + e;
          float& x = s[mt][nt][2 * hrow + e];
          if (!((km >> j) & 1u)) x = -INFINITY;
          m = fmaxf(m, x);
        }
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      float sum = 0.f;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& x = s[mt][nt][2 * hrow + e];
          x = __expf(x - m);
          sum += x;
        }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      const float inv = 1.f / sum;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) s[mt][nt][2 * hrow + e] *= inv;
    }
}

// dropout multipliers in the same layout: 8 consecutive 16-bit draws (4 hashes) per (pair, row, t)
__device__ __forceinline__ void dropout_tile(float (&mult)[2][4][4], const Dropout& d, unsigned long long pair, int g,
                                             int t) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int i = 16 * mt + g + 8 * hrow;
      // draws 8 * ((pair * 32 + i) * 4 + t) .. + 7  =  two whole quads (see common.cuh): word nt covers elements
      // (nt >> 1 selects the quad, nt & 1 its a / b finaliser)
      const unsigned long long quad = ((pair * 32 + i) * 4 + t) * 2;
      const uint32_t hk = drop_hikey(d, quad), q0 = uint32_t(quad);   // quad is even: q0 + 1 cannot carry
#pragma unroll
      for (int hq = 0; hq < 2; ++hq) {
        const uint32_t s1 = drop_stage1(q0 + hq, hk);
        const uint32_t a = drop_fin_a(s1), b = drop_fin_b(s1);
        mult[mt][2 * hq][2 * hrow] = drop_keep_lo(a, d.thr16) ? d.scale : 0.f;
        mult[mt][2 * hq][2 * hrow + 1] = drop_keep_hi(a, d.thr16) ? d.scale : 0.f;
        mult[mt][2 * hq + 1][2 * hrow] = drop_keep_lo(b, d.thr16) ? d.scale : 0.f;
        mult[mt][2 * hq + 1][2 * hrow + 1] = drop_keep_hi(b, d.thr16) ? d.scale : 0.f;
      }
    }
}

__device__ __forceinline__ uint32_t key_mask_of(const uint8_t* valid, size_t row0, int L, int lane) {
  bool ok = lane < L;
  if (ok && valid != nullptr) ok = valid[row0 + lane] != 0;
  return __ballot_sync(0xffffffffu, ok);
}

// S = Q K^T  (both tiles row-major [row][channel]; qs, kst: their row strides in elements)
__device__ __forceinline__ void qk_scores(float (&s)[2][4][4], uint32_t q_tile, uint32_t k_tile, int lane, int qs = kRow,
                                          int kst = kRow) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[mt][nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    uint32_t a[2][4];
    load_a(a[0], q_tile, 0, ks, lane, qs);
    load_a(a[1], q_tile, 1, ks, lane, qs);
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t b[4];
      load_b_nk(b, k_tile, np, ks, lane, kst);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma_bf16(s[mt][2 * np], a[mt], b[0], b[1]);
        mma_bf16(s[mt][2 * np + 1], a[mt], b[2], b[3]);
      }
    }
  }
}

// C-fragment of a 32 x 32 matrix (keys on the column axis) -> A-fragments for a product over those columns
__device__ __forceinline__ void c_to_a(uint32_t (&a)[4], const float (&c)[2][4][4], int mt, int ks) {
  a[0] = pack_bf16(c[mt][2 * ks][0], c[mt][2 * ks][1]);
  a[1] = pack_bf16(c[mt][2 * ks][2], c[mt][2 * ks][3]);
  a[2] = pack_bf16(c[mt][2 * ks + 1][0], c[mt][2 * ks + 1][1]);
  a[3] = pack_bf16(c[mt][2 * ks + 1][2], c[mt][2 * ks + 1][3]);
}
// out[32 x 32] = A(regs, from c_to_a) . Y   with Y row-major [k][n] in smem (row stride ys elements)
__device__ __forceinline__ void mul_regs_kn(float (&o)[2][4][4], const float (&p)[2][4][4], uint32_t y_tile, int lane,
                                            int ys = kRow) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    uint32_t a[2][4];
    c_to_a(a[0], p, 0, ks);
    c_to_a(a[1], p, 1, ks);
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t b[4];
      load_b_kn(b, y_tile, np, ks, lane, ys);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma_bf16(o[mt][2 * np], a[mt], b[0], b[1]);
        mma_bf16(o[mt][2 * np + 1], a[mt], b[2], b[3]);
      }
    }
  }
}
// out[32 x 32] = Z^T . Y   with Z, Y row-major [k][.] in smem (contraction over the smem row index; row strides zs, ys)
__device__ __forceinline__ void mul_t_kn(float (&o)[2][4][4], uint32_t z_tile, uint32_t y_tile, int lane, int zs = kRow,
                                         int ys = kRow) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    uint32_t a[2][4];
    load_a_t(a[0], z_tile, 0, ks, lane, zs);
    load_a_t(a[1], z_tile, 1, ks, lane, zs);
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t b[4];
      load_b_kn(b, y_tile, np, ks, lane, ys);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma_bf16(o[mt][2 * np], a[mt], b[0], b[1]);
        mma_bf16(o[mt][2 * np + 1], a[mt], b[2], b[3]);
      }
    }
  }
}
// store a C-fragment as bf16 (times mul) to rows i < L of a row-major smem tile with row stride st elements; rows >= L
// are left as they are (the zero padding of the streamed tiles)
__device__ __forceinline__ void store_c_rows(bf16* tile, int st, int L, const float (&c)[2][4][4], float mul, int g, int t) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int i = 16 * mt + g + 8 * hrow;
      if (i < L) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
          *reinterpret_cast<uint32_t*>(tile + i * st + 8 * nt + 2 * t) =
              pack_bf16(c[mt][nt][2 * hrow] * mul, c[mt][nt][2 * hrow + 1] * mul);
      }
    }
}
__device__ __forceinline__ void store_c_smem(bf16* tile, const float (&c)[2][4][4], int g, int t) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int i = 16 * mt + g + 8 * hrow;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
        *reinterpret_cast<uint32_t*>(tile + i * kRow + 8 * nt + 2 * t) = pack_bf16(c[mt][nt][2 * hrow], c[mt][nt][2 * hrow + 1]);
    }
}

// ---- sequence streaming ------------------------------------------------------------------------------------------
// The rows of a sequence are contiguous in qkv [nseq*L, 3d] (and dout [nseq*L, d]), so the kernels move whole sequences:
// CTAs are persistent (one wave) and walk the sequences blockIdx.x, + gridDim.x, ...  A producer warp (the last warp)
// copies each sequence into a ring of `stages` shared-memory stages with one bulk copy per row (lane r: row r), completed
// on the stage's `full` mbarrier, while the consumer warps compute the sequence before it.  Consumer warp w takes heads
// w, w + W, ... of the sequence (W = min(H, kStreamWarps)); every (sequence, head) pair runs exactly the arithmetic of the
// earlier warp-per-pair kernels, and its dropout pair index stays seq * H + h.
//
// A stage holds 32 qkv rows with a stride of 3d + 8 elements (and, in the backward, 32 dO rows with a stride of d + 8):
// 16 * odd bytes, so ldmatrix on a head's 32-column slice is free of bank conflicts.  Rows >= L are zeroed once when the
// kernel starts and never written again -- no copy covers them and every output store skips them -- so the padded rows
// of the 32 x 32 tiles reach the MMAs as zeros, as the backward requires (zero Q / dO rows make dS and the dV
// contributions of padded query rows exactly 0).  Outputs are written in place into the stage (o over the head's Q
// columns; dq, dk, dv over Q, K, V) and leave as one bulk store per row, issued by the producer once every consumer has
// released the stage; the producer waits until those stores have read the stage before it refills it.
constexpr int kStreamWarps = 8;          // consumer warps per CTA at most
constexpr int kStreamRows = 32;          // rows of a stage (the 32 x 32 tile height)
constexpr int kStreamMaxStages = 2;
constexpr int kStreamBarBytes = 64;      // full[kStreamMaxStages], empty[kStreamMaxStages] ahead of the stages
constexpr int kStreamSmemMax = 227 * 1024;

__host__ __device__ constexpr int stream_qkv_stride(int H) { return 96 * H + 8; }
__host__ __device__ constexpr int stream_dout_stride(int H) { return 32 * H + 8; }
// elements of one stage
__host__ __device__ constexpr int stream_stage_elems(int H, bool bwd) {
  return kStreamRows * (stream_qkv_stride(H) + (bwd ? stream_dout_stride(H) : 0));
}

// zero every stage, initialise the barriers; all threads, before any copy is issued
__device__ __forceinline__ void stream_init(unsigned char* smem, int stage_bytes, int stages, int consumers) {
  uint4* z = reinterpret_cast<uint4*>(smem + kStreamBarBytes);
  for (int i = threadIdx.x; i < stages * stage_bytes / 16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_smem();   // the zeros precede the bulk copies (async proxy) into the same stage
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&bars[s], 1);
      mbar_init(&bars[kStreamMaxStages + s], consumers);
    }
    fence_barrier_init();
  }
  __syncthreads();
}

// Producer warp: iteration k loads the CTA's k-th sequence into stage k % stages; first it stores the outputs of
// sequence k - stages out of that stage (once all consumers released it) and waits until the stores have read it.
// qkv rows (and dout rows) in; out_cols leading columns of each stage row out, to rows of `dst` with stride dst_ld.
__device__ __forceinline__ void stream_producer(unsigned char* smem, int stage_elems, int stages, const MmaAttnArgs& a,
                                                bool bwd, int lane) {
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + kStreamMaxStages;
  bf16* stage0 = reinterpret_cast<bf16*>(smem + kStreamBarBytes);
  const int L = a.L, d = a.H * 32, rs = stream_qkv_stride(a.H), rd = stream_dout_stride(a.H);
  const int n = (a.nseq - int(blockIdx.x) + int(gridDim.x) - 1) / int(gridDim.x);
  const uint32_t row_in = uint32_t(3 * d * 2 + (bwd ? d * 2 : 0));
  const int out_cols = bwd ? 3 * d : d;
  bf16* dst = bwd ? a.dqkv : a.out;
  for (int k = 0; k < n + stages; ++k) {
    const int s = k % stages;
    bf16* qkv_st = stage0 + size_t(s) * stage_elems;
    if (k >= stages) {
      mbar_wait(&empty[s], uint32_t((k / stages - 1) & 1));
      const size_t row0 = size_t(int(blockIdx.x) + (k - stages) * int(gridDim.x)) * L;
      if (lane < L) bulk_store(dst + (row0 + lane) * out_cols, qkv_st + lane * rs, uint32_t(out_cols * 2));
      tma_store_commit();
    }
    if (k < n) {
      if (k >= stages) tma_store_wait_read();   // this lane's row of the stage has been read out
      const size_t row0 = size_t(int(blockIdx.x) + k * int(gridDim.x)) * L;
      if (lane == 0) mbar_arrive_expect_tx(&full[s], uint32_t(L) * row_in);
      __syncwarp();
      if (lane < L) {
        bulk_load(qkv_st + lane * rs, a.qkv + (row0 + lane) * (3 * d), uint32_t(3 * d * 2), &full[s]);
        if (bwd)
          bulk_load(qkv_st + kStreamRows * rs + lane * rd, a.dout + (row0 + lane) * d, uint32_t(d * 2), &full[s]);
      }
    }
  }
  tma_store_wait_all();   // the stores have completed before the CTA exits
}

__global__ void __launch_bounds__((kStreamWarps + 1) * 32, 2) attn_mma_fwd_kernel(MmaAttnArgs a) {
  pdl_launch_dependents();
  extern __shared__ __align__(128) unsigned char smem[];
  const int W = int(blockDim.x >> 5) - 1, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, H = a.H, d = H * 32, rs = stream_qkv_stride(H), stages = a.stages;
  const int stage_elems = stream_stage_elems(H, false);
  stream_init(smem, stage_elems * 2, stages, W * 32);
  pdl_wait();
  if (warp == W) {
    stream_producer(smem, stage_elems, stages, a, false, lane);
    return;
  }
  drop_resolve(a.drop);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + kStreamMaxStages;
  bf16* stage0 = reinterpret_cast<bf16*>(smem + kStreamBarBytes);
  const int n = (a.nseq - int(blockIdx.x) + int(gridDim.x) - 1) / int(gridDim.x);
  for (int k = 0; k < n; ++k) {
    const int s = k % stages, seq = int(blockIdx.x) + k * int(gridDim.x);
    const size_t row0 = size_t(seq) * L;
    const uint32_t kmask = key_mask_of(a.valid, row0, L, lane);
    bf16* st = stage0 + size_t(s) * stage_elems;
    mbar_wait(&full[s], uint32_t((k / stages) & 1));
    for (int h = warp; h < H; h += W) {
      bf16* Qs = st + h * 32;
      const uint32_t q_t = smem_addr(Qs), k_t = smem_addr(Qs + d), v_t = smem_addr(Qs + 2 * d);
      const long long pair = (long long)seq * H + h;
      float sc[2][4][4];
      qk_scores(sc, q_t, k_t, lane, rs, rs);
      softmax_rows(sc, kmask, t, g, a.causal);
      if (a.drop.p > 0.f) {
        float mult[2][4][4];
        dropout_tile(mult, a.drop, (unsigned long long)pair, g, t);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) sc[mt][nt][e] *= mult[mt][nt][e];
      }
      float o[2][4][4];
      mul_regs_kn(o, sc, v_t, lane, rs);
      __syncwarp();                                // every lane is done with this head's Q
      store_c_rows(Qs, rs, L, o, 1.f, g, t);       // o over Q: the producer stores the first d columns of each row
    }
    fence_proxy_async_smem();                      // the generic-proxy writes above precede the bulk store that reads them
    mbar_arrive(&empty[s]);
  }
}

__global__ void __launch_bounds__((kStreamWarps + 1) * 32, 1) attn_mma_bwd_kernel(MmaAttnArgs a) {
  pdl_launch_dependents();
  extern __shared__ __align__(128) unsigned char smem[];
  const int W = int(blockDim.x >> 5) - 1, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, H = a.H, d = H * 32, rs = stream_qkv_stride(H), rd = stream_dout_stride(H), stages = a.stages;
  const int stage_elems = stream_stage_elems(H, true);
  stream_init(smem, stage_elems * 2, stages, W * 32);
  pdl_wait();
  if (warp == W) {
    stream_producer(smem, stage_elems, stages, a, true, lane);
    return;
  }
  drop_resolve(a.drop);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + kStreamMaxStages;
  bf16* stage0 = reinterpret_cast<bf16*>(smem + kStreamBarBytes);
  bf16* Ps = stage0 + size_t(stages) * stage_elems + warp * 2 * kTile;   // dropout-scaled probabilities (per warp)
  bf16* Ds = Ps + kTile;                                                 // dS
  const uint32_t p_t = smem_addr(Ps), d_t = smem_addr(Ds);
  const int n = (a.nseq - int(blockIdx.x) + int(gridDim.x) - 1) / int(gridDim.x);
  for (int k = 0; k < n; ++k) {
    const int s = k % stages, seq = int(blockIdx.x) + k * int(gridDim.x);
    const size_t row0 = size_t(seq) * L;
    const uint32_t kmask = key_mask_of(a.valid, row0, L, lane);
    bf16* st = stage0 + size_t(s) * stage_elems;
    mbar_wait(&full[s], uint32_t((k / stages) & 1));
    for (int h = warp; h < H; h += W) {
      bf16* Qs = st + h * 32;
      bf16* Ks = Qs + d;
      bf16* Vs = Qs + 2 * d;
      bf16* Gs = st + kStreamRows * rs + h * 32;   // dO
      const uint32_t q_t = smem_addr(Qs), k_t = smem_addr(Ks), v_t = smem_addr(Vs), g_t = smem_addr(Gs);
      const long long pair = (long long)seq * H + h;
      float p[2][4][4], dp[2][4][4];
      qk_scores(p, q_t, k_t, lane, rs, rs);
      softmax_rows(p, kmask, t, g, a.causal);
      qk_scores(dp, g_t, v_t, lane, rd, rs);       // dP = dO . V^T  (same operand shapes as Q . K^T)
      if (a.drop.p > 0.f) {
        float mult[2][4][4];
        dropout_tile(mult, a.drop, (unsigned long long)pair, g, t);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              dp[mt][nt][e] *= mult[mt][nt][e];   // d loss / d p  (through the dropout)
              mult[mt][nt][e] *= p[mt][nt][e];    // dropout-scaled probability (operand of dV)
            }
        store_c_smem(Ps, mult, g, t);
      } else {
        store_c_smem(Ps, p, g, t);
      }
      // dS = P o (dP - rowsum(dP o P))
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
          float delta = 0.f;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e) delta = fmaf(dp[mt][nt][2 * hrow + e], p[mt][nt][2 * hrow + e], delta);
          delta += __shfl_xor_sync(0xffffffffu, delta, 1);
          delta += __shfl_xor_sync(0xffffffffu, delta, 2);
#pragma unroll
          for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              dp[mt][nt][2 * hrow + e] = p[mt][nt][2 * hrow + e] * (dp[mt][nt][2 * hrow + e] - delta);
        }
      store_c_smem(Ds, dp, g, t);
      __syncwarp();
      float oq[2][4][4], ok[2][4][4];
      mul_regs_kn(oq, dp, k_t, lane, rs);          // dQ = dS . K
      mul_t_kn(ok, d_t, q_t, lane, kRow, rs);      // dK = dS^T . Q
      __syncwarp();                                // every lane is done with this head's Q and K (V: since dP)
      store_c_rows(Qs, rs, L, oq, a.scale, g, t);
      store_c_rows(Ks, rs, L, ok, 1.f, g, t);
      mul_t_kn(oq, p_t, g_t, lane, kRow, rd);      // dV = (dropout(P))^T . dO
      store_c_rows(Vs, rs, L, oq, 1.f, g, t);
      __syncwarp();                                // Ps / Ds are rewritten for the next head
    }
    fence_proxy_async_smem();                      // the generic-proxy writes above precede the bulk store that reads them
    mbar_arrive(&empty[s]);
  }
}

// ================================================================================================================
// Parity mode ("bf16x3") on the same 32 x 32 tiles: every activation is a (hi, lo) pair of bf16 planes carrying ~16
// mantissa bits, and every product X . Y is evaluated as Xh.Yh + Xh.Yl + Xl.Yh with fp32 accumulation (the dropped
// Xl.Yl term is 2^-16 of the product) -- the operand format and arithmetic of the bf16x3 GEMMs.  Probabilities and dS
// are produced in fp32 registers and split into (hi, lo) before they become operands.  Replaces the fp32 SIMT kernel
// (attention.cu) for two-plane tensors at head_dim 32, L <= 32: parity mode spent 16 of its 44 ms per step there.
// ================================================================================================================
constexpr int kX3Warps = 2;
constexpr int kX3FwdTiles = 6;    // Qh Ql Kh Kl Vh Vl
constexpr int kX3BwdTiles = 10;   // + Gh Gl Ph Pl ; dS (hi, lo) overlays V once dP = dO . V^T is in registers

__device__ __forceinline__ uint32_t pack_lo(float a, float b, uint32_t hi) {
  const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&hi);
  const float2 hf = __bfloat1622float2(h);
  return pack_bf16(a - hf.x, b - hf.y);
}
// acc += Xl.Yh + Xh.Yl + Xh.Yh for one n-tile (b registers i, j of the (hi, lo) B fragments): small terms first
#define DSVG_MMA3(acc, ah, al, bh, bl, i, j)   \
  mma_bf16(acc, al, bh[i], bh[j]);              \
  mma_bf16(acc, ah, bl[i], bl[j]);              \
  mma_bf16(acc, ah, bh[i], bh[j])
// S += X . Y^T over hi/lo planes (tiles row-major [row][channel]; the lo tile follows its hi tile)
__device__ __forceinline__ void qk_scores_x3(float (&s)[2][4][4], uint32_t x_t, uint32_t y_t, int lane) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[mt][nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    uint32_t ah[2][4], al[2][4];
    load_a(ah[0], x_t, 0, ks, lane);
    load_a(ah[1], x_t, 1, ks, lane);
    load_a(al[0], x_t + kTile * 2, 0, ks, lane);
    load_a(al[1], x_t + kTile * 2, 1, ks, lane);
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t bh[4], bl[4];
      load_b_nk(bh, y_t, np, ks, lane);
      load_b_nk(bl, y_t + kTile * 2, np, ks, lane);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        DSVG_MMA3(s[mt][2 * np], ah[mt], al[mt], bh, bl, 0, 1);
        DSVG_MMA3(s[mt][2 * np + 1], ah[mt], al[mt], bh, bl, 2, 3);
      }
    }
  }
}
__device__ __forceinline__ void c_to_a_x3(uint32_t (&ah)[4], uint32_t (&al)[4], const float (&c)[2][4][4], int mt, int ks) {
  c_to_a(ah, c, mt, ks);
  al[0] = pack_lo(c[mt][2 * ks][0], c[mt][2 * ks][1], ah[0]);
  al[1] = pack_lo(c[mt][2 * ks][2], c[mt][2 * ks][3], ah[1]);
  al[2] = pack_lo(c[mt][2 * ks + 1][0], c[mt][2 * ks + 1][1], ah[2]);
  al[3] = pack_lo(c[mt][2 * ks + 1][2], c[mt][2 * ks + 1][3], ah[3]);
}
// out = A(fp32 registers, split here) . Y   with Y (hi, lo) row-major [k][n] in smem
__device__ __forceinline__ void mul_regs_kn_x3(float (&o)[2][4][4], const float (&p)[2][4][4], uint32_t y_t, int lane) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    uint32_t ah[2][4], al[2][4];
    c_to_a_x3(ah[0], al[0], p, 0, ks);
    c_to_a_x3(ah[1], al[1], p, 1, ks);
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t bh[4], bl[4];
      load_b_kn(bh, y_t, np, ks, lane);
      load_b_kn(bl, y_t + kTile * 2, np, ks, lane);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        DSVG_MMA3(o[mt][2 * np], ah[mt], al[mt], bh, bl, 0, 1);
        DSVG_MMA3(o[mt][2 * np + 1], ah[mt], al[mt], bh, bl, 2, 3);
      }
    }
  }
}
// out = Z^T . Y   with Z, Y (hi, lo) row-major [k][.] in smem
__device__ __forceinline__ void mul_t_kn_x3(float (&o)[2][4][4], uint32_t z_t, uint32_t y_t, int lane) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    uint32_t ah[2][4], al[2][4];
    load_a_t(ah[0], z_t, 0, ks, lane);
    load_a_t(ah[1], z_t, 1, ks, lane);
    load_a_t(al[0], z_t + kTile * 2, 0, ks, lane);
    load_a_t(al[1], z_t + kTile * 2, 1, ks, lane);
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t bh[4], bl[4];
      load_b_kn(bh, y_t, np, ks, lane);
      load_b_kn(bl, y_t + kTile * 2, np, ks, lane);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        DSVG_MMA3(o[mt][2 * np], ah[mt], al[mt], bh, bl, 0, 1);
        DSVG_MMA3(o[mt][2 * np + 1], ah[mt], al[mt], bh, bl, 2, 3);
      }
    }
  }
}
// C-fragment -> (hi, lo) planes in global memory, rows i < L
__device__ __forceinline__ void store_c_global_x3(bf16* dst, size_t lo_off, int ld, int L, const float (&c)[2][4][4],
                                                  float mul, int g, int t) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int i = 16 * mt + g + 8 * hrow;
      if (i < L) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const float x = c[mt][nt][2 * hrow] * mul, y = c[mt][nt][2 * hrow + 1] * mul;
          const uint32_t hi = pack_bf16(x, y);
          bf16* p = dst + size_t(i) * ld + 8 * nt + 2 * t;
          *reinterpret_cast<uint32_t*>(p) = hi;
          *reinterpret_cast<uint32_t*>(p + lo_off) = pack_lo(x, y, hi);
        }
      }
    }
}
// C-fragment -> (hi, lo) tiles in shared memory (lo tile follows the hi tile)
__device__ __forceinline__ void store_c_smem_x3(bf16* tile, const float (&c)[2][4][4], int g, int t) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int i = 16 * mt + g + 8 * hrow;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const uint32_t hi = pack_bf16(c[mt][nt][2 * hrow], c[mt][nt][2 * hrow + 1]);
        bf16* p = tile + i * kRow + 8 * nt + 2 * t;
        *reinterpret_cast<uint32_t*>(p) = hi;
        *reinterpret_cast<uint32_t*>(p + kTile) = pack_lo(c[mt][nt][2 * hrow], c[mt][nt][2 * hrow + 1], hi);
      }
    }
}

struct X3AttnArgs {
  MmaAttnArgs m;
  size_t qkv_lo, out_lo, dout_lo, dqkv_lo;   // element offsets of the lo planes
};

__global__ void __launch_bounds__(kX3Warps * 32) attn_x3_fwd_kernel(X3AttnArgs x) {
  pdl_launch_dependents();
  pdl_wait();
  MmaAttnArgs& a = x.m;
  drop_resolve(a.drop);
  extern __shared__ __align__(16) bf16 sm_dyn[];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, d = a.H * 32, ld = 3 * d;
  bf16* Qs = sm_dyn + wib * kX3FwdTiles * kTile;   // hi tile, lo tile
  bf16* Ks = Qs + 2 * kTile;
  bf16* Vs = Ks + 2 * kTile;
  const uint32_t q_t = smem_addr(Qs), k_t = smem_addr(Ks), v_t = smem_addr(Vs);
  const long long npairs = (long long)a.nseq * a.H;
  for (long long pair = (long long)blockIdx.x * kX3Warps + wib; pair < npairs; pair += (long long)gridDim.x * kX3Warps) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    const bf16* base = a.qkv + row0 * ld + h * 32;
    stage_tile(Qs, base, ld, L, lane);
    stage_tile(Qs + kTile, base + x.qkv_lo, ld, L, lane);
    stage_tile(Ks, base + d, ld, L, lane);
    stage_tile(Ks + kTile, base + d + x.qkv_lo, ld, L, lane);
    stage_tile(Vs, base + 2 * d, ld, L, lane);
    stage_tile(Vs + kTile, base + 2 * d + x.qkv_lo, ld, L, lane);
    const uint32_t kmask = key_mask_of(a.valid, row0, L, lane);
    __syncwarp();
    float s[2][4][4];
    qk_scores_x3(s, q_t, k_t, lane);
    softmax_rows(s, kmask, t, g, a.causal);
    if (a.drop.p > 0.f) {
      float mult[2][4][4];
      dropout_tile(mult, a.drop, (unsigned long long)pair, g, t);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) s[mt][nt][e] *= mult[mt][nt][e];
    }
    float o[2][4][4];
    mul_regs_kn_x3(o, s, v_t, lane);
    store_c_global_x3(a.out + row0 * d + h * 32, x.out_lo, d, L, o, 1.f, g, t);
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kX3Warps * 32) attn_x3_bwd_kernel(X3AttnArgs x) {
  pdl_launch_dependents();
  pdl_wait();
  MmaAttnArgs& a = x.m;
  drop_resolve(a.drop);
  extern __shared__ __align__(16) bf16 sm_dyn[];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, d = a.H * 32, ld = 3 * d;
  bf16* Qs = sm_dyn + wib * kX3BwdTiles * kTile;
  bf16* Ks = Qs + 2 * kTile;
  bf16* Vs = Ks + 2 * kTile;
  bf16* Gs = Vs + 2 * kTile;   // dO
  bf16* Ps = Gs + 2 * kTile;   // dropout-scaled probabilities
  bf16* Ds = Vs;               // dS: V is dead once dP is in registers
  const uint32_t q_t = smem_addr(Qs), k_t = smem_addr(Ks), v_t = smem_addr(Vs), g_t = smem_addr(Gs),
                 p_t = smem_addr(Ps), d_t = smem_addr(Ds);
  const long long npairs = (long long)a.nseq * a.H;
  for (long long pair = (long long)blockIdx.x * kX3Warps + wib; pair < npairs; pair += (long long)gridDim.x * kX3Warps) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    const bf16* base = a.qkv + row0 * ld + h * 32;
    const bf16* gbase = a.dout + row0 * d + h * 32;
    stage_tile(Qs, base, ld, L, lane);
    stage_tile(Qs + kTile, base + x.qkv_lo, ld, L, lane);
    stage_tile(Ks, base + d, ld, L, lane);
    stage_tile(Ks + kTile, base + d + x.qkv_lo, ld, L, lane);
    stage_tile(Vs, base + 2 * d, ld, L, lane);
    stage_tile(Vs + kTile, base + 2 * d + x.qkv_lo, ld, L, lane);
    stage_tile(Gs, gbase, d, L, lane);
    stage_tile(Gs + kTile, gbase + x.dout_lo, d, L, lane);
    const uint32_t kmask = key_mask_of(a.valid, row0, L, lane);
    __syncwarp();
    float p[2][4][4], dp[2][4][4];
    qk_scores_x3(p, q_t, k_t, lane);
    softmax_rows(p, kmask, t, g, a.causal);
    qk_scores_x3(dp, g_t, v_t, lane);          // dP = dO . V^T
    __syncwarp();                              // every lane is done with V before dS overwrites it
    if (a.drop.p > 0.f) {
      float mult[2][4][4];
      dropout_tile(mult, a.drop, (unsigned long long)pair, g, t);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            dp[mt][nt][e] *= mult[mt][nt][e];
            mult[mt][nt][e] *= p[mt][nt][e];
          }
      store_c_smem_x3(Ps, mult, g, t);
    } else {
      store_c_smem_x3(Ps, p, g, t);
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int hrow = 0; hrow < 2; ++hrow) {
        float delta = 0.f;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) delta = fmaf(dp[mt][nt][2 * hrow + e], p[mt][nt][2 * hrow + e], delta);
        delta += __shfl_xor_sync(0xffffffffu, delta, 1);
        delta += __shfl_xor_sync(0xffffffffu, delta, 2);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            dp[mt][nt][2 * hrow + e] = p[mt][nt][2 * hrow + e] * (dp[mt][nt][2 * hrow + e] - delta);
      }
    store_c_smem_x3(Ds, dp, g, t);
    __syncwarp();
    float o[2][4][4];
    bf16* dbase = a.dqkv + row0 * ld + h * 32;
    mul_regs_kn_x3(o, dp, k_t, lane);              // dQ = dS . K
    store_c_global_x3(dbase, x.dqkv_lo, ld, L, o, a.scale, g, t);
    mul_t_kn_x3(o, d_t, q_t, lane);                // dK = dS^T . Q
    store_c_global_x3(dbase + d, x.dqkv_lo, ld, L, o, 1.f, g, t);
    mul_t_kn_x3(o, p_t, g_t, lane);                // dV = (dropout(P))^T . dO
    store_c_global_x3(dbase + 2 * d, x.dqkv_lo, ld, L, o, 1.f, g, t);
    __syncwarp();
  }
}

}  // namespace dsvg
using namespace dsvg;

// Launch of the sequence-streaming 32 x 32 kernels: W = min(H, kStreamWarps) consumer warps plus the producer warp, two
// stages when they fit in shared memory (one otherwise), and exactly one wave of resident CTAs (at most one per sequence).
static int launch_stream(bool bwd, MmaAttnArgs& a, cudaStream_t st) {
  DSVG_CHECK(a.L >= 1 && a.L <= kStreamRows, "attn_mma: L = %d outside 1..%d", a.L, kStreamRows);
  const uintptr_t align = reinterpret_cast<uintptr_t>(a.qkv) | reinterpret_cast<uintptr_t>(a.out) |
                          reinterpret_cast<uintptr_t>(a.dout) | reinterpret_cast<uintptr_t>(a.dqkv);   // unused ones are null
  DSVG_CHECK((align & 15) == 0, "attn_mma: qkv / dout / outputs must be 16-byte aligned for the bulk copies");
  const int W = a.H < kStreamWarps ? a.H : kStreamWarps;
  const long long stage = 2LL * stream_stage_elems(a.H, bwd);
  const long long fixed = kStreamBarBytes + (bwd ? 2LL * W * 2 * kTile : 0);   // + per-warp P / dS tiles
  a.stages = fixed + 2 * stage <= kStreamSmemMax ? 2 : 1;
  const long long smem = fixed + a.stages * stage;
  DSVG_CHECK(smem <= kStreamSmemMax, "attn_mma: H = %d heads need %lld bytes of shared memory per sequence (max %d)", a.H,
             smem, kStreamSmemMax);
  auto kern = bwd ? attn_mma_bwd_kernel : attn_mma_fwd_kernel;
  static bool configured[2][kMaxDevices] = {};
  if (first_use_on_device(configured[bwd]))
    DSVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmemMax));
  int dev = 0, sms = 0, per_sm = 0;
  DSVG_CUDA(cudaGetDevice(&dev));
  DSVG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  DSVG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, (W + 1) * 32, size_t(smem)));
  DSVG_CHECK(per_sm > 0, "attn_mma: %lld bytes of shared memory per CTA do not fit", smem);
  long long blocks = (long long)sms * per_sm;
  if (blocks > a.nseq) blocks = a.nseq;
  DSVG_CUDA(launch_k(kern, dim3(int(blocks)), dim3((W + 1) * 32), size_t(smem), st, a));
  ++g_launches;
  return 0;
}

// Entry points used by attention.cu's dispatcher (not part of the public header: same ABI functions, faster path).
int dsvg_attn_mma_fwd(const bf16* qkv, const uint8_t* valid, bf16* out, int nseq, int L, int H, Dropout drop, int causal,
                      cudaStream_t st) {
  MmaAttnArgs a{};
  a.qkv = qkv; a.valid = valid; a.out = out; a.nseq = nseq; a.L = L; a.H = H; a.scale = 1.f; a.drop = drop;
  a.causal = causal;
  return launch_stream(false, a, st);
}
int dsvg_attn_mma_bwd(const bf16* qkv, const uint8_t* valid, const bf16* dout, bf16* dqkv, int nseq, int L, int H,
                      float q_scale, Dropout drop, int causal, cudaStream_t st) {
  MmaAttnArgs a{};
  a.qkv = qkv; a.valid = valid; a.dout = dout; a.dqkv = dqkv; a.nseq = nseq; a.L = L; a.H = H; a.scale = q_scale;
  a.drop = drop; a.causal = causal;
  return launch_stream(true, a, st);
}

// Parity-mode (two-plane) entry point of the 32 x 32 kernels.
int dsvg_attn_x3(bool bwd, const bf16* qkv, size_t qkv_lo, const uint8_t* valid, bf16* out, size_t out_lo, const bf16* dout,
                 size_t dout_lo, bf16* dqkv, size_t dqkv_lo, int nseq, int L, int H, float q_scale, Dropout drop, int causal,
                 cudaStream_t st) {
  X3AttnArgs x{};
  MmaAttnArgs& a = x.m;
  a.qkv = qkv; a.valid = valid; a.out = out; a.dout = dout; a.dqkv = dqkv; a.nseq = nseq; a.L = L; a.H = H;
  a.scale = q_scale; a.drop = drop; a.causal = causal;
  x.qkv_lo = qkv_lo; x.out_lo = out_lo; x.dout_lo = dout_lo; x.dqkv_lo = dqkv_lo;
  const int smem = kX3Warps * (bwd ? kX3BwdTiles : kX3FwdTiles) * kTile * 2;
  static bool configured[kMaxDevices] = {};
  static long long cap[2] = {0, 0};
  if (first_use_on_device(configured)) {
    DSVG_CUDA(cudaFuncSetAttribute(attn_x3_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kX3Warps * kX3FwdTiles * kTile * 2));
    DSVG_CUDA(cudaFuncSetAttribute(attn_x3_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kX3Warps * kX3BwdTiles * kTile * 2));
  }
  if (cap[bwd] == 0) {
    int n = 0;
    if (bwd) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, attn_x3_bwd_kernel, kX3Warps * 32, size_t(smem));
    else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, attn_x3_fwd_kernel, kX3Warps * 32, size_t(smem));
    cap[bwd] = 132LL * (n > 0 ? n : 4);
  }
  long long blocks = ((long long)nseq * H + kX3Warps - 1) / kX3Warps;
  if (blocks > cap[bwd]) blocks = cap[bwd];
  if (bwd) DSVG_CUDA(launch_k(attn_x3_bwd_kernel, dim3(int(blocks)), dim3(kX3Warps * 32), size_t(smem), st, x));
  else DSVG_CUDA(launch_k(attn_x3_fwd_kernel, dim3(int(blocks)), dim3(kX3Warps * 32), size_t(smem), st, x));
  ++g_launches;
  return 0;
}

// ================================================================================================================
// General tensor-core path: head_dim 32 / 64, sequences of up to 80 positions (one-stage fonts: L = 52 / 51; scaled
// hierarchical: L = 66 / 65 path-level, 16 group-level).  One CTA owns one (sequence, head) pair at a time; warp w owns
// the 16-row query tile w of the LP = 16 * NT padded positions (and, in the backward, the 16-row key tile w of dK / dV).
// Q, K, V (and dO) of the pair are staged once in shared memory; the LP x LP probability / dS tiles of the backward go
// through shared memory as bf16 so that every product is an mma.sync m16n8k16 with ldmatrix-fed operands.
//   reference: functional.py:168-248 (same arithmetic as the 32 x 32 kernel above).
// ================================================================================================================
namespace dsvg {

// fragment loaders on a row-major bf16 tile with `st` elements between rows (st * 2 bytes = odd multiple of 16)
__device__ __forceinline__ void g_load_a(uint32_t (&a)[4], uint32_t tile, int row0, int k0, int st, int lane) {
  const int m = lane >> 3, r = lane & 7;
  ldsm_x4(a, tile + ((row0 + (m & 1) * 8 + r) * st + k0 + (m >> 1) * 8) * 2);
}
__device__ __forceinline__ void g_load_a_t(uint32_t (&a)[4], uint32_t tile, int m0, int k0, int st, int lane) {
  const int m = lane >> 3, r = lane & 7;
  ldsm_x4_t(a, tile + ((k0 + (m >> 1) * 8 + r) * st + m0 + (m & 1) * 8) * 2);
}
__device__ __forceinline__ void g_load_b_nk(uint32_t (&b)[4], uint32_t tile, int n0, int k0, int st, int lane) {
  const int m = lane >> 3, r = lane & 7;
  ldsm_x4(b, tile + ((n0 + (m >> 1) * 8 + r) * st + k0 + (m & 1) * 8) * 2);
}
__device__ __forceinline__ void g_load_b_kn(uint32_t (&b)[4], uint32_t tile, int n0, int k0, int st, int lane) {
  const int m = lane >> 3, r = lane & 7;
  ldsm_x4_t(b, tile + ((k0 + (m & 1) * 8 + r) * st + n0 + (m >> 1) * 8) * 2);
}

template <int HD, int NT>
struct GAttn {
  static constexpr int LP = 16 * NT;
  static constexpr int SH = HD + 8;        // row stride of the [LP x HD] tiles
  static constexpr int SP = LP + 8;        // row stride of the [LP x LP] tiles
  static constexpr int kThreads = 32 * NT;
  static constexpr int kTileH = LP * SH;   // elements
  static constexpr int kTileP = LP * SP;
  static constexpr int kSmemFwd = 3 * kTileH * 2 + LP;
  static constexpr int kSmemBwd = 4 * kTileH * 2 + 2 * kTileP * 2 + LP;
};

// 16-byte asynchronous global -> shared copy (LDGSTS); !valid zero-fills the destination without reading the source
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// Stage one [L x HD] head slice into a zero-padded [LP x HD] tile.  All of a thread's 16-byte pieces are issued as
// asynchronous copies before anything waits: with a load -> store loop every thread had ONE 16-byte load in flight
// (15 KB per SM), which capped the first version of this kernel at 1.35 TB/s.
template <int HD, int NT>
__device__ __forceinline__ void g_stage(bf16* dst, const bf16* src, int ld, int L) {
  using G = GAttn<HD, NT>;
  constexpr int kParts = HD / 8;
  const uint32_t d0 = smem_addr(dst);
#pragma unroll
  for (int it = 0; it < (G::LP * kParts + G::kThreads - 1) / G::kThreads; ++it) {
    const int chunk = threadIdx.x + it * G::kThreads;
    if (chunk < G::LP * kParts) {
      const int row = chunk / kParts, part = chunk % kParts;
      const bool ok = row < L;
      cp_async16(d0 + (row * G::SH + part * 8) * 2, src + (ok ? size_t(row) * ld + part * 8 : 0), ok);
    }
  }
}

// S[16 x LP] = X_w . Y^T with X rows [16 w, +16) of `x_tile`, Y = `y_tile` (both [LP x HD], row-major)
template <int HD, int NT>
__device__ __forceinline__ void g_scores(float (&s)[2 * NT][4], uint32_t x_tile, uint32_t y_tile, int w, int lane) {
  using G = GAttn<HD, NT>;
#pragma unroll
  for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) s[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < HD / 16; ++ks) {
    uint32_t a[4];
    g_load_a(a, x_tile, 16 * w, 16 * ks, G::SH, lane);
#pragma unroll
    for (int np = 0; np < NT; ++np) {
      uint32_t b[4];
      g_load_b_nk(b, y_tile, 16 * np, 16 * ks, G::SH, lane);
      mma_bf16(s[2 * np], a, b[0], b[1]);
      mma_bf16(s[2 * np + 1], a, b[2], b[3]);
    }
  }
}

// this thread's key columns: bit (2 nt + e) <-> column 8 nt + 2 t + e
template <int NT>
__device__ __forceinline__ uint32_t g_my_keys(const uint8_t* kv_sm, int t) {
  uint32_t bits = 0;
#pragma unroll
  for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
    for (int e = 0; e < 2; ++e)
      if (kv_sm[8 * nt + 2 * t + e]) bits |= 1u << (2 * nt + e);
  return bits;
}

// row0: first query row of this warp's tile; t: lane & 3; g: lane >> 2; causal: query i sees keys j <= i only
template <int NT>
__device__ __forceinline__ void g_softmax(float (&s)[2 * NT][4], uint32_t keys, int row0 = 0, int g = 0, int t = 0,
                                          int causal = 0) {
  constexpr uint32_t kAll = (2 * NT * 2 >= 32) ? 0xFFFFFFFFu : ((1u << (2 * NT * 2)) - 1u);
  const bool masked = causal || (keys & kAll) != kAll;   // unmasked tiles skip the selects
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    float m = -INFINITY;
    const int i = row0 + g + 8 * hrow;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& x = s[nt][2 * hrow + e];
        if (masked && (!((keys >> (2 * nt + e)) & 1u) || (causal && 8 * nt + 2 * t + e > i))) x = -INFINITY;
        m = fmaxf(m, x);
      }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    float sum = 0.f;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& x = s[nt][2 * hrow + e];
        x = __expf(x - m);
        sum += x;
      }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    const float inv = 1.f / sum;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) s[nt][2 * hrow + e] *= inv;
  }
}

// dropout multipliers of this thread's elements: one quad (4 draws) per (pair, row, key-tile pair np, t)
template <int NT>
__device__ __forceinline__ void g_dropout(float (&mult)[2 * NT][4], const Dropout& d, unsigned long long pair, int w, int g,
                                          int t) {
  constexpr int LP = 16 * NT;
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int i = 16 * w + g + 8 * hrow;
    const unsigned long long q_row = ((pair * LP + i) * NT) * 4ull;
#pragma unroll
    for (int np = 0; np < NT; ++np) {
      const unsigned long long quad = q_row + (unsigned long long)(np * 4 + t);
      const uint32_t s1 = drop_stage1(uint32_t(quad), drop_hikey(d, quad));
      const uint32_t a = drop_fin_a(s1), b = drop_fin_b(s1);
      mult[2 * np][2 * hrow] = drop_keep_lo(a, d.thr16) ? d.scale : 0.f;
      mult[2 * np][2 * hrow + 1] = drop_keep_hi(a, d.thr16) ? d.scale : 0.f;
      mult[2 * np + 1][2 * hrow] = drop_keep_lo(b, d.thr16) ? d.scale : 0.f;
      mult[2 * np + 1][2 * hrow + 1] = drop_keep_hi(b, d.thr16) ? d.scale : 0.f;
    }
  }
}

// out[16 x HD] = A(regs: 16 x LP in C-fragment layout) . Y,  Y = [LP x HD] row-major tile
template <int HD, int NT>
__device__ __forceinline__ void g_mul_regs(float (&o)[HD / 8][4], const float (&p)[2 * NT][4], uint32_t y_tile, int lane) {
  using G = GAttn<HD, NT>;
#pragma unroll
  for (int nt = 0; nt < HD / 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < NT; ++ks) {
    uint32_t a[4];
    a[0] = pack_bf16(p[2 * ks][0], p[2 * ks][1]);
    a[1] = pack_bf16(p[2 * ks][2], p[2 * ks][3]);
    a[2] = pack_bf16(p[2 * ks + 1][0], p[2 * ks + 1][1]);
    a[3] = pack_bf16(p[2 * ks + 1][2], p[2 * ks + 1][3]);
#pragma unroll
    for (int np = 0; np < HD / 16; ++np) {
      uint32_t b[4];
      g_load_b_kn(b, y_tile, 16 * np, 16 * ks, G::SH, lane);
      mma_bf16(o[2 * np], a, b[0], b[1]);
      mma_bf16(o[2 * np + 1], a, b[2], b[3]);
    }
  }
}
// out[16 x HD] (rows = key tile w) = Z^T . Y with Z = [LP(query) x LP(key)] tile (stride SP), Y = [LP(query) x HD] tile
template <int HD, int NT>
__device__ __forceinline__ void g_mul_t(float (&o)[HD / 8][4], uint32_t z_tile, uint32_t y_tile, int w, int lane) {
  using G = GAttn<HD, NT>;
#pragma unroll
  for (int nt = 0; nt < HD / 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < NT; ++ks) {
    uint32_t a[4];
    g_load_a_t(a, z_tile, 16 * w, 16 * ks, G::SP, lane);
#pragma unroll
    for (int np = 0; np < HD / 16; ++np) {
      uint32_t b[4];
      g_load_b_kn(b, y_tile, 16 * np, 16 * ks, G::SH, lane);
      mma_bf16(o[2 * np], a, b[0], b[1]);
      mma_bf16(o[2 * np + 1], a, b[2], b[3]);
    }
  }
}
template <int HD>
__device__ __forceinline__ void g_store_global(bf16* dst, int ld, int L, int row0, const float (&c)[HD / 8][4], float mul,
                                               int g, int t) {
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int i = row0 + g + 8 * hrow;
    if (i < L) {
#pragma unroll
      for (int nt = 0; nt < HD / 8; ++nt)
        *reinterpret_cast<uint32_t*>(dst + size_t(i) * ld + 8 * nt + 2 * t) =
            pack_bf16(c[nt][2 * hrow] * mul, c[nt][2 * hrow + 1] * mul);
    }
  }
}
template <int NT>
__device__ __forceinline__ void g_store_rows_smem(bf16* tile, int st, int row0, const float (&c)[2 * NT][4], int g, int t) {
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int i = row0 + g + 8 * hrow;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt)
      *reinterpret_cast<uint32_t*>(tile + i * st + 8 * nt + 2 * t) = pack_bf16(c[nt][2 * hrow], c[nt][2 * hrow + 1]);
  }
}

// DB: two sets of Q/K/V tiles -- the next pair's asynchronous copies fly while the current pair is computed
// The forward is issue/latency-bound rather than HBM-bound (several thousand warp instructions per (sequence, head) pair): it
// keeps its natural register count and the double-buffered staging instead of capping registers for more resident warps.
template <int HD, int NT, bool DB>
__global__ void __launch_bounds__(32 * NT) attn_gmma_fwd_kernel(MmaAttnArgs a) {
  using G = GAttn<HD, NT>;
  pdl_launch_dependents();
  pdl_wait();
  drop_resolve(a.drop);
  extern __shared__ __align__(16) bf16 sm_dyn[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, d = a.H * HD, ld = 3 * d;
  constexpr int kSet = 3 * G::kTileH;                       // elements of one Q/K/V set
  uint8_t* kv_base = reinterpret_cast<uint8_t*>(sm_dyn + (DB ? 2 : 1) * kSet);
  const long long npairs = (long long)a.nseq * a.H;
  auto issue = [&](long long pair, int b) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    const bf16* base = a.qkv + row0 * ld + h * HD;
    bf16* Qs = sm_dyn + b * kSet;
    g_stage<HD, NT>(Qs, base, ld, L);
    g_stage<HD, NT>(Qs + G::kTileH, base + d, ld, L);
    g_stage<HD, NT>(Qs + 2 * G::kTileH, base + 2 * d, ld, L);
    cp_async_commit();
    uint8_t* kv = kv_base + b * G::LP;
    for (int j = threadIdx.x; j < G::LP; j += G::kThreads) kv[j] = (j < L && (a.valid == nullptr || a.valid[row0 + j] != 0)) ? 1 : 0;
  };
  long long pair = blockIdx.x;
  int b = 0;
  if (pair < npairs) issue(pair, 0);
  for (; pair < npairs; pair += gridDim.x) {
    const long long next = pair + gridDim.x;
    if (DB && next < npairs) {
      issue(next, b ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");   // everything but the group just committed has landed
    } else {
      cp_async_wait_all();
    }
    __syncthreads();
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    const uint32_t q_t = smem_addr(sm_dyn + b * kSet), k_t = q_t + G::kTileH * 2, v_t = k_t + G::kTileH * 2;
    float s[2 * NT][4];
    g_scores<HD, NT>(s, q_t, k_t, w, lane);
    g_softmax<NT>(s, g_my_keys<NT>(kv_base + b * G::LP, t), 16 * w, g, t, a.causal);
    if (a.drop.p > 0.f) {
      float mult[2 * NT][4];
      g_dropout<NT>(mult, a.drop, (unsigned long long)pair, w, g, t);
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[nt][e] *= mult[nt][e];
    }
    float o[HD / 8][4];
    g_mul_regs<HD, NT>(o, s, v_t, lane);
    g_store_global<HD>(a.out + row0 * d + h * HD, d, L, 16 * w, o, 1.f, g, t);
    __syncthreads();                                          // all warps are done with this set before it is refilled
    if (DB) b ^= 1;
    else if (next < npairs) issue(next, 0);
  }
}

// backward: 168 registers allowed 2 CTAs per SM; capped at 128 (no spills) for 3: 885 -> 802 us at (4096 x 66, head_dim 64)
__host__ __device__ constexpr int gmma_bwd_min_ctas(int nt) { return nt >= 5 ? 3 : (nt == 4 ? 4 : 6); }
template <int HD, int NT>
__global__ void __launch_bounds__(32 * NT, gmma_bwd_min_ctas(NT)) attn_gmma_bwd_kernel(MmaAttnArgs a) {
  using G = GAttn<HD, NT>;
  pdl_launch_dependents();
  pdl_wait();
  drop_resolve(a.drop);
  extern __shared__ __align__(16) bf16 sm_dyn[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, d = a.H * HD, ld = 3 * d;
  bf16* Qs = sm_dyn;
  bf16* Ks = Qs + G::kTileH;
  bf16* Vs = Ks + G::kTileH;
  bf16* Gs = Vs + G::kTileH;   // dO
  bf16* Ps = Gs + G::kTileH;   // dropout-scaled probabilities  [query][key]
  bf16* Ds = Ps + G::kTileP;   // dS                            [query][key]
  uint8_t* kv = reinterpret_cast<uint8_t*>(Ds + G::kTileP);
  const uint32_t q_t = smem_addr(Qs), k_t = smem_addr(Ks), v_t = smem_addr(Vs), g_t = smem_addr(Gs), p_t = smem_addr(Ps),
                 d_t = smem_addr(Ds);
  const long long npairs = (long long)a.nseq * a.H;
  for (long long pair = blockIdx.x; pair < npairs; pair += gridDim.x) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    const bf16* base = a.qkv + row0 * ld + h * HD;
    g_stage<HD, NT>(Qs, base, ld, L);
    g_stage<HD, NT>(Ks, base + d, ld, L);
    g_stage<HD, NT>(Vs, base + 2 * d, ld, L);
    g_stage<HD, NT>(Gs, a.dout + row0 * d + h * HD, d, L);
    cp_async_commit();
    for (int j = threadIdx.x; j < G::LP; j += G::kThreads) kv[j] = (j < L && (a.valid == nullptr || a.valid[row0 + j] != 0)) ? 1 : 0;
    cp_async_wait_all();
    __syncthreads();
    float p[2 * NT][4], dp[2 * NT][4];
    g_scores<HD, NT>(p, q_t, k_t, w, lane);
    g_softmax<NT>(p, g_my_keys<NT>(kv, t), 16 * w, g, t, a.causal);
    g_scores<HD, NT>(dp, g_t, v_t, w, lane);          // dP = dO . V^T
    if (a.drop.p > 0.f) {
      float mult[2 * NT][4];
      g_dropout<NT>(mult, a.drop, (unsigned long long)pair, w, g, t);
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          dp[nt][e] *= mult[nt][e];
          mult[nt][e] *= p[nt][e];
        }
      g_store_rows_smem<NT>(Ps, G::SP, 16 * w, mult, g, t);
    } else {
      g_store_rows_smem<NT>(Ps, G::SP, 16 * w, p, g, t);
    }
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      float delta = 0.f;
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) delta = fmaf(dp[nt][2 * hrow + e], p[nt][2 * hrow + e], delta);
      delta += __shfl_xor_sync(0xffffffffu, delta, 1);
      delta += __shfl_xor_sync(0xffffffffu, delta, 2);
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) dp[nt][2 * hrow + e] = p[nt][2 * hrow + e] * (dp[nt][2 * hrow + e] - delta);
    }
    g_store_rows_smem<NT>(Ds, G::SP, 16 * w, dp, g, t);
    float o[HD / 8][4];
    bf16* dbase = a.dqkv + row0 * ld + h * HD;
    g_mul_regs<HD, NT>(o, dp, k_t, lane);                 // dQ rows of this warp = dS_w . K
    g_store_global<HD>(dbase, ld, L, 16 * w, o, a.scale, g, t);
    __syncthreads();                                      // every warp's rows of P and dS are in shared memory
    g_mul_t<HD, NT>(o, d_t, q_t, w, lane);                // dK rows [16 w, +16) = dS^T . Q
    g_store_global<HD>(dbase + d, ld, L, 16 * w, o, 1.f, g, t);
    g_mul_t<HD, NT>(o, p_t, g_t, w, lane);                // dV rows = dropout(P)^T . dO
    g_store_global<HD>(dbase + 2 * d, ld, L, 16 * w, o, 1.f, g, t);
    __syncthreads();
  }
}

template <int HD, int NT, bool BWD, bool DB>
static int launch_gmma_k(const MmaAttnArgs& a, cudaStream_t st) {
  using G = GAttn<HD, NT>;
  const int smem = BWD ? G::kSmemBwd : (DB ? 2 : 1) * G::kSmemFwd;
  auto kern = [] {
    if constexpr (BWD) return attn_gmma_bwd_kernel<HD, NT>;
    else return attn_gmma_fwd_kernel<HD, NT, DB>;
  }();
  // one wave of resident CTAs (registers AND shared memory decide how many fit: a grid sized from shared memory alone ran a
  // ragged second wave at half occupancy); the kernel strides over the pairs
  static int per_sm = 0;
  static bool configured[kMaxDevices] = {};
  if (first_use_on_device(configured)) {
    DSVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int n = 0;
    DSVG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, G::kThreads, size_t(smem)));
    per_sm = n > 0 ? n : 1;
  }
  int sms = 132;
  {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  const long long npairs = (long long)a.nseq * a.H;
  long long blocks = (long long)sms * per_sm;
  if (blocks > npairs) blocks = npairs;
  DSVG_CUDA(launch_k(kern, dim3(int(blocks)), dim3(G::kThreads), size_t(smem), st, a));
  ++g_launches;
  return 0;
}
template <int HD, int NT>
static int launch_gmma(bool bwd, const MmaAttnArgs& a, cudaStream_t st) {
  if (bwd) return launch_gmma_k<HD, NT, true, false>(a, st);
  // double-buffered staging when two sets leave room for >= 2 CTAs per SM (measured: 401 vs 413 us at 4096 x 66, head_dim 64)
  if (2 * GAttn<HD, NT>::kSmemFwd <= 100 * 1024) return launch_gmma_k<HD, NT, false, true>(a, st);
  return launch_gmma_k<HD, NT, false, false>(a, st);
}
template <int HD>
static int launch_gmma_nt(bool bwd, const MmaAttnArgs& a, cudaStream_t st) {
  switch ((a.L + 15) / 16) {
    case 1: return launch_gmma<HD, 1>(bwd, a, st);
    case 2: return launch_gmma<HD, 2>(bwd, a, st);
    case 3: return launch_gmma<HD, 3>(bwd, a, st);
    case 4: return launch_gmma<HD, 4>(bwd, a, st);
    case 5: return launch_gmma<HD, 5>(bwd, a, st);
    default: DSVG_CHECK(false, "tensor-core attention: L = %d exceeds 80 positions", a.L);
  }
}


// ----------------------------------------------------------------------------------------------------------------
// Parity mode (two bf16 planes, three products per contraction) of the general kernels: same tiling, every operand tile
// followed by its lo tile, probabilities / dS split into (hi, lo) when they become operands.  Replaces the fp32 SIMT
// kernels for BASELINE configs[3] / [4] in bf16x3 (scaled hierarchical: 794 ms per parity step, most of it SIMT attention).
// ----------------------------------------------------------------------------------------------------------------
template <int HD, int NT>
struct GX3 {
  using G = GAttn<HD, NT>;
  static constexpr int kSmemFwd = 6 * G::kTileH * 2 + G::LP;
  static constexpr int kSmemBwd = 8 * G::kTileH * 2 + 4 * G::kTileP * 2 + G::LP;
};

template <int HD, int NT>
__device__ __forceinline__ void gx3_scores(float (&s)[2 * NT][4], uint32_t x_tile, uint32_t y_tile, int w, int lane) {
  using G = GAttn<HD, NT>;
  constexpr uint32_t kLo = G::kTileH * 2;
#pragma unroll
  for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) s[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < HD / 16; ++ks) {
    uint32_t ah[4], al[4];
    g_load_a(ah, x_tile, 16 * w, 16 * ks, G::SH, lane);
    g_load_a(al, x_tile + kLo, 16 * w, 16 * ks, G::SH, lane);
#pragma unroll
    for (int np = 0; np < NT; ++np) {
      uint32_t bh[4], bl[4];
      g_load_b_nk(bh, y_tile, 16 * np, 16 * ks, G::SH, lane);
      g_load_b_nk(bl, y_tile + kLo, 16 * np, 16 * ks, G::SH, lane);
      DSVG_MMA3(s[2 * np], ah, al, bh, bl, 0, 1);
      DSVG_MMA3(s[2 * np + 1], ah, al, bh, bl, 2, 3);
    }
  }
}
template <int HD, int NT>
__device__ __forceinline__ void gx3_mul_regs(float (&o)[HD / 8][4], const float (&p)[2 * NT][4], uint32_t y_tile, int lane) {
  using G = GAttn<HD, NT>;
  constexpr uint32_t kLo = G::kTileH * 2;
#pragma unroll
  for (int nt = 0; nt < HD / 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < NT; ++ks) {
    uint32_t ah[4], al[4];
    ah[0] = pack_bf16(p[2 * ks][0], p[2 * ks][1]);
    ah[1] = pack_bf16(p[2 * ks][2], p[2 * ks][3]);
    ah[2] = pack_bf16(p[2 * ks + 1][0], p[2 * ks + 1][1]);
    ah[3] = pack_bf16(p[2 * ks + 1][2], p[2 * ks + 1][3]);
    al[0] = pack_lo(p[2 * ks][0], p[2 * ks][1], ah[0]);
    al[1] = pack_lo(p[2 * ks][2], p[2 * ks][3], ah[1]);
    al[2] = pack_lo(p[2 * ks + 1][0], p[2 * ks + 1][1], ah[2]);
    al[3] = pack_lo(p[2 * ks + 1][2], p[2 * ks + 1][3], ah[3]);
#pragma unroll
    for (int np = 0; np < HD / 16; ++np) {
      uint32_t bh[4], bl[4];
      g_load_b_kn(bh, y_tile, 16 * np, 16 * ks, G::SH, lane);
      g_load_b_kn(bl, y_tile + kLo, 16 * np, 16 * ks, G::SH, lane);
      DSVG_MMA3(o[2 * np], ah, al, bh, bl, 0, 1);
      DSVG_MMA3(o[2 * np + 1], ah, al, bh, bl, 2, 3);
    }
  }
}
template <int HD, int NT>
__device__ __forceinline__ void gx3_mul_t(float (&o)[HD / 8][4], uint32_t z_tile, uint32_t y_tile, int w, int lane) {
  using G = GAttn<HD, NT>;
  constexpr uint32_t kLoH = G::kTileH * 2, kLoP = G::kTileP * 2;
#pragma unroll
  for (int nt = 0; nt < HD / 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < NT; ++ks) {
    uint32_t ah[4], al[4];
    g_load_a_t(ah, z_tile, 16 * w, 16 * ks, G::SP, lane);
    g_load_a_t(al, z_tile + kLoP, 16 * w, 16 * ks, G::SP, lane);
#pragma unroll
    for (int np = 0; np < HD / 16; ++np) {
      uint32_t bh[4], bl[4];
      g_load_b_kn(bh, y_tile, 16 * np, 16 * ks, G::SH, lane);
      g_load_b_kn(bl, y_tile + kLoH, 16 * np, 16 * ks, G::SH, lane);
      DSVG_MMA3(o[2 * np], ah, al, bh, bl, 0, 1);
      DSVG_MMA3(o[2 * np + 1], ah, al, bh, bl, 2, 3);
    }
  }
}
template <int HD>
__device__ __forceinline__ void gx3_store_global(bf16* dst, size_t lo_off, int ld, int L, int row0, const float (&c)[HD / 8][4],
                                                 float mul, int g, int t) {
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int i = row0 + g + 8 * hrow;
    if (i < L) {
#pragma unroll
      for (int nt = 0; nt < HD / 8; ++nt) {
        const float x = c[nt][2 * hrow] * mul, y = c[nt][2 * hrow + 1] * mul;
        const uint32_t hi = pack_bf16(x, y);
        bf16* p = dst + size_t(i) * ld + 8 * nt + 2 * t;
        *reinterpret_cast<uint32_t*>(p) = hi;
        *reinterpret_cast<uint32_t*>(p + lo_off) = pack_lo(x, y, hi);
      }
    }
  }
}
template <int NT>
__device__ __forceinline__ void gx3_store_rows_smem(bf16* tile, int lo_elems, int st, int row0, const float (&c)[2 * NT][4],
                                                    int g, int t) {
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int i = row0 + g + 8 * hrow;
#pragma unroll
    for (int nt = 0; nt < 2 * NT; ++nt) {
      const uint32_t hi = pack_bf16(c[nt][2 * hrow], c[nt][2 * hrow + 1]);
      bf16* p = tile + i * st + 8 * nt + 2 * t;
      *reinterpret_cast<uint32_t*>(p) = hi;
      *reinterpret_cast<uint32_t*>(p + lo_elems) = pack_lo(c[nt][2 * hrow], c[nt][2 * hrow + 1], hi);
    }
  }
}

template <int HD, int NT>
__global__ void __launch_bounds__(32 * NT) attn_gx3_fwd_kernel(X3AttnArgs x) {
  using G = GAttn<HD, NT>;
  pdl_launch_dependents();
  pdl_wait();
  MmaAttnArgs& a = x.m;
  drop_resolve(a.drop);
  extern __shared__ __align__(16) bf16 sm_dyn[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, d = a.H * HD, ld = 3 * d;
  bf16* Qs = sm_dyn;                   // hi, lo
  bf16* Ks = Qs + 2 * G::kTileH;
  bf16* Vs = Ks + 2 * G::kTileH;
  uint8_t* kv = reinterpret_cast<uint8_t*>(Vs + 2 * G::kTileH);
  const uint32_t q_t = smem_addr(Qs), k_t = smem_addr(Ks), v_t = smem_addr(Vs);
  const long long npairs = (long long)a.nseq * a.H;
  for (long long pair = blockIdx.x; pair < npairs; pair += gridDim.x) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    const bf16* base = a.qkv + row0 * ld + h * HD;
#pragma unroll
    for (int pl = 0; pl < 2; ++pl) {
      const bf16* b = base + (pl ? x.qkv_lo : 0);
      g_stage<HD, NT>(Qs + pl * G::kTileH, b, ld, L);
      g_stage<HD, NT>(Ks + pl * G::kTileH, b + d, ld, L);
      g_stage<HD, NT>(Vs + pl * G::kTileH, b + 2 * d, ld, L);
    }
    cp_async_commit();
    for (int j = threadIdx.x; j < G::LP; j += G::kThreads) kv[j] = (j < L && (a.valid == nullptr || a.valid[row0 + j] != 0)) ? 1 : 0;
    cp_async_wait_all();
    __syncthreads();
    float s[2 * NT][4];
    gx3_scores<HD, NT>(s, q_t, k_t, w, lane);
    g_softmax<NT>(s, g_my_keys<NT>(kv, t), 16 * w, g, t, a.causal);
    if (a.drop.p > 0.f) {
      float mult[2 * NT][4];
      g_dropout<NT>(mult, a.drop, (unsigned long long)pair, w, g, t);
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[nt][e] *= mult[nt][e];
    }
    float o[HD / 8][4];
    gx3_mul_regs<HD, NT>(o, s, v_t, lane);
    gx3_store_global<HD>(a.out + row0 * d + h * HD, x.out_lo, d, L, 16 * w, o, 1.f, g, t);
    __syncthreads();
  }
}

template <int HD, int NT>
__global__ void __launch_bounds__(32 * NT) attn_gx3_bwd_kernel(X3AttnArgs x) {
  using G = GAttn<HD, NT>;
  pdl_launch_dependents();
  pdl_wait();
  MmaAttnArgs& a = x.m;
  drop_resolve(a.drop);
  extern __shared__ __align__(16) bf16 sm_dyn[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, d = a.H * HD, ld = 3 * d;
  bf16* Qs = sm_dyn;
  bf16* Ks = Qs + 2 * G::kTileH;
  bf16* Vs = Ks + 2 * G::kTileH;
  bf16* Gs = Vs + 2 * G::kTileH;   // dO
  bf16* Ps = Gs + 2 * G::kTileH;   // dropout-scaled probabilities  [query][key], hi then lo
  bf16* Ds = Ps + 2 * G::kTileP;   // dS
  uint8_t* kv = reinterpret_cast<uint8_t*>(Ds + 2 * G::kTileP);
  const uint32_t q_t = smem_addr(Qs), k_t = smem_addr(Ks), v_t = smem_addr(Vs), g_t = smem_addr(Gs), p_t = smem_addr(Ps),
                 d_t = smem_addr(Ds);
  const long long npairs = (long long)a.nseq * a.H;
  for (long long pair = blockIdx.x; pair < npairs; pair += gridDim.x) {
    const int seq = int(pair / a.H), h = int(pair % a.H);
    const size_t row0 = size_t(seq) * L;
    const bf16* base = a.qkv + row0 * ld + h * HD;
    const bf16* gbase = a.dout + row0 * d + h * HD;
#pragma unroll
    for (int pl = 0; pl < 2; ++pl) {
      const bf16* b = base + (pl ? x.qkv_lo : 0);
      g_stage<HD, NT>(Qs + pl * G::kTileH, b, ld, L);
      g_stage<HD, NT>(Ks + pl * G::kTileH, b + d, ld, L);
      g_stage<HD, NT>(Vs + pl * G::kTileH, b + 2 * d, ld, L);
      g_stage<HD, NT>(Gs + pl * G::kTileH, gbase + (pl ? x.dout_lo : 0), d, L);
    }
    cp_async_commit();
    for (int j = threadIdx.x; j < G::LP; j += G::kThreads) kv[j] = (j < L && (a.valid == nullptr || a.valid[row0 + j] != 0)) ? 1 : 0;
    cp_async_wait_all();
    __syncthreads();
    float p[2 * NT][4], dp[2 * NT][4];
    gx3_scores<HD, NT>(p, q_t, k_t, w, lane);
    g_softmax<NT>(p, g_my_keys<NT>(kv, t), 16 * w, g, t, a.causal);
    gx3_scores<HD, NT>(dp, g_t, v_t, w, lane);          // dP = dO . V^T
    if (a.drop.p > 0.f) {
      float mult[2 * NT][4];
      g_dropout<NT>(mult, a.drop, (unsigned long long)pair, w, g, t);
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          dp[nt][e] *= mult[nt][e];
          mult[nt][e] *= p[nt][e];
        }
      gx3_store_rows_smem<NT>(Ps, G::kTileP, G::SP, 16 * w, mult, g, t);
    } else {
      gx3_store_rows_smem<NT>(Ps, G::kTileP, G::SP, 16 * w, p, g, t);
    }
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      float delta = 0.f;
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) delta = fmaf(dp[nt][2 * hrow + e], p[nt][2 * hrow + e], delta);
      delta += __shfl_xor_sync(0xffffffffu, delta, 1);
      delta += __shfl_xor_sync(0xffffffffu, delta, 2);
#pragma unroll
      for (int nt = 0; nt < 2 * NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) dp[nt][2 * hrow + e] = p[nt][2 * hrow + e] * (dp[nt][2 * hrow + e] - delta);
    }
    gx3_store_rows_smem<NT>(Ds, G::kTileP, G::SP, 16 * w, dp, g, t);
    float o[HD / 8][4];
    bf16* dbase = a.dqkv + row0 * ld + h * HD;
    gx3_mul_regs<HD, NT>(o, dp, k_t, lane);                 // dQ rows of this warp = dS_w . K
    gx3_store_global<HD>(dbase, x.dqkv_lo, ld, L, 16 * w, o, a.scale, g, t);
    __syncthreads();                                        // every warp's rows of P and dS are in shared memory
    gx3_mul_t<HD, NT>(o, d_t, q_t, w, lane);                // dK rows [16 w, +16) = dS^T . Q
    gx3_store_global<HD>(dbase + d, x.dqkv_lo, ld, L, 16 * w, o, 1.f, g, t);
    gx3_mul_t<HD, NT>(o, p_t, g_t, w, lane);                // dV rows = dropout(P)^T . dO
    gx3_store_global<HD>(dbase + 2 * d, x.dqkv_lo, ld, L, 16 * w, o, 1.f, g, t);
    __syncthreads();
  }
}

template <int HD, int NT, bool BWD>
static int launch_gx3_k(const X3AttnArgs& x, cudaStream_t st) {
  using G = GAttn<HD, NT>;
  const int smem = BWD ? GX3<HD, NT>::kSmemBwd : GX3<HD, NT>::kSmemFwd;
  auto kern = [] {
    if constexpr (BWD) return attn_gx3_bwd_kernel<HD, NT>;
    else return attn_gx3_fwd_kernel<HD, NT>;
  }();
  static int per_sm = 0;
  static bool configured[kMaxDevices] = {};
  if (first_use_on_device(configured)) {
    DSVG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int n = 0;
    DSVG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, G::kThreads, size_t(smem)));
    per_sm = n > 0 ? n : 1;
  }
  int sms = 132;
  {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  const long long npairs = (long long)x.m.nseq * x.m.H;
  long long blocks = (long long)sms * per_sm;
  if (blocks > npairs) blocks = npairs;
  DSVG_CUDA(launch_k(kern, dim3(int(blocks)), dim3(G::kThreads), size_t(smem), st, x));
  ++g_launches;
  return 0;
}
template <int HD>
static int launch_gx3_nt(bool bwd, const X3AttnArgs& x, cudaStream_t st) {
#define DSVG_GX3_CASE(NT) \
  case NT: return bwd ? launch_gx3_k<HD, NT, true>(x, st) : launch_gx3_k<HD, NT, false>(x, st)
  switch ((x.m.L + 15) / 16) {
    DSVG_GX3_CASE(1);
    DSVG_GX3_CASE(2);
    DSVG_GX3_CASE(3);
    DSVG_GX3_CASE(4);
    DSVG_GX3_CASE(5);
    default: DSVG_CHECK(false, "tensor-core attention: L = %d exceeds 80 positions", x.m.L);
  }
#undef DSVG_GX3_CASE
}

}  // namespace dsvg

// head_dim 32 / 64, L <= 80, single-plane operands
int dsvg_attn_gmma(bool bwd, const bf16* qkv, const uint8_t* valid, bf16* out, const bf16* dout, bf16* dqkv, int nseq, int L,
                   int H, int head_dim, float q_scale, Dropout drop, int causal, cudaStream_t st) {
  MmaAttnArgs a{};
  a.qkv = qkv; a.valid = valid; a.out = out; a.dout = dout; a.dqkv = dqkv; a.nseq = nseq; a.L = L; a.H = H;
  a.scale = q_scale; a.drop = drop; a.causal = causal;
  if (head_dim == 32) return launch_gmma_nt<32>(bwd, a, st);
  if (head_dim == 64) return launch_gmma_nt<64>(bwd, a, st);
  DSVG_CHECK(false, "tensor-core attention: head_dim %d unsupported", head_dim);
}

// head_dim 32 / 64, L <= 80, two-plane (bf16x3) operands
int dsvg_attn_gx3(bool bwd, const bf16* qkv, size_t qkv_lo, const uint8_t* valid, bf16* out, size_t out_lo, const bf16* dout,
                  size_t dout_lo, bf16* dqkv, size_t dqkv_lo, int nseq, int L, int H, int head_dim, float q_scale, Dropout drop,
                  int causal, cudaStream_t st) {
  X3AttnArgs x{};
  MmaAttnArgs& a = x.m;
  a.qkv = qkv; a.valid = valid; a.out = out; a.dout = dout; a.dqkv = dqkv; a.nseq = nseq; a.L = L; a.H = H;
  a.scale = q_scale; a.drop = drop; a.causal = causal;
  x.qkv_lo = qkv_lo; x.out_lo = out_lo; x.dout_lo = dout_lo; x.dqkv_lo = dqkv_lo;
  if (head_dim == 32) return launch_gx3_nt<32>(bwd, x, st);
  if (head_dim == 64) return launch_gx3_nt<64>(bwd, x, st);
  DSVG_CHECK(false, "tensor-core attention: head_dim %d unsupported", head_dim);
}
