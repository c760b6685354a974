/*
 * dsvg_b200.h -- C ABI of libdsvg_b200.so: the sm_90a kernels behind deepsvg_b200.SVGTransformer / SVGLoss.
 *
 * The reference (alexandre01/deepsvg) has NO native/FFI interface: its hot path is Python calling ATen.  Each entry
 * point below therefore names the reference Python call site(s) (file:line under the reference repo) whose
 * arithmetic it replaces.  Conventions (SURVEY.md 8b):
 *   - plain C types only; every pointer is a CUDA device pointer unless the name ends in _host;
 *   - the caller (PyTorch) owns every buffer; the library never allocates user-visible memory, never
 *     synchronises the device, and launches on the `stream` argument (a cudaStream_t passed as void*);
 *   - return value 0 = success; anything else = failure with a message available from dsvg_last_error()
 *     (thread-local); no C++ exception crosses this boundary;
 *   - "act" tensors are bf16 with an optional second "lo" plane `lo_off` ELEMENTS after the first
 *     (lo_off = 0: fast single-plane bf16; lo_off != 0: parity mode, value = hi + lo, GEMMs run as bf16x3);
 *   - dropout masks come from a stateless counter hash keyed by (seed, site, element index); p = 0 disables it
 *     (eval mode); the backward pass regenerates the forward mask from the same triple.  If bit 31 of `drop_site`
 *     (DSVG_SEED_IS_DEVICE_PTR) is set, `seed` is not the seed itself but a DEVICE POINTER to a uint64 holding it, read by
 *     the kernel at run time: a captured CUDA graph then draws fresh masks on every replay (the caller rewrites the
 *     uint64 between replays).
 */
#ifndef DSVG_B200_H
#define DSVG_B200_H

#include <stddef.h>
#define DSVG_SEED_IS_DEVICE_PTR 0x80000000u
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint16_t dsvg_bf16; /* raw bfloat16 bits */

/* ---- library --------------------------------------------------------------------------------------- */
const char* dsvg_last_error(void);
int dsvg_abi_version(void);
/* number of kernels this library has launched since load (per process); bench.py reports it as gpu_launches */
unsigned long long dsvg_launch_count(void);

/* ---- dense contractions on the tensor cores (wgmma) -------------------------------------------------- */
/* Fused epilogue of dsvg_linear, applied to the fp32 accumulator in this order:
 *   v = acc * (*acc_scale_dev); v += bias[col]; if (col < scale_cols) v *= scale; if (relu) v = max(v,0);
 *   v *= dropout(p, seed, site, idx = row*N+col); v += rowvec[(row / rows_per_group)*rowvec_ld + col];
 *   v *= (mask[row*mask_ld+col] != 0) ? mask_scale : 0;  v += residual[row*res_ld+col];
 *   out_f32[row*out_f32_ld+col] = v;  out_act[row*out_act_ld+col] = v (hi[/lo] bf16).
 * NULL pointers skip their step. */
typedef struct dsvg_epilogue {
  const float* acc_scale_dev; /* optional DEVICE scalar (upstream autograd gradient x loss weight) */
  const float* bias;
  int scale_cols;
  float scale;
  int relu;
  float drop_p;
  uint32_t drop_site;
  uint64_t seed;
  const float* rowvec;
  int rowvec_ld;
  int rows_per_group;
  const dsvg_bf16* mask;
  size_t mask_lo_off;
  int mask_ld;
  float mask_scale;
  const float* residual;
  int res_ld;
  float* out_f32;
  int out_f32_ld;
  dsvg_bf16* out_act;
  size_t out_lo_off;
  int out_act_ld;
} dsvg_epilogue;

/* Y[M,N] = epilogue(X[M,K] . W[N,K]^T).  X, W row-major bf16 act tensors (K contiguous; lda/ldb in elements,
 * multiples of 8).  Replaces every F.linear on the path: functional.py:92,249 (QKV / out-proj),
 * improved_transformer.py:52,131,139 (FFN, linear_global), basic_blocks.py:18-21,36-37,60-63 (heads, ResNet),
 * model.py:50,182-183,197 (embed_fcn, VAE/bottleneck) -- and, with W^T, their input gradients. */
int dsvg_linear(const dsvg_bf16* X, size_t x_lo_off, int lda, const dsvg_bf16* W, size_t w_lo_off, int ldb, int M,
                int N, int K, const dsvg_epilogue* ep, void* stream);

/* C[P,Q] += alpha * (*alpha_dev) * A[M,P]^T . B[M,Q]   (contraction over the M rows; A, B row-major act tensors;
 * alpha_dev optional DEVICE scalar).  fp32 atomic adds into C (the M range is split across CTAs), so C is the
 * gradient accumulator itself.  colsum_out (optional, [P]) += alpha * column sums of A, computed by one extra
 * [128 x 64] MMA against an all-ones operand: weight AND bias gradient of every F.linear above from one pass over
 * dY (autograd of the reference, loss.backward() at train.py:98). */
int dsvg_outer(const dsvg_bf16* A, size_t a_lo_off, int lda, const dsvg_bf16* B, size_t b_lo_off, int ldb, int M,
               int P, int Q, float alpha, const float* alpha_dev, float* C, int ldc, float* colsum_out, void* stream);

/* Several weight gradients with the SAME row count M in one launch (single-plane operands, path-level row counts): the four
 * Linear layers of one transformer block (in_proj, out_proj, linear1, linear2: improved_transformer.py:43-53, gradients taken by
 * loss.backward() at train.py:98).  Semantics per problem as dsvg_outer; the problems share one wave of CTAs, so the M range is
 * split ~4x less finely than when each is launched alone (less fp32 atomic traffic, longer streaming loops per CTA). */
typedef struct dsvg_outer_problem {
  const dsvg_bf16* A; /* [M, P], row stride lda */
  int lda;
  const dsvg_bf16* B; /* [M, Q], row stride ldb */
  int ldb;
  int P, Q;
  float alpha;
  const float* alpha_dev; /* optional device scalar */
  float* C;               /* [P, Q] fp32 accumulator, row stride ldc */
  int ldc;
  float* colsum_out;      /* optional [P] */
} dsvg_outer_problem;
int dsvg_outer_group(int n_problems, const dsvg_outer_problem* problems, int M, void* stream);

/* GEMM + LayerNorm in one kernel (fast mode).  When the CTA tile of dsvg_linear owns whole rows (N = d_model = 256,
 * path-level row counts, single-plane operands: ask dsvg_linear_ln_fusable) the LayerNorm that follows a residual-stream
 * linear runs in that GEMM's epilogue: the fp32 residual stream is not re-read by a separate kernel.
 *   (improved_transformer.py:43-44 -> :51, :52-53 -> next layer's :43 / transformer.py:185-186):
 *       x1 = epilogue `e` (bias, dropout, row vector, residual -> e->out_f32 [M,256], row stride e->out_f32_ld)
 *       y  = bf16(LayerNorm(x1) * gamma + beta) [M,256];  mean[M], rstd[M] saved for the backward
 * Results equal dsvg_linear followed by dsvg_ln_fwd (tests/test_kernels_gpu.py). */
int dsvg_linear_ln_fusable(int M, int N, int n_planes);
int dsvg_linear_ln_fwd(const dsvg_bf16* X, size_t x_lo_off, int lda, const dsvg_bf16* W, size_t w_lo_off, int ldb, int M,
                       int N, int K, const dsvg_epilogue* e, const float* gamma, const float* beta, dsvg_bf16* y,
                       float* mean, float* rstd, void* stream);

/* ---- input side: packed batch format (SURVEY.md 8f rank 3) --------------------------------------------- */
/* HOST function.  Assembles one batch the way SVGTensorDataset.get_data does per icon (svgtensor_dataset.py:164-205 with
 * SVGTensor.add_eos / add_sos / pad, difflib/tensor.py:108-143) followed by the default collate, directly into the packed
 * format: cmd_out uint8 [n_icons, G, seq_len+2], args_out int16 [n_icons, G, seq_len+2, 11] (PAD = -1).
 * rows: the icons' raw (len, 14) path tensors concatenated (14 columns: cmd, rx, ry, phi, fA, fS, x0, y0, c1x, c1y, c2x, c2y,
 * x, y -- difflib/tensor.py:23-32); group_offsets [n_icons*max_groups + 1]: row offset of every path (missing paths are
 * empty ranges).  grouped = 0: the per-path tensors (`commands` / `args`, G = max_groups, seq_len = MAX_SEQ_LEN);
 * grouped = 1: the `_grouped` variants (G = 1, all paths of an icon concatenated, seq_len = MAX_TOTAL_LEN).
 * Fails (non-zero) where the reference's torch.stack would: a sequence that does not fit the window. */
int dsvg_pack_icons(const float* rows, const long long* group_offsets, int n_icons, int max_groups, int seq_len, int grouped,
                    unsigned char* cmd_out, short* args_out);
/* Device: packed batch -> the float32 tensors the forward consumes (commands [n_positions], args [n_positions, n_args]). */
int dsvg_unpack_batch(const unsigned char* cmd, const short* args, float* commands_f32, float* args_f32, size_t n_positions,
                      int n_args, void* stream);

/* ---- Hungarian self-matching (cfg.self_match; SURVEY.md 8f rank 4) -------------------------------------- */
/* SVGTransformer.perfect_matching, model.py:311-350, without the host round trip: cost[N, G, Gp] (fp64) = 2 * masked-mean
 * CE_args + masked-mean CE_cmd + CE_visibility between target path g (the SHIFTED targets commands[..., 1:], args[..., 1:, :],
 * read from the unshifted commands [N*G, L] / args [N*G, L, n_args]) and predicted slot p; visible[N*G]; then one thread per
 * icon solves the assignment over its visible targets (replacing scipy.optimize.linear_sum_assignment, model.py:344) and
 * writes assignment[N, Gp] exactly as the reference lists it: slot of the i-th visible target, then the unused slots in
 * ascending order.  lse_cmd [N*Gp*(L-1)], lse_args [N*Gp*(L-1)*n_args] are scratch. */
int dsvg_match_assign(const float* cmd_logits, int n_cmd, const float* args_logits, int ld_args, int n_args, int n_classes,
                      const float* vis_logits, const float* commands, const float* args, int N, int G, int Gp, int L,
                      float* lse_cmd, float* lse_args, double* cost, unsigned char* visible, long long* assignment,
                      void* stream);
/* torch.gather along the slot axis (model.py:389-391) as a group-granular copy: dst group (n, i) = src group
 * (n, assignment[n, i]); inverse != 0 scatters instead (the backward of the gather).  A group is group_bytes contiguous
 * bytes (multiple of 4): L * row bytes of one slot's tokens. */
int dsvg_permute_groups(const void* src, void* dst, const long long* assignment, int N, int G, size_t group_bytes,
                        int inverse, void* stream);

/* ---- sequence bookkeeping (model/utils.py:7-66) ------------------------------------------------------ */
/* From commands[nseq, L] (ids stored as float): first_eos[nseq], visible[nseq] (#EOS < L-1), key_valid[nseq*L]
 * (1 before the first EOS), grp[nseq*L] (# of "m" so far), counts[2] += {loss_cmd positions, loss_args slots}.
 * Any output pointer may be NULL. */
int dsvg_seq_prep(const float* commands, int nseq, int L, int* first_eos, uint8_t* visible, uint8_t* key_valid,
                  uint8_t* grp, float* counts, void* stream);

/* ---- embeddings (model.py:46-57, 70-73; positional_encoding.py:40-43) -------------------------------- */
/* table[k*V+v] = arg_embed[v] . W[:, 64k:64k+64]^T, stored as differences to row v=0 (v>=1); base = bias + sum_k row0 */
int dsvg_embed_fold(const float* arg_embed, const float* W, const float* bias, float* table, float* base, int V,
                    int n_args, int d, void* stream);
/* x[t] = dropout(base + cmd_tab[cmd] + pos_tab[t % L] (+ grp_tab[grp[t]]) + sum_{k: arg_k != -1} table[k*V+arg_k+1]) */
int dsvg_embed_fwd(const float* commands, const float* args, const uint8_t* grp, const float* cmd_tab,
                   const float* table, const float* base, const float* pos_tab, const float* grp_tab, float* x, int T,
                   int L, int V, int n_args, int d, float drop_p, uint32_t drop_site, uint64_t seed, void* stream);
/* all embedding-parameter gradients from dx (accumulating); scratch_table: n_args*V*d floats of workspace */
int dsvg_embed_bwd(const float* commands, const float* args, const uint8_t* grp, const float* dx,
                   const float* arg_embed, const float* W, float* d_cmd_tab, float* d_pos_tab, float* d_grp_tab,
                   float* d_arg_embed, float* d_W, float* d_bias, float* scratch_table, int nseq, int L, int V,
                   int n_args, int d, int n_grp, float drop_p, uint32_t drop_site, uint64_t seed, void* stream);
/* x[r] = dropout(add[r] + tab[r % L]) (add may be NULL: ConstEmbedding) and its backward */
int dsvg_rows_embed_fwd(const float* add, const float* tab, float* x, int R, int L, int d, float drop_p,
                        uint32_t drop_site, uint64_t seed, void* stream);
int dsvg_rows_embed_bwd(const float* dx, float* dadd, float* dtab, int nseq, int L, int d, float drop_p,
                        uint32_t drop_site, uint64_t seed, void* stream);

/* ---- LayerNorm (+ masked mean over the sequence: model.py:137,161) ------------------------------------ */
int dsvg_ln_fwd(const float* x, const float* gamma, const float* beta, dsvg_bf16* y, size_t y_lo_off, float* mean,
                float* rstd, int M, int D, void* stream);
int dsvg_ln_pool_fwd(const float* x, const float* gamma, const float* beta, const uint8_t* valid, float* z,
                     float* mean, float* rstd, float* inv_cnt, int nseq, int L, int D, void* stream);
/* dy from an act tensor, or (dz != NULL) dy[r] = dz[r / L] * valid[r] * inv_cnt[r / L].  dx_out = dx_in + LN'(dy);
 * dact = dropout_mask * dx_out as act; dgamma/dbeta accumulate. */
int dsvg_ln_bwd(const float* x, const float* mean, const float* rstd, const float* gamma, const dsvg_bf16* dy,
                size_t dy_lo_off, const float* dz, const uint8_t* valid, const float* inv_cnt, int L,
                const float* dx_in, float* dx_out, dsvg_bf16* dact, size_t dact_lo_off, float drop_p,
                uint32_t drop_site, uint64_t seed, float* dgamma, float* dbeta, int M, int D, void* stream);

/* ---- self-attention over short sequences (functional.py:168-248) --------------------------------------
 * key_valid (optional, [nseq*L]): key_padding_mask (functional.py:235-240); causal != 0: attn_mask = square_subsequent_mask
 * (query i sees keys j <= i; model/utils.py:69-72, the autoregressive decoder, model.py:269). */
int dsvg_attn_fwd(const dsvg_bf16* qkv, size_t qkv_lo_off, const uint8_t* key_valid, dsvg_bf16* out, size_t out_lo_off,
                  int nseq, int L, int H, int head_dim, int causal, float drop_p, uint32_t drop_site, uint64_t seed,
                  void* stream);
int dsvg_attn_bwd(const dsvg_bf16* qkv, size_t qkv_lo_off, const uint8_t* key_valid, const dsvg_bf16* dout,
                  size_t dout_lo_off, dsvg_bf16* dqkv, size_t dqkv_lo_off, int nseq, int L, int H, int head_dim, int causal,
                  float q_scale, float drop_p, uint32_t drop_site, uint64_t seed, void* stream);

/* ---- incremental autoregressive decoding (SVGTransformer._greedy_sample / greedy_sample, model.py:428-448) --------
 * One new row per sequence per step over per-layer key/value caches.  `step` is a DEVICE int[2]: step[0] = t, the position
 * being decoded, step[1] = 0 (a block ticket); the caller zeroes both before step 0, dsvg_decode_sample advances step[0].
 * Every entry point reads t from there, so one captured CUDA graph of a whole step replays for every t. */
/* SVGEmbedding (model.py:46-57, use_group=True) of the token at position t into x[N, d]: SOS with PAD arguments at t = 0
 * (model.py:428), else cmd_in[N] / args_in[N, n_args].  Same table, base and sum order as dsvg_embed_fwd.  Also carries
 * the bookkeeping of dsvg_seq_prep (model/utils.py:7-17, 35-42) over from t - 1: grp[N] = number of "m" in 0..t,
 * key_valid[n * Tmax + t] = no EOS in 0..t. */
int dsvg_decode_embed(const int* step, const int* cmd_in, const int* args_in, int* grp, uint8_t* key_valid,
                      const float* cmd_tab, const float* table, const float* base, const float* pos_tab, const float* grp_tab,
                      float* x, int N, int Tmax, int V, int n_args, int d, void* stream);
/* Causal self-attention of row t (functional.py:168-248 with square_subsequent_mask and key_padding_mask, model.py:269):
 * appends K and V of qkv[N, 3d] (q pre-scaled) to k_cache / v_cache [N, H, Tmax, head_dim] at position t (every plane;
 * the lo plane cache_lo_off elements after the first), then out[N, d] = softmax(q K^T over valid keys 0..t) V in fp32.
 * qkv, the caches and out have one plane each or two each.  Tmax <= 256. */
int dsvg_decode_attn(const int* step, const dsvg_bf16* qkv, size_t qkv_lo_off, dsvg_bf16* k_cache, dsvg_bf16* v_cache,
                     size_t cache_lo_off, const uint8_t* key_valid, dsvg_bf16* out, size_t out_lo_off, int N, int H,
                     int head_dim, int Tmax, void* stream);
/* Token choice of step t (model.py:415-418 pick() + _make_valid, :450-459): *temperature < 1e-3 takes the argmax of the
 * n_cmd command logits and of each argument slot's n_classes logits (ties to the lowest index); otherwise Gumbel-max with
 * noise from a counter hash of (*seed, t, sequence, slot, class).  Argument slots CMD_ARGS_MASK marks unused become -1,
 * the others class - 1.  Writes out_cmd[n * Tmax + t], out_args[(n * Tmax + t) * n_args + k] and the next step's
 * cmd_in / args_in, then step[0] = t + 1. */
int dsvg_decode_sample(int* step, const float* cmd_logits, int ld_cmd, const float* args_logits, int ld_args,
                       const float* temperature, const unsigned long long* seed, int* cmd_in, int* args_in, long long* out_cmd,
                       long long* out_args, int N, int Tmax, int n_cmd, int n_args, int n_classes, void* stream);

/* ---- SVGLoss (model/loss.py:19-65): loss sums + unit-scale d(loss)/d(logits) --------------------------- */
int dsvg_ce_args(const float* logits, int ld_logits, const float* commands, const float* args, const float* counts,
                 dsvg_bf16* dlogits, size_t dl_lo_off, int ld_dl, float* acc, int nseq, int L, int n_args,
                 int n_classes, void* stream);
int dsvg_ce_cmd(const float* logits, const float* commands, const int* first_eos, const uint8_t* visible,
                const float* counts, dsvg_bf16* dlogits, size_t dl_lo_off, int ld_dl, float* acc, int nseq, int L,
                int n_classes, void* stream);
int dsvg_ce_vis(const float* logits, const uint8_t* visible, dsvg_bf16* dlogits, size_t dl_lo_off, int ld_dl,
                float* acc, int nseq, float inv_total, void* stream);
int dsvg_kl_sum(const float* mu, const float* logsigma, float* acc, int n, void* stream);
/* out[0..4] = loss, loss_cmd, loss_args, loss_visibility, loss_kl; out[5] = 1 if the KL clamp passes gradient */
int dsvg_loss_finalize(const float* acc, const float* counts, float* out, float w_cmd, float w_args, float w_vis,
                       float w_kl, float kl_tolerance, float inv_vis_total, float inv_kl_total, int has_vis,
                       int has_kl, void* stream);
/* VAE reparameterisation (model.py:182-187) */
int dsvg_vae_fwd(const float* mu, const float* logsigma, const float* eps, float* z, int n, void* stream);
int dsvg_vae_bwd(const float* mu, const float* logsigma, const float* eps, const float* dz, const float* kl_coef_dev,
                 const float* loss_out, float inv_total, float* dmu, float* dls, int n, void* stream);

/* ---- helpers -------------------------------------------------------------------------------------------- */
/* fp32 -> act cast (optional transposed copy, optional (mask != 0) * mask_scale, optional dropout) */
int dsvg_cast_act(const float* in, int ld_in, int R, int C, dsvg_bf16* out, size_t out_lo_off, int ld_out,
                  dsvg_bf16* outT, size_t outT_lo_off, int ld_t, const dsvg_bf16* mask, size_t mask_lo_off,
                  int ld_mask, float mask_scale, float drop_p, uint32_t drop_site, uint64_t seed, void* stream);
/* dst[c] += (*alpha_dev) * sum_r a[r, c]  (bias gradients) */
int dsvg_colsum(const dsvg_bf16* a, size_t lo_off, int ld, int M, int N, const float* alpha_dev, float* dst,
                void* stream);
/* out[q] = dropout(sum_{s<L} in[q*L+s])  (backward of the linear_global broadcast, improved_transformer.py:131-136) */
int dsvg_seg_sum(const float* in, int nseq, int L, int d, dsvg_bf16* out, size_t out_lo_off, float* out_f32,
                 float drop_p, uint32_t drop_site, uint64_t seed, void* stream);
/* LabelEmbedding (model.py:87-89) gather and its gradient scatter-add; table / dtable have n_rows rows of w floats.  An id
 * outside [0, n_rows) traps on the device (the launch fails), like nn.Embedding's device-side assert. */
int dsvg_gather_rows(const float* table, const long long* idx, int n, int w, int n_rows, dsvg_bf16* out, size_t out_lo_off,
                     void* stream);
int dsvg_scatter_rows(const float* g, const long long* idx, int n, int w, int n_rows, float* dtable, void* stream);
int dsvg_add_f32(const float* a, const float* b, float* y, size_t n, void* stream);

/* ---- optimiser step on a table of tensors (SURVEY.md 8f rank 2; config.py:64-65, train.py:99-102) ------------ */
/* table: DEVICE array of n_tensors rows {float* param; const float* grad; float* exp_avg; float* exp_avg_sq;
 * long long numel}.  max_chunks = ceil(max numel / 4096) capped by the caller (grid.x). */
int dsvg_grad_sqnorm(const void* table, int n_tensors, int max_chunks, float* out_sq, void* stream);
/* AdamW (decoupled weight decay), gradients scaled by min(1, max_norm / (sqrt(*grad_sqnorm_dev) + 1e-6)) when max_norm > 0 */
int dsvg_adamw_step(const void* table, int n_tensors, int max_chunks, float lr, float beta1, float beta2, float eps,
                    float weight_decay, float bias_corr1, float bias_corr2, float max_norm, const float* grad_sqnorm_dev,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DSVG_B200_H */
