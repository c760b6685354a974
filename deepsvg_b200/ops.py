"""Thin Python wrappers over the C ABI (include/dsvg_b200.h): pointer marshalling only, no arithmetic.

Every wrapper launches on torch's current CUDA stream and raises RuntimeError on a non-zero return code.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import Epilogue

BF16 = torch.bfloat16


def _stream():
    return torch.cuda.current_stream().cuda_stream


# Optional launch profiler (bench.py): when PROFILE is a list, linear/outer/attention launches are bracketed by CUDA
# events on the launching stream and recorded as (family, algorithmic flops, start event, end event).
PROFILE = None


class _Prof:
    def __init__(self, family, flops, shape=None, nbytes=0.0):
        self.family, self.flops, self.shape, self.nbytes = family, flops, shape, nbytes

    def __enter__(self):
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *a):
        if PROFILE is not None:
            self.e1.record()
            PROFILE.append((self.family, self.flops, self.e0, self.e1, self.shape, self.nbytes))
        return False


def _p(t):
    return 0 if t is None else t.data_ptr()


class Act:
    """A (split-)bf16 activation tensor: `planes` x [rows, ld]; value = plane0 (+ plane1)."""
    __slots__ = ("t", "rows", "cols", "ld", "lo", "planes")

    def __init__(self, rows, cols, planes, device, ld=None, zero=False):
        self.rows, self.cols, self.planes = rows, cols, planes
        self.ld = ld if ld is not None else cols
        alloc = torch.zeros if zero else torch.empty
        self.t = alloc(planes, rows, self.ld, dtype=BF16, device=device)
        self.lo = rows * self.ld if planes == 2 else 0

    @property
    def ptr(self):
        return self.t.data_ptr()

    def float(self):
        """fp32 value (test / debug helper)."""
        v = self.t[0].float()
        if self.planes == 2:
            v = v + self.t[1].float()
        return v[:, :self.cols]


def act_from_float(x, planes, ld=None):
    """host-side helper for tests: fp32 [R, C] -> Act (rounding on the GPU via torch)."""
    R, Cc = x.shape
    a = Act(R, Cc, planes, x.device, ld=ld, zero=True)
    hi = x.to(BF16)
    a.t[0, :, :Cc] = hi
    if planes == 2:
        a.t[1, :, :Cc] = (x - hi.float()).to(BF16)
    return a


def ln_fusable(M, N, planes):
    """True when the GEMM's CTA tile owns whole LayerNorm rows, so that the fused LayerNorm of linear(ln=...) applies."""
    return bool(_lib.load().dsvg_linear_ln_fusable(M, N, planes))


def linear(X, W, M, N, K, *, bias=None, scale_cols=0, scale=1.0, relu=False, drop=(0.0, 0, 0), rowvec=None,
           rows_per_group=1, mask=None, mask_scale=1.0, residual=None, out_f32=None, out_act=None, acc_scale=None,
           ln=None):
    """out = epilogue(X[M,K] . W[N,K]^T); X, W are Act.
    ln = (gamma, beta, y Act, mean, rstd): additionally y = LayerNorm(out_f32) in the same kernel (needs ln_fusable)."""
    ep = Epilogue()
    ep.acc_scale_dev = _p(acc_scale)
    ep.bias = _p(bias)
    ep.scale_cols, ep.scale, ep.relu = scale_cols, scale, 1 if relu else 0
    ep.drop_p, ep.drop_site, ep.seed = drop
    if rowvec is not None:
        ep.rowvec, ep.rowvec_ld, ep.rows_per_group = rowvec.data_ptr(), rowvec.stride(0), rows_per_group
    if mask is not None:
        ep.mask, ep.mask_lo_off, ep.mask_ld, ep.mask_scale = mask.ptr, mask.lo, mask.ld, mask_scale
    if residual is not None:
        ep.residual, ep.res_ld = residual.data_ptr(), residual.stride(0)
    if out_f32 is not None:
        ep.out_f32, ep.out_f32_ld = out_f32.data_ptr(), out_f32.stride(0)
    if out_act is not None:
        ep.out_act, ep.out_lo_off, ep.out_act_ld = out_act.ptr, out_act.lo, out_act.ld
    # algorithmic HBM bytes of this launch (operands read once, outputs written once)
    nb = 2.0 * X.planes * M * K + 2.0 * W.planes * N * K
    nb += (4.0 * M * N if residual is not None else 0) + (2.0 * M * N if mask is not None else 0)
    nb += (4.0 * M * N if out_f32 is not None else 0) + (2.0 * out_act.planes * M * N if out_act is not None else 0)
    if ln is not None:
        gamma, beta, y, mean, rstd = ln
        nb += 2.0 * y.planes * M * N + 8.0 * M
        with _Prof("linear", 2.0 * M * N * K, (M, N, K), nb):
            rc = _lib.load().dsvg_linear_ln_fwd(X.ptr, X.lo, X.ld, W.ptr, W.lo, W.ld, M, N, K, C.byref(ep), gamma.data_ptr(),
                                                beta.data_ptr(), y.ptr, mean.data_ptr(), rstd.data_ptr(), _stream())
        _lib.check(rc, "dsvg_linear_ln_fwd")
        return
    with _Prof("linear", 2.0 * M * N * K, (M, N, K), nb):
        rc = _lib.load().dsvg_linear(X.ptr, X.lo, X.ld, W.ptr, W.lo, W.ld, M, N, K, C.byref(ep), _stream())
    _lib.check(rc, "dsvg_linear")


def outer(A, B, M, P, Q, Cout, *, alpha=1.0, alpha_dev=None, colsum=None):
    """Cout[P,Q] += alpha * A[M,P]^T . B[M,Q]; Cout fp32 (row stride = Cout.stride(0)); colsum[P] += alpha * sum_rows A."""
    with _Prof("outer", 2.0 * M * P * Q, (M, P, Q), 2.0 * A.planes * M * P + 2.0 * B.planes * M * Q + 4.0 * P * Q):
        rc = _lib.load().dsvg_outer(A.ptr, A.lo, A.ld, B.ptr, B.lo, B.ld, M, P, Q, alpha, _p(alpha_dev),
                                    Cout.data_ptr(), Cout.stride(0), _p(colsum), _stream())
    _lib.check(rc, "dsvg_outer")


def outer_group(problems, M):
    """problems: list of (A, B, P, Q, Cout, colsum) with single-plane Act operands sharing the row count M (the weight gradients
    of one transformer block): Cout += A^T . B and colsum += column sums of A for each, in ONE launch (dsvg_outer_group)."""
    n = len(problems)
    arr = (_lib.OuterProblem * n)()
    flops = nbytes = 0.0
    for i, (A, B, P, Q, Cout, colsum) in enumerate(problems):
        assert A.planes == 1 and B.planes == 1
        arr[i].A, arr[i].lda, arr[i].B, arr[i].ldb = A.ptr, A.ld, B.ptr, B.ld
        arr[i].P, arr[i].Q, arr[i].alpha, arr[i].alpha_dev = P, Q, 1.0, None
        arr[i].C, arr[i].ldc, arr[i].colsum_out = Cout.data_ptr(), Cout.stride(0), _p(colsum) or None
        flops += 2.0 * M * P * Q
        nbytes += 2.0 * M * (P + Q) + 4.0 * P * Q
    with _Prof("outer", flops, None, nbytes):
        rc = _lib.load().dsvg_outer_group(n, C.cast(arr, C.c_void_p), M, _stream())
    _lib.check(rc, "dsvg_outer_group")


def seq_prep(commands, nseq, L, first_eos, visible, key_valid, grp, counts):
    rc = _lib.load().dsvg_seq_prep(commands.data_ptr(), nseq, L, _p(first_eos), _p(visible), _p(key_valid), _p(grp),
                                   _p(counts), _stream())
    _lib.check(rc, "dsvg_seq_prep")


def embed_fold(arg_embed, W, bias, table, base, V, n_args, d):
    rc = _lib.load().dsvg_embed_fold(arg_embed.data_ptr(), W.data_ptr(), bias.data_ptr(), table.data_ptr(),
                                     base.data_ptr(), V, n_args, d, _stream())
    _lib.check(rc, "dsvg_embed_fold")


def embed_fwd(commands, args, grp, cmd_tab, table, base, pos_tab, grp_tab, x, T, L, V, n_args, d, drop):
    rc = _lib.load().dsvg_embed_fwd(commands.data_ptr(), args.data_ptr(), _p(grp), cmd_tab.data_ptr(),
                                    table.data_ptr(), base.data_ptr(), pos_tab.data_ptr(), _p(grp_tab), x.data_ptr(),
                                    T, L, V, n_args, d, drop[0], drop[1], drop[2], _stream())
    _lib.check(rc, "dsvg_embed_fwd")


def embed_bwd(commands, args, grp, dx, arg_embed, W, d_cmd, d_pos, d_grp, d_arg_embed, d_W, d_bias, scratch, nseq, L,
              V, n_args, d, n_grp, drop):
    rc = _lib.load().dsvg_embed_bwd(commands.data_ptr(), args.data_ptr(), _p(grp), dx.data_ptr(),
                                    arg_embed.data_ptr(), W.data_ptr(), d_cmd.data_ptr(), d_pos.data_ptr(),
                                    _p(d_grp), d_arg_embed.data_ptr(), d_W.data_ptr(), d_bias.data_ptr(),
                                    scratch.data_ptr(), nseq, L, V, n_args, d, n_grp, drop[0], drop[1], drop[2],
                                    _stream())
    _lib.check(rc, "dsvg_embed_bwd")


def rows_embed_fwd(add, tab, x, R, L, d, drop):
    rc = _lib.load().dsvg_rows_embed_fwd(_p(add), tab.data_ptr(), x.data_ptr(), R, L, d, drop[0], drop[1], drop[2],
                                         _stream())
    _lib.check(rc, "dsvg_rows_embed_fwd")


def rows_embed_bwd(dx, dadd, dtab, nseq, L, d, drop):
    rc = _lib.load().dsvg_rows_embed_bwd(dx.data_ptr(), _p(dadd), dtab.data_ptr(), nseq, L, d, drop[0], drop[1],
                                         drop[2], _stream())
    _lib.check(rc, "dsvg_rows_embed_bwd")


def ln_fwd(x, gamma, beta, y, mean, rstd, M, D):
    rc = _lib.load().dsvg_ln_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.ptr, y.lo, mean.data_ptr(),
                                 rstd.data_ptr(), M, D, _stream())
    _lib.check(rc, "dsvg_ln_fwd")


def ln_pool_fwd(x, gamma, beta, valid, z, mean, rstd, inv_cnt, nseq, L, D):
    rc = _lib.load().dsvg_ln_pool_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), valid.data_ptr(),
                                      z.data_ptr(), mean.data_ptr(), rstd.data_ptr(), inv_cnt.data_ptr(), nseq, L, D,
                                      _stream())
    _lib.check(rc, "dsvg_ln_pool_fwd")


def ln_bwd(x, mean, rstd, gamma, M, D, *, dy=None, dz=None, valid=None, inv_cnt=None, L=0, dx_in=None, dx_out=None,
           dact=None, drop=(0.0, 0, 0), dgamma=None, dbeta=None):
    rc = _lib.load().dsvg_ln_bwd(x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(),
                                 dy.ptr if dy is not None else 0, dy.lo if dy is not None else 0, _p(dz), _p(valid),
                                 _p(inv_cnt), L, _p(dx_in), _p(dx_out), dact.ptr if dact is not None else 0,
                                 dact.lo if dact is not None else 0, drop[0], drop[1], drop[2], _p(dgamma), _p(dbeta),
                                 M, D, _stream())
    _lib.check(rc, "dsvg_ln_bwd")


def attn_fwd(qkv, key_valid, out, nseq, L, H, hd, drop, causal=False):
    with _Prof("attn_fwd", 4.0 * nseq * L * L * H * hd, None, 2.0 * qkv.planes * nseq * L * H * hd * 4):
        rc = _lib.load().dsvg_attn_fwd(qkv.ptr, qkv.lo, _p(key_valid), out.ptr, out.lo, nseq, L, H, hd, int(causal), drop[0],
                                       drop[1], drop[2], _stream())
    _lib.check(rc, "dsvg_attn_fwd")


def attn_bwd(qkv, key_valid, dout, dqkv, nseq, L, H, hd, q_scale, drop, causal=False):
    with _Prof("attn_bwd", 8.0 * nseq * L * L * H * hd, None, 2.0 * qkv.planes * nseq * L * H * hd * 7):
        rc = _lib.load().dsvg_attn_bwd(qkv.ptr, qkv.lo, _p(key_valid), dout.ptr, dout.lo, dqkv.ptr, dqkv.lo, nseq, L, H,
                                       hd, int(causal), q_scale, drop[0], drop[1], drop[2], _stream())
    _lib.check(rc, "dsvg_attn_bwd")


def decode_embed(step, cmd_in, args_in, grp, key_valid, cmd_tab, table, base, pos_tab, grp_tab, x, N, Tmax, V, n_args, d):
    rc = _lib.load().dsvg_decode_embed(step.data_ptr(), cmd_in.data_ptr(), args_in.data_ptr(), grp.data_ptr(),
                                       key_valid.data_ptr(), cmd_tab.data_ptr(), table.data_ptr(), base.data_ptr(),
                                       pos_tab.data_ptr(), grp_tab.data_ptr(), x.data_ptr(), N, Tmax, V, n_args, d, _stream())
    _lib.check(rc, "dsvg_decode_embed")


def decode_cache(N, H, hd, Tmax, planes, device):
    """One layer's key or value cache: bf16 [planes, N, H, Tmax, hd] (the lo plane after the hi plane)."""
    return torch.empty(planes, N, H, Tmax, hd, dtype=BF16, device=device)


def decode_attn(step, qkv, k_cache, v_cache, key_valid, out, N, H, hd, Tmax):
    """k_cache / v_cache from decode_cache(); qkv, out: Act with the caches' plane count."""
    lo = k_cache[0].numel() if k_cache.shape[0] == 2 else 0
    rc = _lib.load().dsvg_decode_attn(step.data_ptr(), qkv.ptr, qkv.lo, k_cache.data_ptr(), v_cache.data_ptr(), lo,
                                      key_valid.data_ptr(), out.ptr, out.lo, N, H, hd, Tmax, _stream())
    _lib.check(rc, "dsvg_decode_attn")


def decode_sample(step, cmd_logits, args_logits, temperature, seed, cmd_in, args_in, out_cmd, out_args, N, Tmax, n_args,
                  n_classes):
    rc = _lib.load().dsvg_decode_sample(step.data_ptr(), cmd_logits.data_ptr(), cmd_logits.stride(0),
                                        args_logits.data_ptr(), args_logits.stride(0), temperature.data_ptr(),
                                        seed.data_ptr(), cmd_in.data_ptr(), args_in.data_ptr(), out_cmd.data_ptr(),
                                        out_args.data_ptr(), N, Tmax, cmd_logits.shape[1], n_args, n_classes, _stream())
    _lib.check(rc, "dsvg_decode_sample")


def ce_args(logits, ld_logits, commands, args, counts, dl, acc, nseq, L, n_args, n_classes):
    rc = _lib.load().dsvg_ce_args(logits.data_ptr(), ld_logits, commands.data_ptr(), args.data_ptr(),
                                  counts.data_ptr(), dl.ptr, dl.lo, dl.ld, acc.data_ptr(), nseq, L, n_args, n_classes,
                                  _stream())
    _lib.check(rc, "dsvg_ce_args")


def ce_cmd(logits, commands, first_eos, visible, counts, dl, acc, nseq, L, n_classes):
    rc = _lib.load().dsvg_ce_cmd(logits.data_ptr(), commands.data_ptr(), first_eos.data_ptr(), visible.data_ptr(),
                                 counts.data_ptr(), dl.ptr, dl.lo, dl.ld, acc.data_ptr(), nseq, L, n_classes, _stream())
    _lib.check(rc, "dsvg_ce_cmd")


def ce_vis(logits, visible, dl, acc, nseq, inv_total):
    rc = _lib.load().dsvg_ce_vis(logits.data_ptr(), visible.data_ptr(), dl.ptr, dl.lo, dl.ld, acc.data_ptr(), nseq,
                                 inv_total, _stream())
    _lib.check(rc, "dsvg_ce_vis")


def kl_sum(mu, ls, acc, n):
    rc = _lib.load().dsvg_kl_sum(mu.data_ptr(), ls.data_ptr(), acc.data_ptr(), n, _stream())
    _lib.check(rc, "dsvg_kl_sum")


def loss_finalize(acc, counts, out, w_cmd, w_args, w_vis, w_kl, kl_tol, inv_vis_total, inv_kl_total, has_vis, has_kl):
    rc = _lib.load().dsvg_loss_finalize(acc.data_ptr(), counts.data_ptr(), out.data_ptr(), w_cmd, w_args, w_vis, w_kl,
                                        kl_tol, inv_vis_total, inv_kl_total, int(has_vis), int(has_kl), _stream())
    _lib.check(rc, "dsvg_loss_finalize")


def vae_fwd(mu, ls, eps, z, n):
    rc = _lib.load().dsvg_vae_fwd(mu.data_ptr(), ls.data_ptr(), eps.data_ptr(), z.data_ptr(), n, _stream())
    _lib.check(rc, "dsvg_vae_fwd")


def vae_bwd(mu, ls, eps, dz, kl_coef, loss_out, inv_total, dmu, dls, n):
    rc = _lib.load().dsvg_vae_bwd(mu.data_ptr(), ls.data_ptr(), eps.data_ptr(), dz.data_ptr(), _p(kl_coef),
                                  _p(loss_out), inv_total, dmu.data_ptr(), dls.data_ptr(), n, _stream())
    _lib.check(rc, "dsvg_vae_bwd")


def cast_act(x, R, Ccols, *, out=None, outT=None, mask=None, mask_scale=1.0, drop=(0.0, 0, 0)):
    """fp32 x[R, C] (row stride x.stride(0)) -> Act out [R, ld] and/or transposed Act outT [C, ld_t]."""
    rc = _lib.load().dsvg_cast_act(x.data_ptr(), x.stride(0) if x.dim() > 1 else Ccols, R, Ccols,
                                   out.ptr if out is not None else 0, out.lo if out is not None else 0,
                                   out.ld if out is not None else 0,
                                   outT.ptr if outT is not None else 0, outT.lo if outT is not None else 0,
                                   outT.ld if outT is not None else 0,
                                   mask.ptr if mask is not None else 0, mask.lo if mask is not None else 0,
                                   mask.ld if mask is not None else 0, mask_scale, drop[0], drop[1], drop[2],
                                   _stream())
    _lib.check(rc, "dsvg_cast_act")


def colsum(a, M, N, dst, alpha_dev=None):
    rc = _lib.load().dsvg_colsum(a.ptr, a.lo, a.ld, M, N, _p(alpha_dev), dst.data_ptr(), _stream())
    _lib.check(rc, "dsvg_colsum")


def seg_sum(x, nseq, L, d, *, out=None, out_f32=None, drop=(0.0, 0, 0)):
    rc = _lib.load().dsvg_seg_sum(x.data_ptr(), nseq, L, d, out.ptr if out is not None else 0,
                                  out.lo if out is not None else 0, _p(out_f32), drop[0], drop[1], drop[2], _stream())
    _lib.check(rc, "dsvg_seg_sum")


def gather_rows(table, idx, n, w, out):
    rc = _lib.load().dsvg_gather_rows(table.data_ptr(), idx.data_ptr(), n, w, table.shape[0], out.ptr, out.lo, _stream())
    _lib.check(rc, "dsvg_gather_rows")


def scatter_rows(g, idx, n, w, dtable):
    rc = _lib.load().dsvg_scatter_rows(g.data_ptr(), idx.data_ptr(), n, w, dtable.shape[0], dtable.data_ptr(), _stream())
    _lib.check(rc, "dsvg_scatter_rows")


def add_f32(a, b, y):
    rc = _lib.load().dsvg_add_f32(a.data_ptr(), b.data_ptr(), y.data_ptr(), y.numel(), _stream())
    _lib.check(rc, "dsvg_add_f32")


def match_assign(cmd_logits, args_logits, ld_args, vis_logits, commands, args, N, G, Gp, L, n_args, n_classes):
    """Hungarian self-matching (model.py:311-350) on the GPU: returns (assignment int64 [N, Gp], cost fp64 [N, G, Gp],
    visible uint8 [N, G])."""
    dev = cmd_logits.device
    n_tok = N * Gp * (L - 1)
    lse_c = torch.empty(n_tok, device=dev)
    lse_a = torch.empty(n_tok * n_args, device=dev)
    cost = torch.empty(N, G, Gp, dtype=torch.float64, device=dev)
    vis = torch.empty(N, G, dtype=torch.uint8, device=dev)
    asg = torch.empty(N, Gp, dtype=torch.int64, device=dev)
    rc = _lib.load().dsvg_match_assign(cmd_logits.data_ptr(), cmd_logits.shape[-1], args_logits.data_ptr(), ld_args, n_args,
                                       n_classes, vis_logits.data_ptr(), commands.data_ptr(), args.data_ptr(), N, G, Gp, L,
                                       lse_c.data_ptr(), lse_a.data_ptr(), cost.data_ptr(), vis.data_ptr(), asg.data_ptr(),
                                       _stream())
    _lib.check(rc, "dsvg_match_assign")
    return asg, cost, vis


def permute_groups(src, dst, asg, N, G, group_bytes, inverse=False):
    """dst group (n, i) = src group (n, asg[n, i]) (or the inverse scatter); src / dst: tensors or raw pointers."""
    sp = src if isinstance(src, int) else src.data_ptr()
    dp = dst if isinstance(dst, int) else dst.data_ptr()
    rc = _lib.load().dsvg_permute_groups(sp, dp, asg.data_ptr(), N, G, group_bytes, 1 if inverse else 0, _stream())
    _lib.check(rc, "dsvg_permute_groups")


def permute_act(src, dst, asg, N, G, rows_per_group, inverse=False):
    """Group permutation of an Act (every plane)."""
    gb = rows_per_group * src.ld * 2
    for pl in range(src.planes):
        off = pl * src.rows * src.ld * 2
        permute_groups(src.ptr + off, dst.ptr + off, asg, N, G, gb, inverse)
