"""End-to-end parity on the GPU: deepsvg_b200.SVGTransformer + SVGLoss (CUDA, through the C ABI) against the CPU oracle
(oracle/svg_oracle.py, itself pinned to the reference by tests/test_oracle_golden.py) and against the committed
reference goldens, on the same seeded weights and inputs.

Tolerances (BASELINE.json north_star): logits / loss rtol=1e-3, atol=1e-4 and bit-exact argmax in parity mode
("bf16x3": split-bf16 operands on the same wgmma kernels).  Fast mode ("bf16", single-pass bf16 operands) cannot
meet that end-to-end for ANY implementation (SURVEY.md section 7, hard part 1); it is held to a looser, stated bound.
"""
import os

import numpy as np
import pytest
import torch

from oracle import svg_oracle as O
from tests.golden_cases import load_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W = dict(O.DEFAULT_WEIGHTS)


def _build(cfg_o, precision, seed=7):
    from deepsvg_b200 import SVGLoss, SVGTransformer
    from deepsvg_b200.config import _DefaultConfig
    cfg = _DefaultConfig(**{k: v for k, v in vars(cfg_o).items()})
    model = SVGTransformer(cfg, precision=precision)
    params = O.make_params(cfg_o, seed=seed)
    missing, unexpected = model.load_state_dict(params, strict=False)
    assert not unexpected and all(("position" in k or k in ("cmd_args_mask", "decoder.square_subsequent_mask")) for k in missing)
    return model.to(DEV).eval(), SVGLoss(cfg).to(DEV), params


def _run(model, loss_fn, cmd, arg, label=None, eps=None):
    model._eps_override = eps.to(DEV) if eps is not None else None
    model.zero_grad(set_to_none=True)
    out = model(cmd.to(DEV), arg.to(DEV), cmd.to(DEV), arg.to(DEV), label=None if label is None else label.to(DEV),
                params={})
    ls = loss_fn(out, None, weights=W)
    ls["loss"].backward()
    grads = {k: p.grad.detach().cpu() for k, p in model.named_parameters()}
    return out, ls, grads


def _check_grads(grads, ref, rel_tol):
    worst = ("", 0.0)
    for k, g in ref.items():
        denom = g.norm().item() + 1e-12
        e = (grads[k] - g).norm().item() / denom
        if e > worst[1]:
            worst = (k, e)
        assert e < rel_tol, (k, e)
    return worst


CASES = {
    "hier": ("hierarchical", dict(use_vae=False), 4),
    "hier_vae_label": ("hierarchical", dict(use_vae=True, label_condition=True, n_labels=52, dim_z=128), 3),
    "one_stage_fonts": ("one_stage", dict(use_vae=True, label_condition=True, n_labels=52, max_total_len=50), 5),
    "small_d128": ("hierarchical", dict(use_vae=False, d_model=128, n_heads=4, dim_feedforward=256, dim_z=64, n_layers=2,
                                        n_layers_decode=2, max_num_groups=4, max_seq_len=10), 6),
    # attention on the fp32 SIMT kernels end to end: head_dim 16, and a one-stage sequence of 102 positions (> 80)
    "hier_hd16": ("hierarchical", dict(use_vae=False, d_model=128, n_heads=8), 2),
    "one_stage_long": ("one_stage", dict(use_vae=False, d_model=256, n_heads=4, max_total_len=100), 2),
}


@pytest.mark.parametrize("name", list(CASES))
def test_parity_mode_matches_oracle(name):
    kind, over, n = CASES[name]
    cfg = O.make_cfg(kind, **over)
    model, loss_fn, params = _build(cfg, "bf16x3")
    cmd, arg = O.synth_batch(cfg, n, seed=21)
    label = torch.randint(0, cfg.n_labels, (n,), generator=torch.Generator().manual_seed(2)) if cfg.label_condition else None
    eps = torch.randn(n, cfg.dim_z, generator=torch.Generator().manual_seed(3)) if cfg.use_vae else None
    out, ls, grads = _run(model, loss_fn, cmd, arg, label, eps)
    ro, rl, rg = O.train_step(params, cfg, cmd, arg, label=label, eps=eps)
    for k in ("command_logits", "args_logits", "visibility_logits", "mu", "logsigma"):
        if k in ro:
            got = out[k].detach().cpu()
            assert got.shape == ro[k].shape, k
            np.testing.assert_allclose(got.numpy(), ro[k].numpy(), rtol=1e-3, atol=1e-4, err_msg=k)
    # bit-exact argmax of command / argument predictions (positions whose fp32 top-2 margin is below the parity
    # tolerance itself are genuine ties of the random-init logits and are excluded; there are a handful per 10^4)
    for k in ("command_logits", "args_logits"):
        top2 = ro[k].topk(2, dim=-1).values
        decided = (top2[..., 0] - top2[..., 1]) > 2e-4
        same = out[k].argmax(-1).cpu() == ro[k].argmax(-1)
        assert bool((same | ~decided).all()), k
        assert decided.float().mean().item() > 0.995, k
    for k, v in rl.items():
        assert abs(ls[k].item() - v.item()) <= 1e-3 * abs(v.item()) + 1e-4, (k, ls[k].item(), v.item())
    # Gradients: split-bf16 operands carry 16 mantissa bits, so ~1e-5 of the ReLU pre-activations sit on the other side
    # of zero than in fp32 and flip their mask; expected relative L2 error sqrt(n_flip / n) ~ 4e-3 on the tensors
    # behind few rows (measured 3.6e-3 on decoder.decoder.layers.0.*; the CPU oracle run with matmul='bf16x3' shows
    # the same 3.6e-3 on the same tensors -- see DESIGN.md 'Gradient tolerance').
    _check_grads(grads, rg, 1e-2)


@pytest.mark.parametrize("name", ["hier_cfg1", "scaled_cfg5", "fonts_cfg4"])
def test_parity_mode_matches_reference_golden(name):
    """BASELINE.json configs[0] (hierarchical_ordered, batch 2), configs[4] (scaled: d_model 512, 8 layers, 16 x 64,
    head_dim 64, batch 2) and configs[3] (one-stage fonts, 52 labels, VAE, batch 3) -- against numbers produced by the
    reference itself (tests/golden/make_golden.py)."""
    cfg, fx, _ = load_case(name)
    model, loss_fn, _ = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    cmd, arg = torch.from_numpy(fx["commands"]), torch.from_numpy(fx["args"])
    label = torch.from_numpy(fx["label"]) if "label" in fx else None
    eps = torch.from_numpy(fx["eps"]).float() if "eps" in fx else None
    out, ls, grads = _run(model, loss_fn, cmd, arg, label, eps)
    idx = lambda t, n: t.reshape(-1)[torch.linspace(0, t.numel() - 1, n).long().clamp_(max=t.numel() - 1)]
    for k in ("command_logits", "args_logits", "visibility_logits", "mu", "logsigma"):
        if "O_" + k not in fx:
            continue
        assert tuple(out[k].shape) == tuple(fx["O_shape_" + k]), k
        got = idx(out[k].detach().cpu(), 4096) if out[k].numel() > 4096 else out[k].detach().cpu().reshape(-1)
        np.testing.assert_allclose(got.numpy(), fx["O_" + k].reshape(-1), rtol=1e-3, atol=1e-4, err_msg=k)
    for k in ("loss", "loss_cmd", "loss_args", "loss_visibility", "loss_kl"):
        if "L_" + k in fx:
            assert abs(ls[k].item() - float(fx["L_" + k])) <= 1e-3 * float(fx["L_" + k]), k
    for k, g in grads.items():
        ref_norm = float(fx["Gnorm_" + k])
        assert abs(g.double().norm().item() - ref_norm) <= 1e-2 * ref_norm + 1e-9, k


@pytest.mark.parametrize("name", ["scaled_cfg5", "fonts_cfg4"])
def test_fast_mode_on_baseline_configs_4_and_5(name):
    """Fast mode (single-plane bf16) on the two other BASELINE configs: head_dim 64 / L = 66, 65, 16 and L = 52, 51 run the
    general tensor-core attention kernel; bounded like test_fast_mode_deviation_is_bounded."""
    cfg, fx, _ = load_case(name)
    model, loss_fn, _ = _build(cfg, "bf16", seed=int(fx["seed_params"]))
    cmd, arg = torch.from_numpy(fx["commands"]), torch.from_numpy(fx["args"])
    label = torch.from_numpy(fx["label"]) if "label" in fx else None
    eps = torch.from_numpy(fx["eps"]).float() if "eps" in fx else None
    out, ls, grads = _run(model, loss_fn, cmd, arg, label, eps)
    idx = lambda t, n: t.reshape(-1)[torch.linspace(0, t.numel() - 1, n).long().clamp_(max=t.numel() - 1)]
    got = idx(out["args_logits"].detach().cpu(), 4096)
    assert (got - torch.from_numpy(fx["O_args_logits"].reshape(-1)).float()).abs().max().item() < 0.08
    assert abs(ls["loss"].item() - float(fx["L_loss"])) < 2e-2 * float(fx["L_loss"])
    bad = [(k, abs(g.double().norm().item() - float(fx["Gnorm_" + k])) / (float(fx["Gnorm_" + k]) + 1e-12))
           for k, g in grads.items()]
    worst = max(bad, key=lambda kv: kv[1])
    assert worst[1] < 0.2, worst


def test_fast_mode_deviation_is_bounded():
    """Single-pass bf16 operands (bf16 probabilities inside the mma.sync attention): reported honestly, bounded loosely
    (loss within 1 %, logits within 0.05 abs, argument argmax agreement > 97 %, gradients within 15 % relative L2;
    measured worst tensor: encoder.embedding.command_embed.weight at 8.8 %)."""
    kind, over, n = CASES["hier"]
    cfg = O.make_cfg(kind, **over)
    model, loss_fn, params = _build(cfg, "bf16")
    cmd, arg = O.synth_batch(cfg, n, seed=21)
    out, ls, grads = _run(model, loss_fn, cmd, arg)
    ro, rl, rg = O.train_step(params, cfg, cmd, arg)
    err = (out["args_logits"].detach().cpu() - ro["args_logits"]).abs().max().item()
    agree = (out["args_logits"].argmax(-1).cpu() == ro["args_logits"].argmax(-1)).float().mean().item()
    assert err < 0.05 and agree > 0.97, (err, agree)
    assert abs(ls["loss"].item() - rl["loss"].item()) < 1e-2 * rl["loss"].item()
    _check_grads(grads, rg, 1.5e-1)


def test_train_mode_dropout_statistics_and_loss_api():
    """train(): stochastic, seeded per call, finite; the loss dict has the reference's keys and .item() works."""
    cfg = O.make_cfg("hierarchical", use_vae=True)
    model, loss_fn, _ = _build(cfg, "bf16")
    model.train()
    cmd, arg = O.synth_batch(cfg, 4, seed=5)
    c, a = cmd.to(DEV), arg.to(DEV)
    o1 = model(c, a, c, a, params={})
    o2 = model(c, a, c, a, params={})
    assert not torch.equal(o1["args_logits"], o2["args_logits"])
    ls = loss_fn(o1, None, weights=W)
    assert set(ls) == {"loss", "loss_cmd", "loss_args", "loss_visibility", "loss_kl"}
    ls["loss"].backward()
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())
    assert all(np.isfinite(v.item()) for v in ls.values())
    assert set(o1) == {"command_logits", "args_logits", "visibility_logits", "tgt_commands", "tgt_args", "mu", "logsigma"}
    assert o1["args_logits"].shape == (4, 8, 31, 11, 257) and o1["visibility_logits"].shape == (4, 8, 1, 2)


def test_generic_autograd_path_matches_fused_path():
    """A user loss on the logits (no SVGLoss): gradients must flow through the explicit-gradient path."""
    cfg = O.make_cfg("hierarchical", use_vae=False)
    model, loss_fn, _ = _build(cfg, "bf16x3")
    cmd, arg = O.synth_batch(cfg, 2, seed=9)
    c, a = cmd.to(DEV), arg.to(DEV)
    model.zero_grad(set_to_none=True)
    out = model(c, a, c, a, params={})
    ls = loss_fn(out, None, weights=W)
    ls["loss"].backward()
    g_fused = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    out = model(c, a, c, a, params={})
    O.CMD_ARGS_MASK = O.CMD_ARGS_MASK.to(DEV)
    try:
        plain = {k: (v if k.startswith("tgt") else v) for k, v in out.items()}
        O.loss(plain, cfg, W)["loss"].backward()
    finally:
        O.CMD_ARGS_MASK = O.CMD_ARGS_MASK.cpu()
    for k, p in model.named_parameters():
        e = (p.grad - g_fused[k]).norm().item() / (g_fused[k].norm().item() + 1e-12)
        assert e < 1e-2, (k, e)


def test_encode_mode_and_z_injection():
    cfg = O.make_cfg("hierarchical", use_vae=False)
    model, _, params = _build(cfg, "bf16x3")
    cmd, arg = O.synth_batch(cfg, 3, seed=4)
    c, a = cmd.to(DEV), arg.to(DEV)
    with torch.no_grad():
        z = model(c, a, None, None, encode_mode=True)
        assert z.shape == (1, 1, 3, cfg.dim_z)
        ro = O.forward(params, cfg, cmd, arg)
        np.testing.assert_allclose(z.view(3, -1).cpu().numpy(), ro["z"].numpy(), rtol=1e-3, atol=1e-4)
        out = model(None, None, None, None, z=z.view(3, 1, 1, -1), return_tgt=False)
        np.testing.assert_allclose(out["args_logits"].cpu().numpy(), ro["args_logits"].numpy(), rtol=1e-3, atol=1e-4)
        assert "tgt_commands" not in out


def test_greedy_sample_matches_oracle_decoding():
    """SURVEY.md 8f rank 1: one-shot greedy decoding on top of the CUDA forward, against the same post-processing of the
    oracle's logits (argmax, visibility threshold 0.7, CMD_ARGS_MASK, EOS truncation)."""
    cfg = O.make_cfg("hierarchical", use_vae=False)
    model, _, params = _build(cfg, "bf16x3")
    cmd, arg = O.synth_batch(cfg, 3, seed=12)
    c, a = cmd.to(DEV), arg.to(DEV)
    cy, ay = model.greedy_sample(c, a, None, None, concat_groups=False)
    ro = O.forward(params, cfg, cmd, arg)
    rc, ra = ro["command_logits"].argmax(-1), ro["args_logits"].argmax(-1) - 1
    vis = torch.softmax(ro["visibility_logits"], -1)[..., 1].squeeze(-1) > 0.7
    blank = torch.full((rc.shape[-1],), 4)
    blank[0] = 0
    rc = torch.where(~vis[..., None], blank, rc)
    ra = torch.where(~vis[..., None, None], torch.full_like(ra, -1), ra)
    ra = torch.where(O.CMD_ARGS_MASK[rc].bool(), ra, torch.full_like(ra, -1))
    # tokens must agree wherever the oracle's decision is not a tie at the parity tolerance
    t2 = ro["command_logits"].topk(2, -1).values
    sure_c = (t2[..., 0] - t2[..., 1]) > 2e-4
    assert bool(((cy.cpu() == rc) | ~sure_c).all())
    t2 = ro["args_logits"].topk(2, -1).values
    sure_a = ((t2[..., 0] - t2[..., 1]) > 2e-4) & sure_c[..., None]
    assert bool(((ay.cpu() == ra) | ~sure_a).all())
    assert cy.shape == (3, 8, 31) and ay.shape == (3, 8, 31, 11)
    # concat_groups=True keeps exactly the tokens before each path's first EOS (N = 1, as every reference caller uses it)
    c1, a1 = model.greedy_sample(c[:1], a[:1], None, None)
    k1, _ = model.greedy_sample(c[:1], a[:1], None, None, concat_groups=False)
    assert c1.shape[0] == 1 and c1.shape[1] == int(((k1 == 4).cumsum(-1) == 0).sum()) and a1.shape[1:] == (c1.shape[1], 11)


def test_parity_mode_on_edge_inputs_matches_reference_golden():
    """One-command / empty / max-length paths, the 'a' and 'z' commands, extreme argument values -- against numbers
    produced by the reference itself (tests/golden/make_golden.py: edge_d128)."""
    cfg, fx, _ = load_case("edge_d128")
    model, loss_fn, _ = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    cmd, arg = torch.from_numpy(fx["commands"]), torch.from_numpy(fx["args"])
    out, ls, grads = _run(model, loss_fn, cmd, arg)
    idx = lambda t, n: t.reshape(-1)[torch.linspace(0, t.numel() - 1, n).long().clamp_(max=t.numel() - 1)]
    for k in ("command_logits", "args_logits", "visibility_logits"):
        assert tuple(out[k].shape) == tuple(fx["O_shape_" + k]), k
        got = idx(out[k].detach().cpu(), 4096) if out[k].numel() > 4096 else out[k].detach().cpu().reshape(-1)
        np.testing.assert_allclose(got.numpy(), fx["O_" + k].reshape(-1), rtol=1e-3, atol=1e-4, err_msg=k)
    for k in ("loss", "loss_cmd", "loss_args", "loss_visibility"):
        assert abs(ls[k].item() - float(fx["L_" + k])) <= 1e-3 * float(fx["L_" + k]), k
    for k, g in grads.items():
        ref_norm = float(fx["Gnorm_" + k])
        assert abs(g.double().norm().item() - ref_norm) <= 1e-2 * ref_norm + 1e-9, k


def test_fused_adamw_updates_reach_the_gemm_weights():
    """ADVICE r1 (high): FusedAdamW writes the fp32 masters through raw pointers; the model's bf16 weight-operand cache is
    keyed on `_version`, so the optimizer must bump it.  Two train steps with FusedAdamW against torch.optim.AdamW +
    clip_grad_norm_ on an identical model: the logits of the SECOND forward (which sees the updated weights) must agree."""
    from deepsvg_b200 import FusedAdamW
    cfg = O.make_cfg("hierarchical", use_vae=False, d_model=128, n_heads=4, dim_feedforward=256, dim_z=64, n_layers=2,
                     n_layers_decode=2, max_num_groups=4, max_seq_len=10)
    cmd, arg = O.synth_batch(cfg, 4, seed=31)
    c, a = cmd.to(DEV), arg.to(DEV)
    logits = []
    for fused in (True, False):
        model, loss_fn, _ = _build(cfg, "bf16x3", seed=11)
        if fused:
            opt = FusedAdamW(model.parameters(), lr=3e-3, weight_decay=1e-2, max_grad_norm=1.0)
        else:
            opt = torch.optim.AdamW(model.parameters(), lr=3e-3, weight_decay=1e-2)
        outs = []
        for _ in range(3):
            model.zero_grad(set_to_none=True)
            out = model(c, a, c, a, params={})
            outs.append(out["args_logits"].detach().clone())
            loss_fn(out, None, weights=W)["loss"].backward()
            if not fused:
                torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
            opt.step()
        logits.append(outs)
    moved = (logits[0][1] - logits[0][0]).abs().max().item()
    assert moved > 1e-3, "the second forward did not see the optimizer update (stale weight cache)"
    for s in (1, 2):
        # two different (both correct) AdamW / clipping implementations: agreement to a few 1e-4 after lr = 3e-3 updates
        np.testing.assert_allclose(logits[0][s].cpu().numpy(), logits[1][s].cpu().numpy(), rtol=5e-3, atol=2e-3)


def test_parity_mode_at_the_benchmarked_shape():
    """BASELINE configs[1] at its real size: 512 icons = 131 072 path-level rows (1 024 row tiles over one persistent CTA per SM,
    one-wave weight-gradient splits), bf16x3, eval mode, against the fp32 CPU oracle: loss terms, sampled logits, argmax on
    decided positions, every gradient tensor's relative L2 error."""
    cfg = O.make_cfg("hierarchical", use_vae=False)
    model, loss_fn, params = _build(cfg, "bf16x3", seed=5)
    import bench
    cmd, arg = bench.synth_icons(512, seed=77)
    out, ls, grads = _run(model, loss_fn, cmd, arg)
    torch.set_num_threads(min(32, torch.get_num_threads() if torch.get_num_threads() > 1 else (os.cpu_count() or 1)))
    ro, rl, rg = O.train_step(params, cfg, cmd, arg)
    for k in ("command_logits", "args_logits", "visibility_logits"):
        got, ref = out[k].detach().cpu(), ro[k]
        assert got.shape == ref.shape
        sel = torch.linspace(0, got.numel() - 1, 200_000, dtype=torch.float64).long().clamp_(max=got.numel() - 1)
        np.testing.assert_allclose(got.reshape(-1)[sel].numpy(), ref.reshape(-1)[sel].numpy(), rtol=1e-3, atol=1e-4,
                                   err_msg=k)
    for k in ("command_logits", "args_logits"):
        top2 = ro[k].topk(2, dim=-1).values
        decided = (top2[..., 0] - top2[..., 1]) > 2e-4
        same = out[k].argmax(-1).cpu() == ro[k].argmax(-1)
        assert bool((same | ~decided).all()), k
    for k, v in rl.items():
        assert abs(ls[k].item() - v.item()) <= 1e-3 * abs(v.item()) + 1e-4, (k, ls[k].item(), v.item())
    _check_grads(grads, rg, 1e-2)


def test_nccl_data_parallel_gradients_match_single_process():
    """The product's NCCL path (per-rank SVGLoss scaled by all-reduced global counts + flat-bucket all-reduce) on 2 GPUs
    against the single-process gradient of the concatenated batch -- bench.py's ddp_check, run under torchrun."""
    import json
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs; bench.py --gpus 2 under torchrun reports the same ddp_check line")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29541", os.path.join(root, "bench.py"), "--gpus", "2",
                        "--steps", "2", "--warmup", "3", "--batch", "32", "--no-parity-mode"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    line = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    chk = line["ddp_check"]
    assert chk["max_rel_grad_err"] < 1e-3 and chk["rel_loss_err"] < 1e-5, chk


# ------------------------------------------------------------------------------------------------ CUDA graphs
def _train_pair(cfg, n=6, seed=3):
    from deepsvg_b200 import SVGLoss, SVGTransformer
    from deepsvg_b200.config import _DefaultConfig
    c = _DefaultConfig(**{k: v for k, v in vars(cfg).items()})
    params = O.make_params(cfg, seed=seed)
    models = []
    for g in (True, False):
        m = SVGTransformer(c, precision="bf16", graphs=g)
        m.load_state_dict(params, strict=False)
        models.append(m.to(DEV).train())
    return models, SVGLoss(c).to(DEV)


def test_cuda_graph_step_matches_eager_step():
    """Train mode, dropout on: from the third call with the same input signature the step is three graph replays.  With
    the same torch CUDA seed both paths draw the same dropout seed, so loss and gradients must agree (fp32 atomics in the
    weight-gradient reductions are the only non-determinism)."""
    cfg = O.make_cfg("hierarchical", use_vae=False, d_model=128, n_heads=4, dim_feedforward=256, dim_z=64, n_layers=2,
                     n_layers_decode=2, max_num_groups=4, max_seq_len=10)
    (mg, me), loss_fn = _train_pair(cfg)
    batches = [O.synth_batch(cfg, 6, seed=40 + i) for i in range(6)]
    for i, (cmd, arg) in enumerate(batches):
        c, a = cmd.to(DEV), arg.to(DEV)
        res = []
        for m in (mg, me):
            torch.manual_seed(1000 + i)
            m.zero_grad(set_to_none=True)
            out = m(c, a, c, a, params={})
            ls = loss_fn(out, None, weights=W)
            ls["loss"].backward()
            res.append((ls["loss"].item(), out["args_logits"].detach().clone(),
                        {k: p.grad.detach().clone() for k, p in m.named_parameters()}))
        assert (mg._gs is not None) == (i >= 2), i
        assert abs(res[0][0] - res[1][0]) < 1e-5 * abs(res[1][0]), (i, res[0][0], res[1][0])
        assert torch.allclose(res[0][1], res[1][1], rtol=1e-5, atol=1e-6), i
        for k, g in res[1][2].items():
            e = (res[0][2][k] - g).norm().item() / (g.norm().item() + 1e-12)
            assert e < 1e-4, (i, k, e)
    assert me._gs is None
    # different dropout masks on consecutive replays (the seed lives in device memory)
    c, a = batches[0][0].to(DEV), batches[0][1].to(DEV)
    o1 = mg(c, a, c, a, params={})["args_logits"].clone()
    o2 = mg(c, a, c, a, params={})["args_logits"].clone()
    assert not torch.equal(o1, o2)


def test_cuda_graph_guards_and_optimizer_updates():
    """(a) backward of an earlier forward after a later replay must raise (one activation set); (b) FusedAdamW updates
    reach the captured graphs (weights are re-cast outside the graph when their version changes); (c) a new input
    signature drops the old capture."""
    from deepsvg_b200 import FusedAdamW
    cfg = O.make_cfg("hierarchical", use_vae=True, d_model=128, n_heads=4, dim_feedforward=256, dim_z=64, n_layers=2,
                     n_layers_decode=2, max_num_groups=4, max_seq_len=10)
    (mg, me), loss_fn = _train_pair(cfg)
    cmd, arg = O.synth_batch(cfg, 5, seed=9)
    c, a = cmd.to(DEV), arg.to(DEV)
    opt = FusedAdamW(mg.parameters(), lr=2e-3, max_grad_norm=1.0)
    losses = []
    for i in range(12):
        mg.zero_grad(set_to_none=True)
        ls = loss_fn(mg(c, a, c, a, params={}), None, weights=W)
        ls["loss"].backward()
        assert all(torch.isfinite(p.grad).all() for p in mg.parameters())
        opt.step()
        losses.append(ls["loss_args"].item() + ls["loss_cmd"].item())
    assert mg._gs is not None and mg._gs.bwd_a is not None
    assert losses[-1] < losses[2] - 0.05, losses          # it learns: the replays see the updated weights
    o1 = mg(c, a, c, a, params={})
    l1 = loss_fn(o1, None, weights=W)["loss"]
    o2 = mg(c, a, c, a, params={})
    with pytest.raises(RuntimeError, match="overwrote the captured"):
        l1.backward()
    gs = mg._gs
    cmd2, arg2 = O.synth_batch(cfg, 3, seed=10)
    c2, a2 = cmd2.to(DEV), arg2.to(DEV)
    for _ in range(3):
        mg.zero_grad(set_to_none=True)
        loss_fn(mg(c2, a2, c2, a2, params={}), None, weights=W)["loss"].backward()
    assert mg._gs is not None and mg._gs is not gs and mg._gs.key != gs.key


# ------------------------------------------------------------------------------------------------ Hungarian self-matching
def test_self_match_matches_reference_golden():
    """HierarchicalSelfMatching (model/config.py:101-108): cost tensor, Hungarian assignment and the slot permutation on the
    GPU against numbers produced by the reference itself (scipy solver, torch.gather) -- assignment bit-exact, permuted
    logits / losses / every gradient within the parity tolerances."""
    cfg, fx, _ = load_case("selfmatch_d128")
    model, loss_fn, _ = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    assert "encoder.hierarchical_PE.pos_embed.weight" not in dict(model.named_parameters())
    cmd, arg = torch.from_numpy(fx["commands"]), torch.from_numpy(fx["args"])
    out, ls, grads = _run(model, loss_fn, cmd, arg)
    idx = lambda t, n: t.reshape(-1)[torch.linspace(0, t.numel() - 1, n).long().clamp_(max=t.numel() - 1)]
    for k in ("command_logits", "args_logits", "visibility_logits"):
        assert tuple(out[k].shape) == tuple(fx["O_shape_" + k]), k
        got = idx(out[k].detach().cpu(), 4096) if out[k].numel() > 4096 else out[k].detach().cpu().reshape(-1)
        np.testing.assert_allclose(got.numpy(), fx["O_" + k].reshape(-1), rtol=1e-3, atol=1e-4, err_msg=k)
    for k in ("loss", "loss_cmd", "loss_args", "loss_visibility"):
        assert abs(ls[k].item() - float(fx["L_" + k])) <= 1e-3 * float(fx["L_" + k]), k
    for k, g in grads.items():
        ref_norm = float(fx["Gnorm_" + k])
        assert abs(g.double().norm().item() - ref_norm) <= 1e-2 * ref_norm + 1e-9, k


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_self_match_assignment_and_gradients_match_oracle(precision):
    """d_model 256, 8 paths: the GPU solver must pick the oracle's (scipy's) assignment wherever the optimum is separated
    from the runner-up by more than the logit tolerance; gradients flow through the permutation."""
    from deepsvg_b200 import ops
    cfg = O.make_cfg("hierarchical", use_vae=False, self_match=True)
    model, loss_fn, params = _build(cfg, precision, seed=13)
    cmd, arg = O.synth_batch(cfg, 5, seed=77)
    out, ls, grads = _run(model, loss_fn, cmd, arg)
    ro, rl, rg = O.train_step(params, cfg, cmd, arg)
    asg_ref = ro["assignment"]
    # the kernel's assignment for the ORACLE's logits is exact (same costs up to fp32 rounding)
    raw = O.forward(params, O.make_cfg("hierarchical", use_vae=False), cmd, arg) if False else None
    if precision == "bf16x3":
        np.testing.assert_allclose(out["args_logits"].detach().cpu().numpy(), ro["args_logits"].numpy(), rtol=1e-3, atol=1e-4)
        for k, v in rl.items():
            assert abs(ls[k].item() - v.item()) <= 1e-3 * abs(v.item()) + 1e-4, k
        _check_grads(grads, rg, 1e-2)
    else:
        assert abs(ls["loss"].item() - rl["loss"].item()) < 2e-2 * rl["loss"].item()
    assert any(r != sorted(r) for r in asg_ref.tolist())


def test_match_kernels_against_scipy_on_random_costs():
    """dsvg_match_assign on synthetic logits: the cost tensor against the oracle's restatement of model.py:313-337 and the
    per-icon assignment against scipy.optimize.linear_sum_assignment (the reference's solver), for G < Gp too."""
    from deepsvg_b200 import ops
    g = torch.Generator().manual_seed(5)
    for (N, G, Gp, S) in ((37, 8, 8, 30), (9, 5, 16, 12), (4, 16, 16, 64)):
        cfg = O.make_cfg("hierarchical", use_vae=False, max_num_groups=G, num_groups_proposal=Gp, max_seq_len=S)
        cmd, arg = O.synth_batch(cfg, N, seed=N)
        Ld, C = S + 1, 257
        cl = torch.randn(N, Gp, Ld, 7, generator=g)
        al = torch.randn(N, Gp, Ld, 11, C, generator=g) * 2
        vl = torch.randn(N, Gp, 1, 2, generator=g)
        cost_ref, vis_ref = O.matching_costs(cl.double(), al.double(), vl.double(), cmd[..., 1:], arg[..., 1:, :])
        asg_ref = O.perfect_matching(cl.double(), al.double(), vl.double(), cmd[..., 1:], arg[..., 1:, :], cfg)
        asg, cost, vis = ops.match_assign(cl.to(DEV).view(-1, 7), al.to(DEV).view(-1, 11 * C), 11 * C, vl.to(DEV).view(-1, 2),
                                          cmd.to(DEV), arg.to(DEV), N, G, Gp, S + 2, 11, C)
        assert torch.equal(vis.cpu().bool(), vis_ref)
        m = vis_ref[:, :, None].expand_as(cost_ref)
        np.testing.assert_allclose(cost.cpu()[m].numpy(), cost_ref[m].numpy(), rtol=2e-5, atol=2e-5)
        assert asg.cpu().tolist() == asg_ref.tolist()
        # the permutation kernel and its inverse
        x = torch.randn(N * Gp * 3, 40, device=DEV)
        y, z = torch.empty_like(x), torch.empty_like(x)
        ops.permute_groups(x, y, asg, N, Gp, 3 * 40 * 4)
        want = torch.gather(x.view(N, Gp, 120), 1, asg[:, :, None].expand(N, Gp, 120)).reshape_as(x)
        assert torch.equal(y, want)
        ops.permute_groups(y, z, asg, N, Gp, 3 * 40 * 4, inverse=True)
        assert torch.equal(z, x)


def test_forward_from_hierarch_logits():
    """model.py:246-259: second-stage decoding from the per-path latents and visibility logits of a return_hierarch call."""
    cfg = O.make_cfg("hierarchical", use_vae=False)
    model, _, _ = _build(cfg, "bf16x3")
    cmd, arg = O.synth_batch(cfg, 3, seed=4)
    c, a = cmd.to(DEV), arg.to(DEV)
    with torch.no_grad():
        full = model(c, a, c, a, return_tgt=False)
        vis, zp = model(c, a, None, None, return_hierarch=True)          # (1, Gp, N, 2), (1, Gp, N, dz)
        assert vis.shape == (1, 8, 3, 2) and zp.shape == (1, 8, 3, cfg.dim_z)
        again = model(None, None, None, None, z=zp.permute(2, 1, 0, 3), hierarch_logits=vis, return_tgt=False)
    for k in ("command_logits", "args_logits", "visibility_logits"):
        assert torch.allclose(again[k], full[k], rtol=1e-5, atol=1e-6), k


# ------------------------------------------------------------------------------------------------ autoregressive decoder
def _sketch_inputs(fx):
    cmd, arg = torch.from_numpy(fx["commands"]), torch.from_numpy(fx["args"])
    return cmd, arg, torch.from_numpy(fx["args_dec"])


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_sketchformer_matches_reference_golden(precision):
    """Sketchformer (model/config.py:74-80): one-stage encoder, AUTOREGRESSIVE decoder (its own SVGEmbedding of the shifted
    targets, causal + key-padding attention), relative argument targets (512 classes) -- against numbers produced by the
    reference itself."""
    cfg, fx, _ = load_case("sketchformer_d128")
    model, loss_fn, _ = _build(cfg, precision, seed=int(fx["seed_params"]))
    cmd, arg, arg_dec = _sketch_inputs(fx)
    model.zero_grad(set_to_none=True)
    c, a, ad = cmd.to(DEV), arg.to(DEV), arg_dec.to(DEV)
    out = model(c, a, c, ad, params={})
    ls = loss_fn(out, None, weights=W)
    ls["loss"].backward()
    grads = {k: p.grad.detach().cpu() for k, p in model.named_parameters()}
    assert tuple(out["args_logits"].shape) == tuple(fx["O_shape_args_logits"]) and out["args_logits"].shape[-1] == 512
    idx = lambda t, n: t.reshape(-1)[torch.linspace(0, t.numel() - 1, n).long().clamp_(max=t.numel() - 1)]
    if precision == "bf16x3":
        for k in ("command_logits", "args_logits"):
            got = idx(out[k].detach().cpu(), 4096) if out[k].numel() > 4096 else out[k].detach().cpu().reshape(-1)
            np.testing.assert_allclose(got.numpy(), fx["O_" + k].reshape(-1), rtol=1e-3, atol=1e-4, err_msg=k)
        for k in ("loss", "loss_cmd", "loss_args"):
            assert abs(ls[k].item() - float(fx["L_" + k])) <= 1e-3 * float(fx["L_" + k]), k
        for k, g in grads.items():
            ref_norm = float(fx["Gnorm_" + k])
            assert abs(g.double().norm().item() - ref_norm) <= 1e-2 * ref_norm + 1e-9, k
    else:
        assert abs(ls["loss"].item() - float(fx["L_loss"])) < 2e-2 * float(fx["L_loss"])
        worst = max(abs(g.double().norm().item() - float(fx["Gnorm_" + k])) / (float(fx["Gnorm_" + k]) + 1e-12)
                    for k, g in grads.items())
        assert worst < 0.2, worst
    assert set(ls) == {"loss", "loss_cmd", "loss_args"}


def test_sketchformer_greedy_decoding_is_self_consistent():
    """model.py:428-448: token-by-token decoding.  Teacher-forcing the ORACLE on the decoded prefix must reproduce every
    decoded token (wherever the oracle's own top-2 margin is decisive)."""
    cfg, fx, _ = load_case("sketchformer_d128")
    model, _, params = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    cmd, arg, _ = _sketch_inputs(fx)
    c, a = cmd[:2].to(DEV), arg[:2].to(DEV)
    with torch.no_grad():
        z = model(c, a, None, None, encode_mode=True).permute(2, 0, 1, 3)        # (N, 1, 1, dz)
        # the decoding loop of greedy_sample, kept in relative coordinates (no _make_absolute)
        N, T = 2, cfg.max_total_len
        cy = torch.full((N, 1, 1), 5, dtype=torch.long, device=DEV)
        ay = torch.full((N, 1, 1, 11), -1, dtype=torch.long, device=DEV)
        for _ in range(T):
            res = model(None, None, cy.float(), ay.float(), z=z, return_tgt=False)
            cn, an = res["command_logits"].argmax(-1), res["args_logits"].argmax(-1) - 1
            _, an = model._make_valid(cn, an)
            cy, ay = torch.cat([cy, cn[..., -1:]], -1), torch.cat([ay, an[..., -1:, :]], -2)
        # public API: absolute coordinates, SOS dropped
        cg, ag = model.greedy_sample(c, a, None, None, concat_groups=False)
    assert cg.shape == (N, 1, T) and ag.shape == (N, 1, T, 11) and torch.equal(cg, cy[..., 1:])
    # oracle, teacher-forced on [SOS, y_1 .. y_T] (+ one trailing position that forward drops)
    pad_c = torch.full((N, 1, 1), 4.0)
    pad_a = torch.full((N, 1, 1, 11), -1.0)
    cd = torch.cat([cy.cpu().float(), pad_c], -1)
    ad = torch.cat([ay.cpu().float(), pad_a], -2)
    zo = O.forward(params, cfg, cmd[:2], arg[:2], commands_dec=cd, args_dec=ad)
    lc, la = zo["command_logits"][:, :, :T], zo["args_logits"][:, :, :T]
    t2 = lc.topk(2, -1).values
    sure = (t2[..., 0] - t2[..., 1]) > 1e-3
    assert bool(((lc.argmax(-1) == cy.cpu()[..., 1:]) | ~sure).all()) and sure.float().mean().item() > 0.9
    used = O.CMD_ARGS_MASK[cy.cpu()[..., 1:]].bool()
    t2 = la.topk(2, -1).values
    sure_a = ((t2[..., 0] - t2[..., 1]) > 1e-3) & used & sure[..., None]
    assert bool((((la.argmax(-1) - 1) == ay.cpu()[..., 1:, :]) | ~sure_a).all())
