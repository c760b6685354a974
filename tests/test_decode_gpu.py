"""Cached autoregressive decoding on the GPU (csrc/decode.cu, SVGTransformer._greedy_sample_cached).

The three decode kernels against fp64 / fp32 restatements and the whole-prefix kernels they replace, then the cached
engine against the teacher-forced full forward, the fp64 CPU oracle (oracle/svg_oracle.py) and an explicit
`model.forward` decoding loop.

Tolerances: logits rtol 1e-3 / atol 1e-4 in parity mode ("bf16x3").  Fast mode ("bf16") rounds every activation to 8
mantissa bits; its logits are held to 5 % of the largest logit magnitude against the fp64 oracle.
"""
import numpy as np
import pytest
import torch

from oracle import svg_oracle as O
from tests.golden_cases import load_case
from tests.test_kernels_gpu import kernel_key, launched_kernels
from tests.test_model_gpu import _build

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# the longest max_total_len config.check_supported accepts per head_dim
LONGEST_T = {16: 153, 32: 139, 64: 115}


def _ops():
    from deepsvg_b200 import ops
    return ops


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _rel(a, b):
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def _mask():
    from deepsvg_b200.model import CMD_ARGS_MASK
    return CMD_ARGS_MASK.to(DEV).bool()


# ------------------------------------------------------------------------------------------------ decode attention
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("hd", [16, 32, 64])
def test_decode_attention_matches_fp64(hd, planes):
    """Every step t of the longest accepted sequence: the appended cache rows are the QKV rows bit for bit, and o equals
    softmax(q K^T over valid keys <= t) V.  Sequence 0 has no EOS, sequences 1 and 2 mask every key from 20 / 40 on."""
    ops = _ops()
    T, N, d = LONGEST_T[hd], 3, 128
    H = d // hd
    kv = torch.zeros(N, T, dtype=torch.uint8, device=DEV)
    for n, eos in enumerate((T, 20, 40)):
        kv[n, :eos] = 1
    kc, vc = ops.decode_cache(N, H, hd, T, planes, DEV), ops.decode_cache(N, H, hd, T, planes, DEV)
    step = torch.zeros(2, dtype=torch.int32, device=DEV)
    Ks, Vs = [], []
    for t in range(T):
        qkv = ops.act_from_float(_rand(N, 3 * d, seed=t), planes)
        o = ops.Act(N, d, planes, DEV)
        step[0] = t
        call = lambda: ops.decode_attn(step, qkv, kc, vc, kv, o, N, H, hd, T)
        if t == 1:
            names = {kernel_key(n) for n in launched_kernels(call)}
            assert "decode_attn_kernel<%d, %d>" % (hd, planes) in names, names
        else:
            call()
        raw = qkv.t[:, :, :3 * d].view(planes, N, 3, H, hd)
        assert torch.equal(kc[:, :, :, t], raw[:, :, 1]) and torch.equal(vc[:, :, :, t], raw[:, :, 2]), t
        val = qkv.float().double().view(N, 3, H, hd)
        Ks.append(val[:, 1])
        Vs.append(val[:, 2])
        K, V = torch.stack(Ks, 2), torch.stack(Vs, 2)                        # [N, H, t + 1, hd]
        s = torch.einsum("nhc,nhjc->nhj", val[:, 0], K)
        s = s.masked_fill(~kv[:, None, :t + 1].bool(), float("-inf"))
        ref = torch.einsum("nhj,nhjc->nhc", torch.softmax(s, -1), V).reshape(N, d)
        got = o.float().double()
        if planes == 2:
            assert _rel(got, ref) < 1e-5, (t, _rel(got, ref))
        else:                                                                 # bf16 rounding of the output
            assert bool(((got - ref).abs() <= 2.0 ** -8 * ref.abs() + 1e-6 * ref.abs().max()).all()), t


# ------------------------------------------------------------------------------------------------ decode embedding
@pytest.mark.parametrize("d,V", [(128, 512), (256, 257), (512, 512)])
def test_decode_embedding_matches_embed_fwd(d, V):
    """Row t of the step-t embedding equals row t of embed_fwd on the whole prefix (same table, same summation order:
    bitwise), and the carried group index and key validity equal seq_prep's, for prefixes with "m", EOS (and tokens after
    it) and PAD arguments."""
    ops = _ops()
    N, T, na = 5, 40, 11
    cmd_tab, arg_embed = _rand(7, d, seed=1), _rand(V, 64, seed=2)
    W, bias = _rand(d, 64 * na, seed=3, scale=0.05), _rand(d, seed=4)
    pos, grp_tab = _rand(T + 2, d, seed=5), _rand(T + 2, d, seed=6)
    table, base = torch.empty(na * V, d, device=DEV), torch.empty(d, device=DEV)
    ops.embed_fold(arg_embed, W, bias, table, base, V, na, d)
    g = torch.Generator().manual_seed(0)
    cmds = torch.randint(0, 4, (N, T), generator=g)
    cmds[:, 0] = 5                                                            # SOS
    cmds[1, 12] = 4
    cmds[2, 25:] = 4
    cmds[3, 1:] = 0                                                           # "m" only: the group index keeps growing
    cmds[4, 5] = cmds[4, 9] = 4                                               # tokens between and after two EOS
    args = torch.randint(-1, V - 1, (N, T, na), generator=g)
    args = torch.where(_mask().cpu()[cmds], args, torch.full_like(args, -1))
    args[:, 0] = -1
    cf, af = cmds.float().to(DEV), args.float().to(DEV)
    ref_x = torch.empty(N * T, d, device=DEV)
    grp_ref = torch.empty(N * T, dtype=torch.uint8, device=DEV)
    kv_ref = torch.empty(N * T, dtype=torch.uint8, device=DEV)
    ops.seq_prep(cf, N, T, None, None, kv_ref, grp_ref, None)
    ops.embed_fwd(cf, af, grp_ref, cmd_tab, table, base, pos, grp_tab, ref_x, N * T, T, V, na, d, (0.0, 0, 0))
    step = torch.zeros(2, dtype=torch.int32, device=DEV)
    cmd_in = torch.full((N,), 77, dtype=torch.int32, device=DEV)              # ignored at t = 0
    args_in = torch.zeros(N, na, dtype=torch.int32, device=DEV)
    grp = torch.full((N,), 99, dtype=torch.int32, device=DEV)                 # reset at t = 0
    kv = torch.zeros(N, T, dtype=torch.uint8, device=DEV)
    x = torch.empty(N, d, device=DEV)
    for t in range(T):
        step[0] = t
        if t > 0:
            cmd_in.copy_(cmds[:, t])
            args_in.copy_(args[:, t])
        ops.decode_embed(step, cmd_in, args_in, grp, kv, cmd_tab, table, base, pos, grp_tab, x, N, T, V, na, d)
        assert torch.equal(x, ref_x.view(N, T, d)[:, t]), t
        assert torch.equal(grp, grp_ref.view(N, T)[:, t].int()), t
    assert torch.equal(kv, kv_ref.view(N, T))


# ------------------------------------------------------------------------------------------------ sampler
def _sampler_buffers(N, T, na):
    z = lambda *s, dt=torch.int32: torch.zeros(*s, dtype=dt, device=DEV)
    return dict(step=z(2), cmd_in=z(N), args_in=z(N, na), out_cmd=z(N, T, dt=torch.int64),
                out_args=z(N, T, na, dt=torch.int64))


def _sample(b, cl, al, temperature, seed, N, T, na, C):
    _ops().decode_sample(b["step"], cl, al, torch.full((1,), float(temperature), device=DEV),
                         torch.full((1,), seed, dtype=torch.int64, device=DEV), b["cmd_in"], b["args_in"], b["out_cmd"],
                         b["out_args"], N, T, na, C)


@pytest.mark.parametrize("C", [512, 257])
def test_decode_sampler_argmax_matches_torch(C):
    """Below temperature 1e-3: torch.argmax (exact ties to the lowest index) + _make_valid, over several blocks of
    sequences; the tokens land at position t and in the next step's inputs, and t advances by exactly one."""
    N, T, na = 300, 4, 11
    b = _sampler_buffers(N, T, na)
    mask = _mask()
    g = torch.Generator().manual_seed(3)
    for t in range(T):
        cl, al = _rand(N, 7, seed=10 + t), _rand(N, na * C, seed=20 + t)
        rows = torch.arange(0, N, 2)                                          # every other row gets an exact tie
        j = torch.randint(0, 7, (len(rows),), generator=g).to(DEV)
        cl[rows.to(DEV), j] = cl[rows.to(DEV)].max(-1).values
        a3 = al.view(N, na, C)
        jj = torch.randint(0, C, (len(rows), na), generator=g).to(DEV)
        a3[rows.to(DEV)[:, None], torch.arange(na, device=DEV)[None], jj] = a3[rows.to(DEV)].max(-1).values
        _sample(b, cl, al, 1e-4, 0, N, T, na, C)
        c_ref = cl.argmax(-1)
        a_ref = a3.argmax(-1) - 1
        a_ref = torch.where(mask[c_ref], a_ref, torch.full_like(a_ref, -1))
        assert torch.equal(b["out_cmd"][:, t], c_ref) and torch.equal(b["out_args"][:, t], a_ref), t
        assert torch.equal(b["cmd_in"], c_ref.int()) and torch.equal(b["args_in"], a_ref.int()), t
        assert b["step"].tolist() == [t + 1, 0]


@pytest.mark.parametrize("which", ["cmd", "args"])
def test_decode_sampler_gumbel_matches_softmax(which):
    """Gumbel-max at T = 0.7 over 2^16 copies of one row draws from softmax(logits / T): chi-square test on the 7 command
    classes, and on the 512 classes of an argument slot that every sampled command ("m") uses.  The seed is fixed; the
    bound p > 1e-4 then holds or fails deterministically.  The same seed reproduces the draws, another seed changes them."""
    from scipy.stats import chi2
    R, T, na, C, temp = 1 << 16, 1, 11, 512, 0.7
    g = torch.Generator().manual_seed(5)
    cl = torch.zeros(R, 7, device=DEV)
    al = torch.zeros(R, na * C, device=DEV)
    if which == "cmd":
        row = torch.randn(7, generator=g) * 0.8
        cl[:] = row.to(DEV)
    else:
        row = torch.randn(C, generator=g) * 0.5
        cl[:, 0] = 20.0                                                      # "m" with probability 1 - 1e-12
        al.view(R, na, C)[:, 9] = row.to(DEV)
    b = _sampler_buffers(R, T, na)
    _sample(b, cl, al, temp, 12345, R, T, na, C)
    if which == "cmd":
        got = b["out_cmd"][:, 0]
    else:
        assert bool((b["out_cmd"][:, 0] == 0).all())
        got = b["out_args"][:, 0, 9] + 1
    k = row.numel()
    counts = torch.bincount(got, minlength=k).double().cpu()
    expect = torch.softmax(row.double() / temp, 0) * R
    stat = float(((counts - expect) ** 2 / expect).sum())
    assert chi2.sf(stat, k - 1) > 1e-4, (stat, k)
    b2 = _sampler_buffers(R, T, na)
    _sample(b2, cl, al, temp, 12345, R, T, na, C)
    assert torch.equal(b2["out_cmd"], b["out_cmd"]) and torch.equal(b2["out_args"], b["out_args"])
    b3 = _sampler_buffers(R, T, na)
    _sample(b3, cl, al, temp, 54321, R, T, na, C)
    key = "out_cmd" if which == "cmd" else "out_args"
    assert not torch.equal(b3[key], b[key])


# ------------------------------------------------------------------------------------------------ the engine
def _sketch_cfg(**over):
    kw = dict(d_model=128, n_heads=4, dim_feedforward=256, dim_z=64, n_layers=2, n_layers_decode=2, max_num_groups=4,
              max_total_len=30, use_vae=False, pred_mode="autoregressive", rel_targets=True)
    kw.update(over)
    return O.make_cfg("one_stage", **kw)


MODEL_CASES = {
    "sketchformer_d128": None,                                               # the golden case's seeded weights and icons
    "vae_label": dict(use_vae=True, label_condition=True, n_labels=5, dim_label=16, max_total_len=20),
    "hd16": dict(n_heads=8, max_total_len=24),
    "hd64": dict(n_heads=2, max_total_len=24),
    "longest_hd32": dict(max_total_len=LONGEST_T[32]),
}


def _model_case(name, precision, N=3):
    """(cfg, model, params, z [N, 1, 1, dz] on the GPU, label or None)."""
    if MODEL_CASES[name] is None:
        cfg, fx, _ = load_case(name)
        model, _, params = _build(cfg, precision, seed=int(fx["seed_params"]))
        c, a = torch.from_numpy(fx["commands"])[:N].to(DEV), torch.from_numpy(fx["args"])[:N].to(DEV)
        with torch.no_grad():
            z = model(c, a, None, None, encode_mode=True).permute(2, 0, 1, 3).contiguous()
        return cfg, model, params, z, None
    cfg = _sketch_cfg(**MODEL_CASES[name])
    model, _, params = _build(cfg, precision, seed=11)
    z = _rand(N, 1, 1, cfg.dim_z, seed=12)
    label = torch.arange(N, device=DEV) % cfg.n_labels if cfg.label_condition else None
    return cfg, model, params, z, label


def _run_engine(model, z, label):
    """greedy_sample through the cached engine; returns the per-step logits and the decoded (relative) tokens."""
    logs = []
    model._decode_hook = lambda t, c, a: logs.append((t, c.clone(), a.clone()))
    try:
        model.greedy_sample(z=z, label=label, concat_groups=False)
    finally:
        model._decode_hook = None
    assert [t for t, _, _ in logs] == list(range(len(logs)))
    lc = torch.stack([c for _, c, _ in logs], 1)                            # [N, T, 7]
    la = torch.stack([a for _, _, a in logs], 1)                            # [N, T, 11 * C]
    return lc, la, model._ds.out_cmd.clone(), model._ds.out_args.clone()


def _prefix(cy, ay, n_keep):
    """[SOS, y_1 .. y_n_keep] as the float (N, 1, n_keep + 1[, 11]) decoder inputs."""
    N = cy.shape[0]
    c = torch.cat([torch.full((N, 1), 5, dtype=cy.dtype, device=cy.device), cy[:, :n_keep]], 1)
    a = torch.cat([torch.full((N, 1, 11), -1, dtype=ay.dtype, device=ay.device), ay[:, :n_keep]], 1)
    return c.float().unsqueeze(1), a.float().unsqueeze(1)


def _oracle_logits(params, cfg, z, label, cy, ay):
    """fp64 oracle teacher-forced on [SOS, y_1 .. y_T]: logits [N, T, 7], [N, T, 11, C]."""
    T = cy.shape[1]
    cd, ad = _prefix(cy.cpu(), ay.cpu(), T)
    p64 = {k: v.double() for k, v in params.items()}
    zo = O.forward(p64, cfg, cd.double(), ad.double(), label=None if label is None else label.cpu(),
                   z_in=z.reshape(z.shape[0], -1).double().cpu())
    return zo["command_logits"][:, 0], zo["args_logits"][:, 0]


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("name", list(MODEL_CASES))
def test_decode_logits_match_full_forward_and_oracle(name, precision):
    cfg, model, params, z, label = _model_case(name, precision)
    lc, la, cy, ay = _run_engine(model, z, label)
    N, T = cy.shape
    C = O.out_args_dim(cfg)
    la = la.view(N, T, cfg.n_args, C)
    oc, oa = _oracle_logits(params, cfg, z, label, cy, ay)
    if precision == "bf16x3":
        with torch.no_grad():                                                # teacher-forced full forward, same precision
            cd, ad = _prefix(cy, ay, T - 1)
            res = model(None, None, cd, ad, label=label, z=z, return_tgt=False)
        np.testing.assert_allclose(lc.cpu().numpy(), res["command_logits"][:, 0].cpu().numpy(), rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(la.cpu().numpy(), res["args_logits"][:, 0].cpu().numpy(), rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(lc.double().cpu().numpy(), oc.numpy(), rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(la.double().cpu().numpy(), oa.numpy(), rtol=1e-3, atol=1e-4)
    else:
        assert _rel(lc.double().cpu(), oc) < 5e-2, _rel(lc.double().cpu(), oc)
        assert _rel(la.double().cpu(), oa) < 5e-2, _rel(la.double().cpu(), oa)


@pytest.mark.parametrize("N", [1, 5, 300])
def test_decode_tokens_match_forward_loop(N):
    """bf16x3: the engine's tokens equal those of an explicit model.forward decoding loop (as in
    test_sketchformer_greedy_decoding_is_self_consistent).  Where a sequence's tokens part, the step at which they first
    differ must be a near tie: the fp64 oracle's top-2 margin there is at most 1e-3."""
    cfg, fx, _ = load_case("sketchformer_d128")
    model, _, params = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    z = _rand(N, 1, 1, cfg.dim_z, seed=N)
    T = cfg.max_total_len
    _, _, cy, ay = _run_engine(model, z, None)
    lc_ = torch.full((N, 1, 1), 5, dtype=torch.long, device=DEV)
    la_ = torch.full((N, 1, 1, 11), -1, dtype=torch.long, device=DEV)
    with torch.no_grad():
        for _ in range(T):
            res = model(None, None, lc_.float(), la_.float(), z=z, return_tgt=False)
            cn, an = res["command_logits"].argmax(-1), res["args_logits"].argmax(-1) - 1
            _, an = model._make_valid(cn, an)
            lc_, la_ = torch.cat([lc_, cn[..., -1:]], -1), torch.cat([la_, an[..., -1:, :]], -2)
    fc, fa = lc_[:, 0, 1:], la_[:, 0, 1:]
    same = (fc == cy) & (fa == ay).all(-1)                                  # [N, T]
    if bool(same.all()):
        return
    oc, oa = _oracle_logits(params, cfg, z, None, cy, ay)
    m2 = lambda x: (lambda v: v[..., 0] - v[..., 1])(x.topk(2, -1).values)
    mc, ma = m2(oc), m2(oa)                                                 # [N, T], [N, T, 11]
    used = O.CMD_ARGS_MASK[cy.cpu()].bool()
    for n in torch.nonzero(~same.all(-1)).flatten().tolist():
        t = int(torch.nonzero(~same[n]).min())
        if fc[n, t] != cy[n, t]:
            assert mc[n, t] <= 1e-3, (n, t, float(mc[n, t]))
        else:
            k = (fa[n, t] != ay[n, t]).cpu() & used[n, t]
            assert bool((ma[n, t][k] <= 1e-3).all()), (n, t, ma[n, t][k])
    assert same.all(-1).float().mean().item() > 0.9


# ------------------------------------------------------------------------------------------------ graphs
def test_decode_graph_replays_match_eager_launches():
    """graphs=True and graphs=False decode the same tokens; a FusedAdamW step between two calls changes the replayed
    graph's result exactly as it changes the eager result; consecutive calls with different N work."""
    from deepsvg_b200 import FusedAdamW
    cfg, fx, _ = load_case("sketchformer_d128")
    mg, _, _ = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    me, _, _ = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    mg.graphs, me.graphs = True, False
    z = _rand(6, 1, 1, cfg.dim_z, seed=1)
    first = mg.greedy_sample(z=z, concat_groups=False)
    graph = mg._ds.graph
    again = mg.greedy_sample(z=z, concat_groups=False)                      # replays from t = 0
    ref = me.greedy_sample(z=z, concat_groups=False)
    assert graph is not None and me._ds.graph is None
    for a, b, c in zip(first, again, ref):
        assert torch.equal(a, c) and torch.equal(b, c)
    for m in (mg, me):
        g = torch.Generator().manual_seed(0)
        for p in m.parameters():
            p.grad = (torch.randn(p.shape, generator=g) * 0.1).to(DEV)
        FusedAdamW(m.parameters(), lr=3e-2).step()
    after = mg.greedy_sample(z=z, concat_groups=False)
    assert mg._ds.graph is graph                                            # same capture, refreshed weights
    ref2 = me.greedy_sample(z=z, concat_groups=False)
    assert torch.equal(after[0], ref2[0]) and torch.equal(after[1], ref2[1])
    assert not (torch.equal(after[0], first[0]) and torch.equal(after[1], first[1]))
    for N in (3, 7, 3):
        zn = _rand(N, 1, 1, cfg.dim_z, seed=N)
        a, b = mg.greedy_sample(z=zn, concat_groups=False), me.greedy_sample(z=zn, concat_groups=False)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), N
        assert mg._ds.graph is not None


def test_decode_sampling_is_reproducible_with_manual_seed():
    """temperature >= 1e-3 samples; torch.manual_seed before the call reproduces it, in graph mode and eagerly."""
    cfg, fx, _ = load_case("sketchformer_d128")
    model, _, _ = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    z = _rand(16, 1, 1, cfg.dim_z, seed=2)
    outs = []
    for graphs in (True, True, False):
        model.graphs = graphs
        torch.manual_seed(4)
        outs.append(model.greedy_sample(z=z, concat_groups=False, temperature=1.0))
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1])
    torch.manual_seed(5)
    other = model.greedy_sample(z=z, concat_groups=False, temperature=1.0)
    assert not torch.equal(other[0], outs[0][0])


# ------------------------------------------------------------------------------------------------ dispatch
def test_decode_dispatch_by_training_flag():
    """Eval mode decodes with decode_attn_kernel and launches no whole-sequence attention kernel; train mode keeps the
    prefix loop (attention over the whole prefix) and launches no decode kernel."""
    cfg, fx, _ = load_case("sketchformer_d128")
    model, _, _ = _build(cfg, "bf16x3", seed=int(fx["seed_params"]))
    model.graphs = False
    z = _rand(2, 1, 1, cfg.dim_z, seed=3)
    keys = {kernel_key(n) for n in launched_kernels(lambda: model.greedy_sample(z=z))} - {None}
    assert "decode_attn_kernel<32, 2>" in keys and {"decode_embed_kernel<1>", "decode_sample_kernel"} <= keys, keys
    assert not [k for k in keys if k.startswith("attn_")], keys
    model.train()
    keys = {kernel_key(n) for n in launched_kernels(lambda: model.greedy_sample(z=z))} - {None}
    assert not [k for k in keys if k.startswith("decode_")], keys
    assert [k for k in keys if k.startswith("attn_")], keys
