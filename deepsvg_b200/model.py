"""`SVGTransformer`: drop-in for deepsvg.model.model.SVGTransformer (model.py:288-412) on the accelerated path.

Same constructor (`SVGTransformer(model_cfg)`), forward signature, result-dict keys and `state_dict` names/shapes as the
reference, so `deepsvg/train.py` runs unchanged (SURVEY.md 8b).  Parameters are ordinary fp32 `nn.Parameter`s; the
arithmetic is one `torch.autograd.Function` whose forward and backward are sequences of libdsvg_b200 kernel launches
(wgmma GEMMs, fused LayerNorm / attention / embedding / loss kernels) on torch's current CUDA stream.  There is no
CPU or eager-PyTorch fallback: without the CUDA library, or with CPU tensors, forward raises.

Internal layout is token-major `(icon n, path g, position s)` -- the reference's `_make_seq_first` / `_pack_group_batch`
permutations (utils/utils.py:20-49) never happen; logits land directly at `[n, g, s, ...]`.

Precision: "bf16" (fast: single-plane bf16 operands, fp32 accumulate) or "bf16x3" (parity: split hi/lo operands, three
tensor-core products per K step, ~fp32 accuracy on the same kernels).  Select with `SVGTransformer(cfg, precision=...)`
or env DSVG_PRECISION.
"""
import math
import os

import torch
import torch.nn as nn

from . import ops
from .config import check_supported
from .ops import Act

CMD_ARGS_MASK = torch.tensor([[0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1],   # m      (difflib/tensor.py:15-21)
                              [0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1],   # l
                              [0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1],   # c
                              [1, 1, 1, 1, 1, 0, 0, 0, 0, 1, 1],   # a
                              [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0],   # EOS
                              [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0],   # SOS
                              [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0]])  # z


def _r8(n):
    return (n + 7) // 8 * 8


# ======================================================================================================
# parameter inventory (names / shapes / initialisers of the reference module tree, SURVEY.md 8b)
# ======================================================================================================
def _param_specs(cfg):
    """[(name, shape, init kind)] in the reference's registration order.  init kinds:
    kaiming (model.py:38-44), xavier (attention.py:85-95), linw/linb (nn.Linear defaults), zeros, ones, vae."""
    d, dz, ff = cfg.d_model, cfg.dim_z, cfg.dim_feedforward
    two = cfg.encode_stages == 2
    S = []

    def lin(n, o, i):
        S.append((n + ".weight", (o, i), "linw"))
        S.append((n + ".bias", (o,), "linb:%d" % i))

    def ln(n):
        S.append((n + ".weight", (d,), "ones"))
        S.append((n + ".bias", (d,), "zeros"))

    def layer(p, glob):
        S.append((p + ".self_attn.in_proj_weight", (3 * d, d), "xavier"))
        S.append((p + ".self_attn.in_proj_bias", (3 * d,), "zeros"))
        S.append((p + ".self_attn.out_proj.weight", (d, d), "linw"))
        S.append((p + ".self_attn.out_proj.bias", (d,), "zeros"))
        if glob:
            lin(p + ".linear_global", d, dz)
        if cfg.label_condition:
            lin(p + ".linear_global2", d, cfg.dim_label)
        lin(p + ".linear1", ff, d)
        lin(p + ".linear2", d, ff)
        ln(p + ".norm1")
        ln(p + ".norm2")

    def stack(p, n, glob):
        for i in range(n):
            layer("%s.layers.%d" % (p, i), glob)
        ln(p + ".norm")

    enc_len = cfg.max_seq_len if two else cfg.max_total_len
    S.append(("encoder.embedding.command_embed.weight", (cfg.n_commands, d), "kaiming"))
    S.append(("encoder.embedding.arg_embed.weight", (cfg.args_dim + 1, 64), "kaiming"))
    S.append(("encoder.embedding.embed_fcn.weight", (d, 64 * cfg.n_args), "kaiming"))
    S.append(("encoder.embedding.embed_fcn.bias", (d,), "linb:%d" % (64 * cfg.n_args)))
    if not two:
        S.append(("encoder.embedding.group_embed.weight", (cfg.max_num_groups + 2, d), "kaiming"))
    S.append(("encoder.embedding.pos_encoding.pos_embed.weight", (enc_len + 2, d), "kaiming"))
    if cfg.label_condition:
        S.append(("encoder.label_embedding.label_embedding.weight", (cfg.n_labels, cfg.dim_label), "kaiming"))
    stack("encoder.encoder", cfg.n_layers, False)
    if two:
        if not getattr(cfg, "self_match", False):        # model.py:114-115: no positional code over paths when self-matching
            S.append(("encoder.hierarchical_PE.pos_embed.weight", (cfg.max_num_groups, d), "kaiming"))
        stack("encoder.hierarchical_encoder", cfg.n_layers, False)
    if cfg.use_resnet:
        for i in range(1, 5):
            lin("resnet.linear%d.0" % i, d, d)
    if cfg.use_vae:
        for n in ("vae.enc_mu_fcn", "vae.enc_sigma_fcn"):
            S.append((n + ".weight", (dz, d), "vae"))
            S.append((n + ".bias", (dz,), "zeros"))
    else:
        lin("bottleneck.bottleneck", dz, d)
    if cfg.label_condition:
        S.append(("decoder.label_embedding.label_embedding.weight", (cfg.n_labels, cfg.dim_label), "kaiming"))
    if two:
        S.append(("decoder.hierarchical_embedding.PE.pos_embed.weight", (cfg.num_groups_proposal, d), "kaiming"))
        stack("decoder.hierarchical_decoder", cfg.n_layers_decode, True)
        lin("decoder.hierarchical_fcn.visibility_fcn", 2, d)
        lin("decoder.hierarchical_fcn.z_fcn", dz, d)
    dec_len = (cfg.max_seq_len if two else cfg.max_total_len) + 1
    out_classes = 2 * cfg.args_dim if getattr(cfg, "rel_targets", False) else cfg.args_dim + 1     # model.py:37,233
    if getattr(cfg, "pred_mode", "one_shot") == "autoregressive":        # model.py:218-222: SVGEmbedding of the shifted targets
        S.append(("decoder.embedding.command_embed.weight", (cfg.n_commands, d), "kaiming"))
        S.append(("decoder.embedding.arg_embed.weight", (out_classes, 64), "kaiming"))
        S.append(("decoder.embedding.embed_fcn.weight", (d, 64 * cfg.n_args), "kaiming"))
        S.append(("decoder.embedding.embed_fcn.bias", (d,), "linb:%d" % (64 * cfg.n_args)))
        S.append(("decoder.embedding.group_embed.weight", (cfg.max_total_len + 2, d), "kaiming"))
        S.append(("decoder.embedding.pos_encoding.pos_embed.weight", (cfg.max_total_len + 2, d), "kaiming"))
    else:
        S.append(("decoder.embedding.PE.pos_embed.weight", (dec_len, d), "kaiming"))
    stack("decoder.decoder", cfg.n_layers_decode, True)
    lin("decoder.fcn.command_fcn", cfg.n_commands, d)
    lin("decoder.fcn.args_fcn", cfg.n_args * out_classes, d)
    return S


def _init_tensor(shape, kind):
    t = torch.empty(*shape)
    if kind == "kaiming":
        nn.init.kaiming_normal_(t, mode="fan_in")
    elif kind == "xavier":
        nn.init.xavier_uniform_(t)
    elif kind == "linw":
        nn.init.kaiming_uniform_(t, a=math.sqrt(5))
    elif kind.startswith("linb:"):
        b = 1.0 / math.sqrt(int(kind[5:]))
        nn.init.uniform_(t, -b, b)
    elif kind == "zeros":
        t.zero_()
    elif kind == "ones":
        t.fill_(1.0)
    elif kind == "vae":
        nn.init.normal_(t, std=0.001)
    else:
        raise ValueError(kind)
    return t


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference's dotted parameter paths."""


def _register(root, dotted, tensor, is_buffer=False):
    parts = dotted.split(".")
    m = root
    for p in parts[:-1]:
        if p not in m._modules:
            m.add_module(p, _Node())
        m = m._modules[p]
    if is_buffer:
        m.register_buffer(parts[-1], tensor)
    else:
        m.register_parameter(parts[-1], nn.Parameter(tensor))


# ======================================================================================================
# saved state of one forward call
# ======================================================================================================
class _Saved:
    """Everything the backward pass (and the fused loss) needs; one instance per forward call."""

    def __init__(self):
        self.layers = {}
        self.t = {}


class LossHandle:
    """Side channel between SVGTransformer's autograd node and SVGLoss (attached to the logits tensors).
    The loss kernels leave unit-scale d(loss)/d(logits) in `dl_*` (act tensors) and the per-term upstream scales in
    `scales` (device float[4]: args, cmd, visibility, kl); the model's backward consumes them directly."""

    def __init__(self, token):
        # NOTE: no reference back to the _Saved state: a _Saved <-> LossHandle cycle would keep ~10 GB of activations
        # alive until Python's cyclic GC runs, which defeats the caching allocator (measured: 238 cudaMallocs and
        # 20-350 ms stalls inside a 40-step timed region).
        self.token = token
        self.dl_args = self.dl_cmd = self.dl_vis = None
        self.scales = None
        self.loss_out = None
        self.used = False
        self.bufs = None          # CUDA-graph mode: static buffers SVGLoss writes into (see _GraphState)
        self.tgt_prep = None      # data-parallel mode: target bookkeeping + globally reduced counts, started before the forward


class _SVGFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, inputs, token, *params):
        ctx.set_materialize_grads(False)
        outs, saved = model._run_forward(inputs)
        ctx.model, ctx.saved = model, saved
        ctx.gen = getattr(saved, "gen", 0)
        saved.token = token
        ctx.n_outs = len(outs)
        return tuple(outs) + (token.detach().clone(),)

    @staticmethod
    def backward(ctx, *grads):
        model, saved = ctx.model, ctx.saved
        flat = model._run_backward(saved, grads[:-1], grads[-1], ctx.gen)
        return (None, None, None) + tuple(flat)


# ======================================================================================================
class SVGTransformer(nn.Module):
    def __init__(self, cfg, precision=None, process_group=None, graphs=None):
        super().__init__()
        check_supported(cfg)
        self.cfg = cfg
        # CUDA graphs: by default the train-mode step (forward; backward in two halves) is captured once the same input
        # signature has been seen on three consecutive calls and replayed from then on (~400 kernel launches per step
        # become three graph launches); graphs=False never captures.  Env DSVG_GRAPHS=0 / 1 sets the default.
        if graphs is None:
            graphs = os.environ.get("DSVG_GRAPHS", "1") != "0"
        self.graphs = bool(graphs)
        self._aligned = None       # DataParallel replicas: aligned stand-ins of the broadcast parameter views
        self._gs = None            # the one live _GraphState
        self.graph_kernel_launches = 0   # kernels launched through graph replays (the library's own counter sees captures only)
        self._gs_streak = (None, 0)
        self.rel_targets = bool(getattr(cfg, "rel_targets", False))
        self.autoregressive = getattr(cfg, "pred_mode", "one_shot") == "autoregressive"
        self.args_dim = 2 * cfg.args_dim if self.rel_targets else cfg.args_dim + 1      # model.py:293
        self.precision = precision or os.environ.get("DSVG_PRECISION", "bf16")
        if self.precision not in ("bf16", "bf16x3"):
            raise ValueError("precision must be 'bf16' or 'bf16x3'")
        self.process_group = process_group                    # set => gradients are all-reduced (SUM) in backward
        self._specs = _param_specs(cfg)
        two = cfg.encode_stages == 2
        first_layer = {}
        for name, shape, kind in self._specs:
            t = _init_tensor(shape, kind)
            # transformer.py:383-384: _get_clones deep-copies => all layers of a stack start identical
            if ".layers." in name:
                stack, rest = name.split(".layers.")
                idx, leaf = rest.split(".", 1)
                key = stack + "|" + leaf
                if idx == "0":
                    first_layer[key] = t
                else:
                    t = first_layer[key].clone()
            _register(self, name, t)
        enc_len = (cfg.max_seq_len if two else cfg.max_total_len) + 2
        dec_len = (cfg.max_seq_len if two else cfg.max_total_len) + 1
        pos = lambda n: torch.arange(0, n, dtype=torch.long).unsqueeze(1)   # positional_encoding.py:30-31
        _register(self, "encoder.embedding.pos_encoding.position", pos(enc_len), True)
        self.self_match = bool(getattr(cfg, "self_match", False))
        if two:
            if not self.self_match:
                _register(self, "encoder.hierarchical_PE.position", pos(cfg.max_num_groups), True)
            _register(self, "decoder.hierarchical_embedding.PE.position", pos(cfg.num_groups_proposal), True)
        if self.autoregressive:
            _register(self, "decoder.embedding.pos_encoding.position", pos(cfg.max_total_len + 2), True)
            n = cfg.max_total_len + 1                                     # model/utils.py:69-72, registered at model.py:221-222
            _register(self, "decoder.square_subsequent_mask",
                      torch.zeros(n, n).masked_fill(torch.triu(torch.ones(n, n, dtype=torch.bool), 1), float("-inf")), True)
        else:
            _register(self, "decoder.embedding.PE.position", pos(dec_len), True)
        self.register_buffer("cmd_args_mask", CMD_ARGS_MASK.clone())       # model.py:309
        self._pnames = [n for n, _, _ in self._specs]
        self._sites = {}
        self._wcache = {}
        self._eps_override = None      # tests inject the VAE noise here (SURVEY.md 8c hazard 2)
        self._ds = None                # the one live _DecodeState (cached autoregressive decoding)
        self._decode_hook = None       # tests: called as hook(t, cmd_logits [N, 7], args_logits [N, 11 * C]) after each step

    # -------------------------------------------------------------------------------------------------
    def _param(self, name):
        al = self.__dict__.get("_aligned")
        if al is not None:
            return al[name]
        m = self
        for p in name.split("."):
            if p in m._modules:
                m = m._modules[p]
            elif p in m._parameters:
                m = m._parameters[p]
            else:
                # nn.DataParallel replicas (train.py:74 on several GPUs): replicate() empties `_parameters` and sets the
                # broadcast copies as plain attributes
                m = getattr(m, p)
        return m

    def _pdict(self):
        return {n: self._param(n) for n in self._pnames}

    def _site(self, tag):
        if tag not in self._sites:
            self._sites[tag] = len(self._sites) + 1
        return self._sites[tag]

    @property
    def planes(self):
        return 2 if self.precision == "bf16x3" else 1

    # -------------------------------------------------------------------------------------------------
    def forward(self, commands_enc, args_enc, commands_dec, args_dec, label=None, z=None, hierarch_logits=None,
                return_tgt=True, params=None, encode_mode=False, return_hierarch=False):
        """model.py:352-412.  Tensors are batch-first float32 CUDA tensors: commands (N, G, S+2), args (N, G, S+2, 11)."""
        cfg = self.cfg
        if hierarch_logits is not None:
            # model.py:246-259: the per-path stage was run before (return_hierarch=True); `z` now holds the PER-PATH latents,
            # batch-first (N, Gp, 1, dz), and hierarch_logits the visibility logits as that call returned them (1, Gp, N, 2)
            if z is None or cfg.decode_stages != 2 or torch.is_grad_enabled() and z.requires_grad:
                raise ValueError("forward(hierarch_logits=...) needs the two-stage model, z = per-path latents, and no grad")
        if z is None and (commands_enc is None or args_enc is None):
            raise ValueError("encoder inputs are required when z is not given")
        ref = commands_enc if commands_enc is not None else z
        if not ref.is_cuda:
            raise RuntimeError("deepsvg_b200 has no CPU path: inputs and parameters must live on a CUDA device")
        if cfg.label_condition:
            if label is None:
                raise ValueError("label_condition=True needs `label`")
            # the kernels read `const long long*` through a raw pointer: normalise dtype / device / layout here
            label = label.to(device=ref.device, dtype=torch.long).contiguous().view(-1)
            if label.numel() != ref.shape[0]:
                raise ValueError("label must hold one class id per icon (%d), got %d" % (ref.shape[0], label.numel()))
            if os.environ.get("DSVG_DEBUG_CHECKS") and (int(label.min()) < 0 or int(label.max()) >= cfg.n_labels):
                raise ValueError("label ids must lie in [0, n_labels)")
        inputs = dict(commands=commands_enc, args=args_enc, label=label, z=z, encode_mode=encode_mode,
                      return_hierarch=return_hierarch, training=self.training, hierarch_logits=hierarch_logits)
        if self.autoregressive and not encode_mode:
            if commands_dec is None or args_dec is None:
                raise ValueError("the autoregressive decoder needs its input tokens (commands_dec, args_dec)")
            cd, ad = commands_dec.detach().float(), args_dec.detach().float()
            if return_tgt:                                   # teacher forcing: the last position is only a target (model.py:372)
                cd, ad = cd[..., :-1], ad[..., :-1, :]
            inputs["dec_inputs"] = (cd.contiguous(), ad.contiguous())
        if self.self_match and return_tgt and not encode_mode and not return_hierarch:   # model.py:384
            if commands_dec is None or args_dec is None:
                raise ValueError("self_match needs the decoder targets (commands_dec, args_dec)")
            inputs["match_targets"] = (commands_dec.detach().contiguous().float(), args_dec.detach().contiguous().float())
        self._aligned = None
        plist = [self._param(n) for n in self._pnames]
        if any(p.data_ptr() % 16 for p in plist):
            # nn.DataParallel replica: its parameters are views into one coalesced broadcast buffer and only 4-byte aligned;
            # the kernels read parameters with 16-byte vector loads.  Differentiable aligned copies stand in for them.
            plist = [p if p.data_ptr() % 16 == 0 else p.clone() for p in plist]
            self._aligned = dict(zip(self._pnames, plist))
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in plist)
        token = torch.zeros((), device=ref.device, requires_grad=need_grad)
        need_grad = need_grad and not return_hierarch and hierarch_logits is None   # inference-only exits
        inputs["need_grad"] = need_grad
        tgt_prep = None
        if need_grad and self.process_group is not None and return_tgt and commands_dec is not None and not encode_mode:
            tgt_prep = self._prep_targets(commands_dec)
        if need_grad:
            outs = _SVGFunction.apply(self, inputs, token, *plist)
            outs, tok_out = outs[:-1], outs[-1]
        else:
            with torch.no_grad():
                outs, _ = self._run_forward(inputs)
            tok_out = None
        saved, self._last_saved = self._last_saved, None     # do not pin the activations on the module
        N = ref.shape[0]
        if encode_mode:
            return outs[0].view(1, 1, N, cfg.dim_z)            # seq-first like model.py:371 (reference quirk, 3.4)
        two = cfg.decode_stages == 2
        if return_hierarch:
            Gp = cfg.num_groups_proposal
            return outs[0].view(N, Gp, 2).permute(1, 0, 2).unsqueeze(0), outs[1].view(N, Gp, -1).permute(1, 0, 2).unsqueeze(0)
        G = cfg.num_groups_proposal if two else 1
        Ld = (cfg.max_seq_len if two else cfg.max_total_len) + 1
        if self.autoregressive:
            Ld = inputs["dec_inputs"][0].shape[-1]
        it = iter(outs)
        res = {"command_logits": next(it).view(N, G, Ld, cfg.n_commands),
               "args_logits": next(it).view(N, G, Ld, cfg.n_args, self.args_dim)}
        if two:
            res["visibility_logits"] = next(it).view(N, G, 1, 2)
        if return_tgt:
            res["tgt_commands"] = commands_dec
            res["tgt_args"] = args_dec
            if cfg.use_vae and z is None:
                res["mu"] = next(it).view(N, 1, 1, cfg.dim_z)
                res["logsigma"] = next(it).view(N, 1, 1, cfg.dim_z)
        if tok_out is not None:
            handle = LossHandle(tok_out)
            handle.planes, handle.process_group = self.planes, self.process_group
            handle.bufs = getattr(saved, "loss_bufs", None)     # graph mode: the loss writes into static buffers
            handle.tgt_prep = tgt_prep
            saved.handle = handle
            for k in ("command_logits", "args_logits"):
                res[k]._dsvg_handle = handle
        return res

    def _prep_targets(self, commands_dec):
        """Data-parallel runs: the masked-CE normalisers are GLOBAL counts (SURVEY.md 8e; loss.py:53-54 under train.py:74).
        They depend only on the targets, so their all-reduce is issued here, before the forward, on NCCL's own stream --
        SVGLoss waits for it ~a forward pass later instead of stalling every rank in the middle of the step."""
        import torch.distributed as dist
        tc = commands_dec.detach().contiguous().float()
        nseq, L = tc.shape[0] * tc.shape[1], tc.shape[2]
        dev = tc.device
        first_eos = torch.empty(nseq, dtype=torch.int32, device=dev)
        visible = torch.empty(nseq, dtype=torch.uint8, device=dev)
        counts = torch.zeros(2, device=dev)
        ops.seq_prep(tc, nseq, L, first_eos, visible, None, None, counts)
        work = dist.all_reduce(counts, op=dist.ReduceOp.SUM, group=self.process_group, async_op=True)
        return dict(src=commands_dec, tc=tc, first_eos=first_eos, visible=visible, counts=counts, work=work)

    # -------------------------------------------------------------------------------------------------
    # inference exit (SURVEY.md 8f rank 1): what cfg.visualize (default_icons.py:79-97), the notebooks and the GUI call
    # -------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def greedy_sample(self, commands_enc=None, args_enc=None, commands_dec=None, args_dec=None, label=None, z=None,
                      hierarch_logits=None, concat_groups=True, temperature=0.0001):
        """One-shot decoding (model.py:414-423): logits -> tokens -> validity masking.  The logits come from the CUDA
        forward; the token post-processing below is a handful of tiny torch ops (not on the train-step hot path).
        At the reference's default temperature (1e-4) `Categorical(logits / T).sample()` is an argmax up to exact
        ties; temperatures below 1e-3 therefore take the deterministic argmax, larger ones sample."""
        def pick(logits):
            if temperature < 1e-3:
                return logits.argmax(dim=-1)
            return torch.distributions.Categorical(logits=logits / temperature).sample()

        if self.autoregressive:
            if self.training:
                return self._greedy_sample_autoregressive(commands_enc, args_enc, label, z, pick, concat_groups)
            return self._greedy_sample_cached(commands_enc, args_enc, label, z, temperature, concat_groups)
        res = self.forward(commands_enc, args_enc, commands_dec, args_dec, label=label, z=z,
                           hierarch_logits=hierarch_logits, return_tgt=False)

        commands_y = pick(res["command_logits"])
        args_y = pick(res["args_logits"]) - 1                               # shift back: class 0 is the -1 PAD value
        visible = None
        if self.cfg.decode_stages == 2:                                    # _threshold_sample, model/utils.py:82-84
            visible = torch.softmax(res["visibility_logits"], dim=-1)[..., 1].squeeze(-1) > 0.7
        commands_y, args_y = self._make_valid(commands_y, args_y, visible)
        if concat_groups:                                                   # keep tokens before each path's first EOS
            n = commands_y.size(0)
            keep = (commands_y == 4).cumsum(dim=-1) == 0
            commands_y = commands_y[keep].reshape(n, -1)
            args_y = args_y[keep].reshape(n, -1, self.cfg.n_args)
        return commands_y, args_y

    def _greedy_sample_autoregressive(self, commands_enc, args_enc, label, z, pick, concat_groups):
        """model.py:428-448 in train mode: token-by-token decoding that re-runs the causal decoder on the whole prefix at
        every step, as the reference does, keeps the last position's tokens, and feeds them back.  The reference's loop
        draws fresh dropout masks over the whole prefix at every step, so earlier positions' keys and values change from
        step to step and a cache cannot reproduce it; eval mode runs _greedy_sample_cached instead."""
        cfg = self.cfg
        if z is None:
            z = self.forward(commands_enc, args_enc, None, None, label=label, encode_mode=True)      # (1, 1, N, dz)
            z = z.permute(2, 0, 1, 3)                                                                # batch-first for z=
        N, dev = z.shape[0], z.device
        commands_y = torch.full((N, 1, 1), 5, dtype=torch.long, device=dev)                          # SOS
        args_y = torch.full((N, 1, 1, cfg.n_args), -1, dtype=torch.long, device=dev)
        for _ in range(cfg.max_total_len):
            res = self.forward(None, None, commands_y.float(), args_y.float(), label=label, z=z, return_tgt=False)
            c_new = pick(res["command_logits"])
            a_new = pick(res["args_logits"]) - 1                                                     # shift back: class 0 = PAD
            _, a_new = self._make_valid(c_new, a_new)
            commands_y = torch.cat([commands_y, c_new[..., -1:]], dim=-1)
            args_y = torch.cat([args_y, a_new[..., -1:, :]], dim=-2)
        commands_y, args_y = commands_y[..., 1:], args_y[..., 1:, :]                                 # discard SOS
        return self._autoregressive_output(commands_y, args_y, concat_groups)

    def _autoregressive_output(self, commands_y, args_y, concat_groups):
        """Decoded tokens (N, 1, T[, 11]) in the classes the heads predict -> the public result (model.py:440-448)."""
        cfg = self.cfg
        if self.rel_targets:
            args_y = self._make_absolute(commands_y, args_y)
        if concat_groups:
            n = commands_y.size(0)
            keep = (commands_y == 4).cumsum(dim=-1) == 0
            commands_y = commands_y[keep].reshape(n, -1)
            args_y = args_y[keep].reshape(n, -1, cfg.n_args)
        return commands_y, args_y

    # -------------------------------------------------------------------------------------------------
    # cached autoregressive decoding (eval mode): csrc/decode.cu
    # -------------------------------------------------------------------------------------------------
    def _greedy_sample_cached(self, commands_enc, args_enc, label, z, temperature, concat_groups):
        """model.py:428-448 with key/value caches.  Position t's decoder output depends on tokens <= t only (causal mask),
        so each step embeds the one new token per sequence, pushes that row through the stack (attention over the cached
        keys and values of positions 0..t) and samples the next tokens on the device: max_total_len steps of N rows instead
        of prefixes of up to max_total_len rows.  With self.graphs, one step is captured as a CUDA graph and replayed.

        Device memory of the caches: n_layers_decode * N * max_total_len * 2 d_model * planes * 2 bytes (4 layers, N = 512,
        max_total_len 139, d_model 256, two planes: 0.58 GB), plus N * max_total_len * 12 int64 tokens."""
        cfg = self.cfg
        if z is None:
            z = self.forward(commands_enc, args_enc, None, None, label=label, encode_mode=True)       # (1, 1, N, dz)
            z = z.permute(2, 0, 1, 3)                                                                 # batch-first
        if not z.is_cuda:
            raise RuntimeError("deepsvg_b200 has no CPU path: inputs and parameters must live on a CUDA device")
        N, dev, T = z.shape[0], z.device, cfg.max_total_len
        if cfg.label_condition:
            if label is None:
                raise ValueError("label_condition=True needs `label`")
            label = label.to(device=dev, dtype=torch.long).contiguous().view(-1)
            if label.numel() != N:
                raise ValueError("label must hold one class id per icon (%d), got %d" % (N, label.numel()))
        key = (N, self.planes, str(dev), hash(tuple(self._param(n).data_ptr() for n in self._pnames)))
        st = self._ds
        if st is None or st.key != key:
            self._ds = None                       # at most one set of caches and one decode graph pool alive
            st = self._ds = _DecodeState(self, key, N, dev)
        # ---- per call: weight operands, folded embedding table, per-layer row vectors, sampling parameters ----
        P = self._param
        sv = st.sv
        for name in st.weights:
            self._pack(name)
        ops.embed_fold(P("decoder.embedding.arg_embed.weight"), P("decoder.embedding.embed_fcn.weight"),
                       P("decoder.embedding.embed_fcn.bias"), st.table, st.base, self.args_dim, cfg.n_args, cfg.d_model)
        z_act = Act(N, cfg.dim_z, self.planes, dev)
        ops.cast_act(z.reshape(N, cfg.dim_z).contiguous().float(), N, cfg.dim_z, out=z_act)
        lab_d = None
        if cfg.label_condition:
            lab_d = Act(N, cfg.dim_label, self.planes, dev)
            ops.gather_rows(P("decoder.label_embedding.label_embedding.weight"), label, N, cfg.dim_label, lab_d)
        for i, rv in enumerate(st.rowvec):                           # improved_transformer.py:131-136, fixed over the steps
            rv.copy_(self._globals_fwd(sv, "decoder.decoder.layers.%d" % i, z_act, N, lab_d, 1))
        st.temperature.fill_(float(temperature))
        if temperature >= 1e-3:
            st.seed.random_()                                         # torch's CUDA generator: manual_seed reproduces a run
        st.step.zero_()
        hook = self._decode_hook
        t = 0
        if self.graphs and not st.graph_failed and st.graph is None:
            self._decode_step(st)                  # step 0 eagerly: also configures every kernel on this device
            if hook is not None:
                hook(0, st.cmd_logits, st.args_logits)
            t = 1
            try:
                torch.cuda.synchronize(dev)
                g = torch.cuda.CUDAGraph()
                from . import _lib
                n0 = _lib.launch_count()
                with torch.cuda.graph(g, pool=st.pool):
                    self._decode_step(st)
                st.graph, st.n_launches = g, _lib.launch_count() - n0
            except Exception as e:                   # capture is an optimisation: fall back to eager launches
                import sys
                sys.stderr.write("deepsvg_b200: WARNING: CUDA-graph capture of the decode step failed (%r); running "
                                 "eagerly\n" % (e,))
                st.graph, st.graph_failed = None, True
        for t in range(t, T):
            if self.graphs and st.graph is not None:
                st.graph.replay()
                self.graph_kernel_launches += st.n_launches
            else:
                self._decode_step(st)
            if hook is not None:
                hook(t, st.cmd_logits, st.args_logits)
        commands_y = st.out_cmd.view(N, 1, T).clone()
        args_y = st.out_args.view(N, 1, T, cfg.n_args).clone()
        return self._autoregressive_output(commands_y, args_y, concat_groups)

    def _decode_step(self, st):
        """One decode step on the state's static buffers: embed -> layers -> final LayerNorm -> heads -> sample, t += 1."""
        cfg = self.cfg
        P = self._param
        N, T, dev, pl = st.N, cfg.max_total_len, st.dev, self.planes
        d, H, nl = cfg.d_model, cfg.n_heads, cfg.n_layers_decode
        hd = d // H
        x = torch.empty(N, d, device=dev)
        ops.decode_embed(st.step, st.cmd_in, st.args_in, st.grp, st.key_valid, P("decoder.embedding.command_embed.weight"),
                         st.table, st.base, P("decoder.embedding.pos_encoding.pos_embed.weight"),
                         P("decoder.embedding.group_embed.weight"), x, N, T, self.args_dim, cfg.n_args, d)
        nxt = None
        for i in range(nl):
            lp = "decoder.decoder.layers.%d" % i
            nm = "decoder.decoder.layers.%d.norm1" % (i + 1) if i + 1 < nl else "decoder.decoder.norm"
            attn = (lambda qkv, o, i=i: ops.decode_attn(st.step, qkv, st.k_cache[i], st.v_cache[i], st.key_valid, o, N, H,
                                                        hd, T))
            x, nxt = self._layer_fwd(st.sv, lp, x, N, 1, N, None, st.rowvec[i], 1, a_pre=nxt,
                                     next_ln=(P(nm + ".weight"), P(nm + ".bias")), attn=attn)
        if nxt is not None:
            y = nxt[0]
        else:
            y = Act(N, d, pl, dev)
            ops.ln_fwd(x, P("decoder.decoder.norm.weight"), P("decoder.decoder.norm.bias"), y, torch.empty(N, device=dev),
                       torch.empty(N, device=dev), N, d)
        w, _ = self._pack("decoder.fcn.command_fcn.weight")
        ops.linear(y, w, N, cfg.n_commands, d, bias=P("decoder.fcn.command_fcn.bias"), out_f32=st.cmd_logits)
        w, _ = self._pack("decoder.fcn.args_fcn.weight")
        ops.linear(y, w, N, cfg.n_args * self.args_dim, d, bias=P("decoder.fcn.args_fcn.bias"), out_f32=st.args_logits)
        ops.decode_sample(st.step, st.cmd_logits, st.args_logits, st.temperature, st.seed, st.cmd_in, st.args_in,
                          st.out_cmd, st.out_args, N, T, cfg.n_args, self.args_dim)

    def _make_absolute(self, commands_y, args_y):
        """model.py:461-478: relative argument classes back to absolute coordinates (running sum of the end positions over
        the real commands, as the reference does over the flattened batch)."""
        args_y = args_y.clone()
        mask = self.cmd_args_mask[commands_y].bool()
        args_y[mask] -= self.cfg.args_dim - 1
        real = commands_y < 4
        a = args_y[real]
        end_pos = a[:-1, 9:11].cumsum(dim=0)
        a[1:, 5:7] += end_pos
        a[1:, 7:9] += end_pos
        a[1:, 9:11] += end_pos
        args_y[real] = a
        _, args_y = self._make_valid(commands_y, args_y)
        return args_y

    def _make_valid(self, commands_y, args_y, visibility_y=None, PAD_VAL=-1):
        """model.py:450-459: invisible paths become `m EOS EOS ...` with PAD arguments; argument slots a command does
        not use (CMD_ARGS_MASK) become PAD."""
        if visibility_y is not None:
            blank = torch.full((commands_y.size(-1),), 4, dtype=commands_y.dtype, device=commands_y.device)
            blank[0] = 0
            hidden = ~visibility_y
            commands_y = torch.where(hidden.unsqueeze(-1), blank, commands_y)
            args_y = torch.where(hidden[..., None, None], torch.full_like(args_y, PAD_VAL), args_y)
        used = self.cmd_args_mask[commands_y].bool()
        args_y = torch.where(used, args_y, torch.full_like(args_y, PAD_VAL))
        return commands_y, args_y

    # =================================================================================================
    # weights: fp32 master -> (split-)bf16 operand + transposed operand, refreshed when the parameter changes
    # =================================================================================================
    def _pack(self, name, need_t=True):
        p = self._param(name)
        key = (p.data_ptr(), p._version, self.planes, p.device)
        # keyed per device: nn.DataParallel replicas share this dict (shallow-copied __dict__) and run in threads
        name = (name, p.device)
        hit = self._wcache.get(name)
        if hit is not None and hit[0] == key:
            return hit[1], hit[2]
        Nn, K = p.shape
        if hit is not None and hit[1].planes == self.planes and hit[1].t.device == p.device:
            w, wt = hit[1], hit[2]
        else:
            w = Act(Nn, K, self.planes, p.device, ld=_r8(K), zero=True)
            wt = Act(K, Nn, self.planes, p.device, ld=_r8(Nn), zero=True)
        ops.cast_act(p.data, Nn, K, out=w, outT=wt)
        self._wcache[name] = (key, w, wt)
        return w, wt

    # =================================================================================================
    # forward
    # =================================================================================================
    def _drop(self, sv, tag, p=None):
        """(p, site, seed) of a dropout call site; p = 0 in eval mode."""
        if not sv.training:
            return (0.0, 0, 0)
        # bit 31 of the site: `seed` is a device pointer (include/dsvg_b200.h, DSVG_SEED_IS_DEVICE_PTR)
        return (self.cfg.dropout if p is None else p, self._site(tag) | 0x80000000, sv.seed_ptr)

    def _layer_fwd(self, sv, pre, x, M, L, nseq, key_valid, rowvec, rpg, a_pre=None, next_ln=None, attn=None):
        """One pre-LN block.  a_pre = (LN1(x) Act, mean, rstd) when the previous GEMM already produced it in its epilogue;
        next_ln = (gamma, beta) of the LayerNorm that consumes this block's output (next layer's norm1 or the stack's final
        norm): when the GEMM tile owns whole rows (ops.ln_fusable) it is computed in the FFN2 epilogue and returned.
        attn(qkv, o), when given, replaces the self-attention over whole sequences (the cached decoder's one-row step)."""
        cfg = self.cfg
        d, ff, H = cfg.d_model, cfg.dim_feedforward, cfg.n_heads
        hd = d // H
        dev, pl = x.device, self.planes
        P = lambda n: self._param(pre + "." + n)
        fuse = ops.ln_fusable(M, d, pl)
        s = {}
        if a_pre is not None:
            a, s["mean1"], s["rstd1"] = a_pre
        else:
            a = Act(M, d, pl, dev)
            s["mean1"], s["rstd1"] = torch.empty(M, device=dev), torch.empty(M, device=dev)
            ops.ln_fwd(x, P("norm1.weight"), P("norm1.bias"), a, s["mean1"], s["rstd1"], M, d)
        qkv = Act(M, 3 * d, pl, dev)
        w_in, _ = self._pack(pre + ".self_attn.in_proj_weight")
        ops.linear(a, w_in, M, 3 * d, d, bias=P("self_attn.in_proj_bias"), scale_cols=d, scale=float(hd) ** -0.5,
                   out_act=qkv)
        o = Act(M, d, pl, dev)
        if attn is not None:
            attn(qkv, o)
        else:
            ops.attn_fwd(qkv, key_valid, o, nseq, L, H, hd, self._drop(sv, pre + ".attn"),
                         causal=pre.startswith(getattr(sv, "causal_stack", "\0")))
        x1 = torch.empty(M, d, device=dev)
        w_o, _ = self._pack(pre + ".self_attn.out_proj.weight")
        b = Act(M, d, pl, dev)
        s["mean2"], s["rstd2"] = torch.empty(M, device=dev), torch.empty(M, device=dev)
        ops.linear(o, w_o, M, d, d, bias=P("self_attn.out_proj.bias"), drop=self._drop(sv, pre + ".drop1"),
                   rowvec=rowvec, rows_per_group=rpg, residual=x, out_f32=x1,
                   ln=(P("norm2.weight"), P("norm2.bias"), b, s["mean2"], s["rstd2"]) if fuse else None)
        if not fuse:
            ops.ln_fwd(x1, P("norm2.weight"), P("norm2.bias"), b, s["mean2"], s["rstd2"], M, d)
        h = Act(M, ff, pl, dev)
        w1, _ = self._pack(pre + ".linear1.weight")
        ops.linear(b, w1, M, ff, d, bias=P("linear1.bias"), relu=True, drop=self._drop(sv, pre + ".dropff"), out_act=h)
        x2 = torch.empty(M, d, device=dev)
        w2, _ = self._pack(pre + ".linear2.weight")
        nxt = None
        if fuse and next_ln is not None:
            nxt = (Act(M, d, pl, dev), torch.empty(M, device=dev), torch.empty(M, device=dev))
        ops.linear(h, w2, M, d, ff, bias=P("linear2.bias"), drop=self._drop(sv, pre + ".drop2"), residual=x1,
                   out_f32=x2, ln=(next_ln[0], next_ln[1]) + nxt if nxt is not None else None)
        s.update(x=x, a=a, qkv=qkv, o=o, x1=x1, b=b, h=h)
        sv.layers[pre] = s
        return x2, nxt

    def _globals_fwd(self, sv, pre, zmem, n_groups, lab, lab_rpg):
        """rowvec of a layer: dropout(linear_global(zmem)) [+ dropout(linear_global2(label))]
        (improved_transformer.py:47-49,131-136).  zmem: Act [n_groups, dz] or None; lab: Act [N, dim_label] or None.
        lab_rpg: how many zmem groups share one label row (1 when both are per icon)."""
        cfg = self.cfg
        d = cfg.d_model
        g2 = None
        if lab is not None:
            N = lab.rows
            g2 = torch.empty(N, d, device=lab.t.device)
            w, _ = self._pack(pre + ".linear_global2.weight")
            ops.linear(lab, w, N, d, cfg.dim_label, bias=self._param(pre + ".linear_global2.bias"),
                       drop=self._drop(sv, pre + ".dropg2"), out_f32=g2)
        if zmem is None:
            return g2
        g = torch.empty(n_groups, d, device=zmem.t.device)
        w, _ = self._pack(pre + ".linear_global.weight")
        ops.linear(zmem, w, n_groups, d, cfg.dim_z, bias=self._param(pre + ".linear_global.bias"),
                   drop=self._drop(sv, pre + ".dropg"), rowvec=g2, rows_per_group=lab_rpg, out_f32=g)
        return g

    def _stack_fwd(self, sv, pre, n_layers, x, M, L, nseq, key_valid, zmem=None, lab=None, lab_rows_per_group=1,
                   lab_rpg=1, final_ln=False):
        """L = sequence length; rows of one rowvec group = L (zmem per sequence) or lab_rows_per_group (label only).
        Returns (x, final) -- final = (LN_f(x) Act, mean, rstd) when final_ln was requested AND the last FFN2 epilogue
        could produce it (otherwise None: the caller runs the stand-alone LayerNorm kernel)."""
        nxt = None
        for i in range(n_layers):
            lp = "%s.layers.%d" % (pre, i)
            rv = self._globals_fwd(sv, lp, zmem, nseq, lab, lab_rpg) if (zmem is not None or lab is not None) else None
            rpg = L if zmem is not None else lab_rows_per_group
            if i + 1 < n_layers:
                nl = "%s.layers.%d" % (pre, i + 1)
                next_ln = (self._param(nl + ".norm1.weight"), self._param(nl + ".norm1.bias"))
            else:
                next_ln = (self._param(pre + ".norm.weight"), self._param(pre + ".norm.bias")) if final_ln else None
            x, nxt = self._layer_fwd(sv, lp, x, M, L, nseq, key_valid, rv, rpg, a_pre=nxt, next_ln=next_ln)
        return x, nxt

    def _forward_impl(self, inp, seed_dev=None):
        cfg = self.cfg
        sv = _Saved()
        self._last_saved = sv
        sv.training = bool(inp["training"])
        sv.seed_dev, sv.seed_ptr = seed_dev, 0
        if sv.training:
            # the seed of this call's dropout masks lives in device memory (one uint64 per forward call, kept alive with the
            # saved activations: the backward regenerates the masks from it); drawn from torch's CUDA generator
            if seed_dev is None:
                ref = inp["commands"] if inp["commands"] is not None else inp["z"]
                sv.seed_dev = torch.empty(1, dtype=torch.int64, device=ref.device).random_()
            sv.seed_ptr = sv.seed_dev.data_ptr()
        d, dz = cfg.d_model, cfg.dim_z
        two = cfg.encode_stages == 2
        pl = self.planes
        P = self._param
        commands, args, label = inp["commands"], inp["args"], inp["label"]
        sv.label = label
        sv.has_encoder = inp["z"] is None
        if sv.has_encoder:
            dev = commands.device
            commands = commands.contiguous().float()
            args = args.contiguous().float()
            N, G, L = commands.shape
            if two and G != cfg.max_num_groups:
                raise ValueError("two-stage model expects %d paths per icon, got %d" % (cfg.max_num_groups, G))
            if not two and G != 1:
                raise ValueError("one-stage model expects grouped tensors with G = 1")
            exp_L = (cfg.max_seq_len if two else cfg.max_total_len) + 2
            if L != exp_L:
                raise ValueError("expected %d positions per sequence, got %d" % (exp_L, L))
            nseq, M1 = N * G, N * G * L
            sv.commands, sv.args, sv.N, sv.G, sv.L = commands, args, N, G, L
            # ---- bookkeeping (model/utils.py) ----
            sv.first_eos = torch.empty(nseq, dtype=torch.int32, device=dev)
            sv.visible = torch.empty(nseq, dtype=torch.uint8, device=dev)
            sv.key_valid = torch.empty(M1, dtype=torch.uint8, device=dev)
            sv.grp = torch.empty(M1, dtype=torch.uint8, device=dev) if not two else None
            sv.counts = torch.zeros(2, device=dev)
            ops.seq_prep(commands, nseq, L, sv.first_eos, sv.visible, sv.key_valid, sv.grp, sv.counts)
            # ---- embedding (model.py:46-57) ----
            V, na = cfg.args_dim + 1, cfg.n_args
            sv.table = torch.empty(na * V, d, device=dev)
            sv.base = torch.empty(d, device=dev)
            ops.embed_fold(P("encoder.embedding.arg_embed.weight"), P("encoder.embedding.embed_fcn.weight"),
                           P("encoder.embedding.embed_fcn.bias"), sv.table, sv.base, V, na, d)
            x = torch.empty(M1, d, device=dev)
            ops.embed_fwd(commands, args, sv.grp, P("encoder.embedding.command_embed.weight"), sv.table, sv.base,
                          P("encoder.embedding.pos_encoding.pos_embed.weight"),
                          None if two else P("encoder.embedding.group_embed.weight"), x, M1, L, V, na, d,
                          self._drop(sv, "enc.pe", 0.1))                       # positional_encoding.py:26 (p fixed)
            lab_e = None
            if cfg.label_condition:
                lab_e = Act(N, cfg.dim_label, pl, dev)
                ops.gather_rows(P("encoder.label_embedding.label_embedding.weight"), label, N, cfg.dim_label, lab_e)
            sv.lab_e = lab_e
            # path-level stack: the reference repeats the label per path BEFORE linear_global2 + dropout (model.py:123), so
            # every (path, icon) draws its own dropout mask: one label row per path here too
            lab_e1, sv.label_e1 = lab_e, label
            if cfg.label_condition and G > 1:
                sv.label_e1 = label.repeat_interleave(G)
                lab_e1 = Act(nseq, cfg.dim_label, pl, dev)
                ops.gather_rows(P("encoder.label_embedding.label_embedding.weight"), sv.label_e1, nseq, cfg.dim_label, lab_e1)
            sv.lab_e1 = lab_e1
            # ---- E1 (model.py:135-137) ----
            x, _ = self._stack_fwd(sv, "encoder.encoder", cfg.n_layers, x, M1, L, nseq, sv.key_valid, lab=lab_e1,
                                   lab_rows_per_group=L)
            sv.e1_x = x
            zp = torch.empty(nseq, d, device=dev)
            sv.e1_mean, sv.e1_rstd = torch.empty(M1, device=dev), torch.empty(M1, device=dev)
            sv.e1_icnt = torch.empty(nseq, device=dev)
            ops.ln_pool_fwd(x, P("encoder.encoder.norm.weight"), P("encoder.encoder.norm.bias"), sv.key_valid, zp,
                            sv.e1_mean, sv.e1_rstd, sv.e1_icnt, nseq, L, d)
            if two:
                # ---- E2 (model.py:153-162): sequences of G path codes per icon ----
                if self.self_match:                      # model.py:157: the path codes enter E2 as they are
                    x = zp
                else:
                    x = torch.empty(nseq, d, device=dev)
                    ops.rows_embed_fwd(zp, P("encoder.hierarchical_PE.pos_embed.weight"), x, nseq, G, d,
                                       self._drop(sv, "enc.pe2", 0.1))
                x, _ = self._stack_fwd(sv, "encoder.hierarchical_encoder", cfg.n_layers, x, nseq, G, N, sv.visible,
                                       lab=lab_e, lab_rows_per_group=G)
                sv.e2_x = x
                z = torch.empty(N, d, device=dev)
                sv.e2_mean, sv.e2_rstd = torch.empty(nseq, device=dev), torch.empty(nseq, device=dev)
                sv.e2_icnt = torch.empty(N, device=dev)
                ops.ln_pool_fwd(x, P("encoder.hierarchical_encoder.norm.weight"),
                                P("encoder.hierarchical_encoder.norm.bias"), sv.visible, z, sv.e2_mean, sv.e2_rstd,
                                sv.e2_icnt, N, G, d)
            else:
                z = zp
            # ---- ResNet (basic_blocks.py:59-65) ----
            sv.res = []
            if cfg.use_resnet:
                for i in range(1, 5):
                    za = Act(N, d, pl, dev)
                    ops.cast_act(z, N, d, out=za)
                    r32, ra = torch.empty(N, d, device=dev), Act(N, d, pl, dev)
                    w, _ = self._pack("resnet.linear%d.0.weight" % i)
                    ops.linear(za, w, N, d, d, bias=P("resnet.linear%d.0.bias" % i), relu=True, out_f32=r32, out_act=ra)
                    zn = torch.empty(N, d, device=dev)
                    ops.add_f32(z, r32, zn)
                    sv.res.append((za, ra))
                    z = zn
            za = Act(N, d, pl, dev)
            ops.cast_act(z, N, d, out=za)
            sv.lat_in = za
            zl = torch.empty(N, dz, device=dev)
            z_act = Act(N, dz, pl, dev)
            if cfg.use_vae:                                                    # model.py:182-187
                sv.mu, sv.ls = torch.empty(N, dz, device=dev), torch.empty(N, dz, device=dev)
                w, _ = self._pack("vae.enc_mu_fcn.weight")
                ops.linear(za, w, N, dz, d, bias=P("vae.enc_mu_fcn.bias"), out_f32=sv.mu)
                w, _ = self._pack("vae.enc_sigma_fcn.weight")
                ops.linear(za, w, N, dz, d, bias=P("vae.enc_sigma_fcn.bias"), out_f32=sv.ls)
                sv.eps = self._eps_override if self._eps_override is not None else torch.randn(N, dz, device=dev)
                ops.vae_fwd(sv.mu, sv.ls, sv.eps, zl, N * dz)
                ops.cast_act(zl, N, dz, out=z_act)
            else:                                                              # model.py:196-197
                w, _ = self._pack("bottleneck.bottleneck.weight")
                ops.linear(za, w, N, dz, d, bias=P("bottleneck.bottleneck.bias"), out_f32=zl, out_act=z_act)
        else:
            zin = inp["z"]
            N = zin.shape[0]
            dev = zin.device
            sv.N = N
            if inp.get("hierarch_logits") is not None:
                zl = z_act = None                                               # the icon-level latent is not needed
            else:
                zl = zin.reshape(N, dz).contiguous().float()                    # batch-first (N,1,1,dz), model.py:369
                z_act = Act(N, dz, pl, dev)
                ops.cast_act(zl, N, dz, out=z_act)
        sv.z32, sv.z_act = zl, z_act
        if inp["encode_mode"]:
            return [zl], sv

        # ---- decoder (model.py:243-285) ----
        lab_d = None
        if cfg.label_condition:
            lab_d = Act(N, cfg.dim_label, pl, dev)
            ops.gather_rows(P("decoder.label_embedding.label_embedding.weight"), label, N, cfg.dim_label, lab_d)
        sv.lab_d = lab_d
        outs = []
        if two and inp.get("hierarch_logits") is not None:
            Gp = cfg.num_groups_proposal
            nq = N * Gp
            zp32 = inp["z"].reshape(nq, dz).contiguous().float()
            zp_act = Act(nq, dz, pl, dev)
            ops.cast_act(zp32, nq, dz, out=zp_act)
            vis_logits = inp["hierarch_logits"].reshape(Gp, N, 2).permute(1, 0, 2).contiguous().float().view(nq, 2)
            zmem, nseq_d, lab_rpg = zp_act, nq, Gp
        elif two:
            Gp = cfg.num_groups_proposal
            nq = N * Gp
            x = torch.empty(nq, d, device=dev)
            ops.rows_embed_fwd(None, P("decoder.hierarchical_embedding.PE.pos_embed.weight"), x, nq, Gp, d,
                               self._drop(sv, "dec.pe2", 0.1))
            x, fin = self._stack_fwd(sv, "decoder.hierarchical_decoder", cfg.n_layers_decode, x, nq, Gp, N, None,
                                     zmem=z_act, lab=lab_d, lab_rpg=1, final_ln=True)
            sv.d2_x = x
            if fin is not None:
                y, sv.d2_mean, sv.d2_rstd = fin
            else:
                y = Act(nq, d, pl, dev)
                sv.d2_mean, sv.d2_rstd = torch.empty(nq, device=dev), torch.empty(nq, device=dev)
                ops.ln_fwd(x, P("decoder.hierarchical_decoder.norm.weight"), P("decoder.hierarchical_decoder.norm.bias"),
                           y, sv.d2_mean, sv.d2_rstd, nq, d)
            sv.d2_y = y
            vis_logits = torch.empty(nq, 2, device=dev)
            w, _ = self._pack("decoder.hierarchical_fcn.visibility_fcn.weight")
            ops.linear(y, w, nq, 2, d, bias=P("decoder.hierarchical_fcn.visibility_fcn.bias"), out_f32=vis_logits)
            zp32, zp_act = torch.empty(nq, dz, device=dev), Act(nq, dz, pl, dev)
            w, _ = self._pack("decoder.hierarchical_fcn.z_fcn.weight")
            ops.linear(y, w, nq, dz, d, bias=P("decoder.hierarchical_fcn.z_fcn.bias"), out_f32=zp32, out_act=zp_act)
            sv.zpath_act = zp_act
            if inp["return_hierarch"]:
                return [vis_logits, zp32], sv
            zmem, nseq_d, lab_rpg = zp_act, nq, Gp
        else:
            vis_logits = None
            zmem, nseq_d, lab_rpg = z_act, N, 1
        Ld = (cfg.max_seq_len if two else cfg.max_total_len) + 1
        Md = nseq_d * Ld
        sv.nseq_d, sv.Ld, sv.Md = nseq_d, Ld, Md
        dec_valid = None
        if self.autoregressive:
            # ---- autoregressive decoder input (model.py:262-269): the shifted target tokens, embedded with the decoder's own
            # SVGEmbedding (group index = number of "m" so far), attended causally with the key-padding mask of those tokens
            cd, ad = inp["dec_inputs"]
            if cd.shape[0] != N or cd.shape[1] != 1:
                raise ValueError("autoregressive decoder expects grouped tokens (N, 1, S)")
            Ld = cd.shape[2]
            if Ld > cfg.max_total_len + 1:
                raise ValueError("at most %d decoder positions" % (cfg.max_total_len + 1))
            Md = nseq_d * Ld
            sv.Ld, sv.Md = Ld, Md
            sv.dec_cmd, sv.dec_arg = cd, ad
            sv.dec_grp = torch.empty(Md, dtype=torch.uint8, device=dev)
            dec_valid = torch.empty(Md, dtype=torch.uint8, device=dev)
            ops.seq_prep(cd, nseq_d, Ld, None, None, dec_valid, sv.dec_grp, None)
            sv.dec_valid = dec_valid
            Vd, na = self.args_dim, cfg.n_args
            sv.dec_table = torch.empty(na * Vd, d, device=dev)
            sv.dec_base = torch.empty(d, device=dev)
            ops.embed_fold(P("decoder.embedding.arg_embed.weight"), P("decoder.embedding.embed_fcn.weight"),
                           P("decoder.embedding.embed_fcn.bias"), sv.dec_table, sv.dec_base, Vd, na, d)
            x = torch.empty(Md, d, device=dev)
            ops.embed_fwd(cd, ad, sv.dec_grp, P("decoder.embedding.command_embed.weight"), sv.dec_table, sv.dec_base,
                          P("decoder.embedding.pos_encoding.pos_embed.weight"), P("decoder.embedding.group_embed.weight"), x,
                          Md, Ld, Vd, na, d, self._drop(sv, "dec.pe", 0.1))
            sv.causal_stack = "decoder.decoder"
        else:
            x = torch.empty(Md, d, device=dev)
            ops.rows_embed_fwd(None, P("decoder.embedding.PE.pos_embed.weight"), x, Md, Ld, d, self._drop(sv, "dec.pe", 0.1))
        lab_d1, sv.label_d1 = lab_d, label
        if cfg.label_condition and two:                       # model.py:255: the label is repeated per predicted path
            sv.label_d1 = label.repeat_interleave(lab_rpg)
            lab_d1 = Act(nseq_d, cfg.dim_label, pl, dev)
            ops.gather_rows(P("decoder.label_embedding.label_embedding.weight"), sv.label_d1, nseq_d, cfg.dim_label, lab_d1)
        sv.lab_d1 = lab_d1
        x, fin = self._stack_fwd(sv, "decoder.decoder", cfg.n_layers_decode, x, Md, Ld, nseq_d, dec_valid, zmem=zmem, lab=lab_d1,
                                 lab_rpg=1, final_ln=True)
        sv.d1_x = x
        if fin is not None:
            y, sv.d1_mean, sv.d1_rstd = fin
        else:
            y = Act(Md, d, pl, dev)
            sv.d1_mean, sv.d1_rstd = torch.empty(Md, device=dev), torch.empty(Md, device=dev)
            ops.ln_fwd(x, P("decoder.decoder.norm.weight"), P("decoder.decoder.norm.bias"), y, sv.d1_mean, sv.d1_rstd, Md, d)
        sv.d1_y = y
        nc, na_out = cfg.n_commands, cfg.n_args * self.args_dim
        cmd_logits = torch.empty(Md, nc, device=dev)
        w, _ = self._pack("decoder.fcn.command_fcn.weight")
        ops.linear(y, w, Md, nc, d, bias=P("decoder.fcn.command_fcn.bias"), out_f32=cmd_logits)   # basic_blocks.py:18
        args_logits = torch.empty(Md, na_out, device=dev)
        w, _ = self._pack("decoder.fcn.args_fcn.weight")
        ops.linear(y, w, Md, na_out, d, bias=P("decoder.fcn.args_fcn.bias"), out_f32=args_logits)  # basic_blocks.py:20
        if inp.get("match_targets") is not None:
            # ---- Hungarian self-matching (model.py:384-394): pick, per icon, which predicted slot explains which target
            # path, then emit the logits in that order.  The permutation is applied to the decoder rows (67 MB) and the two
            # heads run again on the permuted rows -- the same cost as gathering the 1.4 GB logits tensor, and the backward
            # pass then only has to scatter the head input gradients back.
            tc, ta = inp["match_targets"]
            Gt, Gp = tc.shape[1], cfg.num_groups_proposal
            asg, sv.match_cost, _ = ops.match_assign(cmd_logits, args_logits, na_out, vis_logits, tc, ta, N, Gt, Gp, Ld + 1,
                                                     cfg.n_args, self.args_dim)
            sv.asg = asg
            y_perm = Act(Md, d, pl, dev)
            ops.permute_act(y, y_perm, asg, N, Gp, Ld)
            sv.d1_y = y_perm
            w, _ = self._pack("decoder.fcn.command_fcn.weight")
            ops.linear(y_perm, w, Md, nc, d, bias=P("decoder.fcn.command_fcn.bias"), out_f32=cmd_logits)
            w, _ = self._pack("decoder.fcn.args_fcn.weight")
            ops.linear(y_perm, w, Md, na_out, d, bias=P("decoder.fcn.args_fcn.bias"), out_f32=args_logits)
            y2_perm = Act(nq, d, pl, dev)
            ops.permute_act(sv.d2_y, y2_perm, asg, N, Gp, 1)
            sv.d2_y_perm = y2_perm
            vis_perm = torch.empty_like(vis_logits)
            ops.permute_groups(vis_logits, vis_perm, asg, N, Gp, 8)
            vis_logits = vis_perm
        outs = [cmd_logits, args_logits]
        if two:
            outs.append(vis_logits)
        if cfg.use_vae and sv.has_encoder:
            outs += [sv.mu, sv.ls]
        return outs, sv

    # =================================================================================================
    # backward
    # =================================================================================================
    def _layer_bwd(self, sv, gd, pre, dx2, dx2_act, M, L, nseq, key_valid, prev_drop, want_dact):
        """dx2: fp32 grad of the layer output; dx2_act = dropout-masked act copy (operand of the FFN2 backward).
        Returns (dx0, dx0_act or None, dx1) where dx1 is the grad at the post-attention residual (rowvec branch)."""
        cfg = self.cfg
        d, ff, H = cfg.d_model, cfg.dim_feedforward, cfg.n_heads
        hd = d // H
        s = sv.layers[pre]
        dev, pl = dx2.device, self.planes
        P = lambda n: self._param(pre + "." + n)
        G = lambda n: gd[pre + "." + n]
        pff = self._drop(sv, pre + ".dropff")
        # The block's four weight gradients: one grouped launch at the end of the block for the path-level row counts in fast
        # mode (ops.outer_group: they then share one wave of CTAs), separate launches otherwise.
        # Measured (hier, d_model 256: 8 tall tiles per block): `outer` family 2.57 -> 2.14 ms per step, step 12.93 -> 12.69 ms.  With
        # d_model 512 the block has 24 tiles, each launch already fills the machine with few splits, and grouping changes nothing
        # (12.0 vs 12.2 ms): those stay separate launches.
        t256 = lambda n: (n + 255) // 256
        n_tiles = t256(3 * d) * t256(d) + t256(d) * t256(d) + 2 * t256(ff) * t256(d)
        grouped = [] if (pl == 1 and M >= 16384 and n_tiles <= 16) else None

        def wgrad(A, B, P_, Q_, w, b):
            if grouped is None:
                ops.outer(A, B, M, P_, Q_, w, colsum=b)
            else:
                grouped.append((A, B, P_, Q_, w, b))
        # ---- FFN ----
        wgrad(dx2_act, s["h"], d, ff, G("linear2.weight"), G("linear2.bias"))
        dh = Act(M, ff, pl, dev)
        _, w2t = self._pack(pre + ".linear2.weight")
        ops.linear(dx2_act, w2t, M, ff, d, mask=s["h"], mask_scale=1.0 / (1.0 - pff[0]) if pff[0] > 0 else 1.0, out_act=dh)
        wgrad(dh, s["b"], ff, d, G("linear1.weight"), G("linear1.bias"))
        _, w1t = self._pack(pre + ".linear1.weight")
        dx1 = torch.empty(M, d, device=dev)
        dt = Act(M, d, pl, dev)
        db = Act(M, d, pl, dev)
        ops.linear(dh, w1t, M, d, ff, out_act=db)
        ops.ln_bwd(s["x1"], s["mean2"], s["rstd2"], P("norm2.weight"), M, d, dy=db, dx_in=dx2, dx_out=dx1, dact=dt,
                   drop=self._drop(sv, pre + ".drop1"), dgamma=G("norm2.weight"), dbeta=G("norm2.bias"))
        # ---- attention ----
        wgrad(dt, s["o"], d, d, G("self_attn.out_proj.weight"), G("self_attn.out_proj.bias"))
        do = Act(M, d, pl, dev)
        _, wot = self._pack(pre + ".self_attn.out_proj.weight")
        ops.linear(dt, wot, M, d, d, out_act=do)
        dqkv = Act(M, 3 * d, pl, dev)
        ops.attn_bwd(s["qkv"], key_valid, do, dqkv, nseq, L, H, hd, float(hd) ** -0.5, self._drop(sv, pre + ".attn"),
                     causal=pre.startswith(getattr(sv, "causal_stack", "\0")))
        wgrad(dqkv, s["a"], 3 * d, d, G("self_attn.in_proj_weight"), G("self_attn.in_proj_bias"))
        _, wit = self._pack(pre + ".self_attn.in_proj_weight")
        dx0 = torch.empty(M, d, device=dev)
        dx0_act = Act(M, d, pl, dev) if want_dact else None
        da = Act(M, d, pl, dev)
        ops.linear(dqkv, wit, M, d, 3 * d, out_act=da)
        ops.ln_bwd(s["x"], s["mean1"], s["rstd1"], P("norm1.weight"), M, d, dy=da, dx_in=dx1, dx_out=dx0, dact=dx0_act,
                   drop=prev_drop, dgamma=G("norm1.weight"), dbeta=G("norm1.bias"))
        if grouped:
            ops.outer_group(grouped, M)
        return dx0, dx0_act, dx1

    def _globals_bwd(self, sv, gd, pre, dx1, n_groups, L, zmem, dzmem, lab, dlab, lab_rows_per_group, lab_rpg):
        """Gradients of the rowvec branch of one layer (see _globals_fwd).  dzmem / dlab: fp32 accumulators or None."""
        cfg = self.cfg
        d = cfg.d_model
        dev, pl = dx1.device, self.planes
        if zmem is not None:
            dgv = torch.empty(n_groups, d, device=dev)
            ops.seg_sum(dx1, n_groups, L, d, out_f32=dgv)
            dg = Act(n_groups, d, pl, dev)
            ops.cast_act(dgv, n_groups, d, out=dg, drop=self._drop(sv, pre + ".dropg"))
            ops.outer(dg, zmem, n_groups, d, cfg.dim_z, gd[pre + ".linear_global.weight"],
                      colsum=gd[pre + ".linear_global.bias"])
            _, wt = self._pack(pre + ".linear_global.weight")
            ops.linear(dg, wt, n_groups, cfg.dim_z, d, residual=dzmem, out_f32=dzmem)
            if lab is not None:
                N = lab.rows
                if lab_rpg > 1:
                    d2v = torch.empty(N, d, device=dev)
                    ops.seg_sum(dgv, N, lab_rpg, d, out_f32=d2v)
                else:
                    d2v = dgv
        elif lab is not None:
            N = lab.rows
            d2v = torch.empty(N, d, device=dev)
            ops.seg_sum(dx1, N, lab_rows_per_group, d, out_f32=d2v)
        if lab is not None:
            dg2 = Act(N, d, pl, dev)
            ops.cast_act(d2v, N, d, out=dg2, drop=self._drop(sv, pre + ".dropg2"))
            ops.outer(dg2, lab, N, d, cfg.dim_label, gd[pre + ".linear_global2.weight"],
                      colsum=gd[pre + ".linear_global2.bias"])
            _, wt = self._pack(pre + ".linear_global2.weight")
            ops.linear(dg2, wt, N, cfg.dim_label, d, residual=dlab, out_f32=dlab)

    def _stack_bwd(self, sv, gd, pre, n_layers, dx, dx_act, M, L, nseq, key_valid, zmem=None, dzmem=None, lab=None,
                   dlab=None, lab_rows_per_group=1, lab_rpg=1):
        """Reverse pass over a stack; dx / dx_act are the grads at the stack's last residual (after the final-norm bwd)."""
        for i in reversed(range(n_layers)):
            lp = "%s.layers.%d" % (pre, i)
            prev = self._drop(sv, "%s.layers.%d.drop2" % (pre, i - 1)) if i > 0 else (0.0, 0, 0)
            dx, dx_act, dx1 = self._layer_bwd(sv, gd, lp, dx, dx_act, M, L, nseq, key_valid, prev, want_dact=i > 0)
            if zmem is not None or lab is not None:
                self._globals_bwd(sv, gd, lp, dx1, nseq, L, zmem, dzmem, lab, dlab, lab_rows_per_group, lab_rpg)
        return dx

    def _head_bwd(self, gd, name, sources, y, M, n_out, d, dy32):
        """Backward of one output Linear (weights `name`) for a list of (dl act, scale_dev) gradient sources; the input
        gradient is accumulated into the fp32 buffer dy32 [M, d]."""
        _, wt = self._pack(name + ".weight")
        for dl, sc in sources:
            ops.outer(dl, y, M, n_out, d, gd[name + ".weight"], alpha_dev=sc, colsum=gd[name + ".bias"])
            ops.linear(dl, wt, M, d, n_out, acc_scale=sc, residual=dy32, out_f32=dy32)

    def _bucket_split(self):
        """Offset (in elements) of the first decoder parameter in the flat gradient bucket.  The decoder half of the backward
        (heads, D1, D2) completes exactly flat[split:]; the encoder half (latent, E2, E1, embedding) completes flat[:split]."""
        off = 0
        for n in self._pnames:
            if n.startswith("decoder."):
                return off
            off += self._param(n).numel()
        return off

    def _backward_a(self, sv, out_grads, g_token):
        """Decoder half of the backward pass (output heads, D1, D2).  Returns the state the encoder half continues from."""
        cfg = self.cfg
        d, dz = cfg.d_model, cfg.dim_z
        two = cfg.encode_stages == 2
        pl = self.planes
        P = self._param
        params = [P(n) for n in self._pnames]
        dev = params[0].device
        sizes = [p.numel() for p in params]
        flat = torch.zeros(sum(sizes), device=dev)
        gd, off = {}, 0
        for n, p, sz in zip(self._pnames, params, sizes):
            gd[n] = flat[off:off + sz].view(p.shape)
            off += sz
        handle = getattr(sv, "handle", None)
        fused = g_token is not None and handle is not None and handle.dl_args is not None
        N = sv.N

        def explicit(g, rows, cols, ld):
            a = Act(rows, cols, pl, dev, ld=ld, zero=True)
            ops.cast_act(g.contiguous().view(rows, cols), rows, cols, out=a)
            return a

        it = iter(out_grads)
        encode_only = not hasattr(sv, "d1_y")
        dz32 = torch.zeros(N, dz, device=dev)          # gradient w.r.t. the latent z
        dmu_ext = dls_ext = None
        if encode_only:
            g = next(it)
            if g is not None:
                dz32 += g.reshape(N, dz)
        else:
            g_cmd, g_args = next(it), next(it)
            g_vis = next(it) if two else None
            if cfg.use_vae and sv.has_encoder:
                dmu_ext, dls_ext = next(it), next(it)
            Md, Ld, nseq_d = sv.Md, sv.Ld, sv.nseq_d
            nc, na_out = cfg.n_commands, cfg.n_args * self.args_dim
            src_args, src_cmd, src_vis = [], [], []
            if fused:
                sc = handle.scales
                src_args.append((handle.dl_args, sc[0:1]))
                src_cmd.append((handle.dl_cmd, sc[1:2]))
                if two:
                    src_vis.append((handle.dl_vis, sc[2:3]))
            if g_args is not None:
                src_args.append((explicit(g_args, Md, na_out, _r8(na_out)), None))
            if g_cmd is not None:
                src_cmd.append((explicit(g_cmd, Md, nc, 8), None))
            if g_vis is not None:
                src_vis.append((explicit(g_vis, N * cfg.num_groups_proposal, 2, 8), None))
            # ---- D1 heads + final norm ----
            dy32 = torch.zeros(Md, d, device=dev)
            self._head_bwd(gd, "decoder.fcn.args_fcn", src_args, sv.d1_y, Md, na_out, d, dy32)
            self._head_bwd(gd, "decoder.fcn.command_fcn", src_cmd, sv.d1_y, Md, nc, d, dy32)
            asg = getattr(sv, "asg", None)
            if asg is not None:      # the heads saw the slot-permuted rows: scatter their input gradient back (gather backward)
                dy32_p, dy32 = dy32, torch.empty(Md, d, device=dev)
                ops.permute_groups(dy32_p, dy32, asg, N, cfg.num_groups_proposal, Ld * d * 4, inverse=True)
            dy = Act(Md, d, pl, dev)
            ops.cast_act(dy32, Md, d, out=dy)
            nl = cfg.n_layers_decode
            dx, dxa = torch.empty(Md, d, device=dev), Act(Md, d, pl, dev)
            ops.ln_bwd(sv.d1_x, sv.d1_mean, sv.d1_rstd, P("decoder.decoder.norm.weight"), Md, d, dy=dy, dx_out=dx,
                       dact=dxa, drop=self._drop(sv, "decoder.decoder.layers.%d.drop2" % (nl - 1)),
                       dgamma=gd["decoder.decoder.norm.weight"], dbeta=gd["decoder.decoder.norm.bias"])
            dlab_d = torch.zeros(N, cfg.dim_label, device=dev) if cfg.label_condition else None
            if two:
                Gp = cfg.num_groups_proposal
                nq = N * Gp
                dzp32 = torch.zeros(nq, dz, device=dev)
                dlab_d1 = torch.zeros(nq, cfg.dim_label, device=dev) if cfg.label_condition else None
                dx = self._stack_bwd(sv, gd, "decoder.decoder", nl, dx, dxa, Md, Ld, nseq_d, None, zmem=sv.zpath_act,
                                     dzmem=dzp32, lab=sv.lab_d1, dlab=dlab_d1, lab_rpg=1)
                if cfg.label_condition:
                    ops.scatter_rows(dlab_d1, sv.label_d1, nq, cfg.dim_label,
                                     gd["decoder.label_embedding.label_embedding.weight"])
            else:
                dx = self._stack_bwd(sv, gd, "decoder.decoder", nl, dx, dxa, Md, Ld, nseq_d, getattr(sv, "dec_valid", None),
                                     zmem=sv.z_act, dzmem=dz32, lab=sv.lab_d, dlab=dlab_d, lab_rpg=1)
            if self.autoregressive:
                Vd, na = self.args_dim, cfg.n_args
                scratch = torch.empty(na * Vd, d, device=dev)
                ops.embed_bwd(sv.dec_cmd, sv.dec_arg, sv.dec_grp, dx, P("decoder.embedding.arg_embed.weight"),
                              P("decoder.embedding.embed_fcn.weight"), gd["decoder.embedding.command_embed.weight"],
                              gd["decoder.embedding.pos_encoding.pos_embed.weight"], gd["decoder.embedding.group_embed.weight"],
                              gd["decoder.embedding.arg_embed.weight"], gd["decoder.embedding.embed_fcn.weight"],
                              gd["decoder.embedding.embed_fcn.bias"], scratch, nseq_d, Ld, Vd, na, d, cfg.max_total_len + 2,
                              self._drop(sv, "dec.pe", 0.1))
            else:
                ops.rows_embed_bwd(dx, None, gd["decoder.embedding.PE.pos_embed.weight"], nseq_d, Ld, d,
                                   self._drop(sv, "dec.pe", 0.1))
            if two:
                # ---- D2 heads (basic_blocks.py:33-39) ----
                dzp = Act(nq, dz, pl, dev)
                ops.cast_act(dzp32, nq, dz, out=dzp)
                dy32 = torch.zeros(nq, d, device=dev)
                self._head_bwd(gd, "decoder.hierarchical_fcn.z_fcn", [(dzp, None)], sv.d2_y, nq, dz, d, dy32)
                if asg is not None and src_vis:
                    dyv_p, dyv = torch.zeros(nq, d, device=dev), torch.empty(nq, d, device=dev)
                    self._head_bwd(gd, "decoder.hierarchical_fcn.visibility_fcn", src_vis, sv.d2_y_perm, nq, 2, d, dyv_p)
                    ops.permute_groups(dyv_p, dyv, asg, N, Gp, d * 4, inverse=True)
                    dsum = torch.empty(nq, d, device=dev)
                    ops.add_f32(dy32, dyv, dsum)
                    dy32 = dsum
                else:
                    self._head_bwd(gd, "decoder.hierarchical_fcn.visibility_fcn", src_vis, sv.d2_y, nq, 2, d, dy32)
                dy = Act(nq, d, pl, dev)
                ops.cast_act(dy32, nq, d, out=dy)
                dx, dxa = torch.empty(nq, d, device=dev), Act(nq, d, pl, dev)
                ops.ln_bwd(sv.d2_x, sv.d2_mean, sv.d2_rstd, P("decoder.hierarchical_decoder.norm.weight"), nq, d, dy=dy,
                           dx_out=dx, dact=dxa, drop=self._drop(sv, "decoder.hierarchical_decoder.layers.%d.drop2" % (nl - 1)),
                           dgamma=gd["decoder.hierarchical_decoder.norm.weight"],
                           dbeta=gd["decoder.hierarchical_decoder.norm.bias"])
                dx = self._stack_bwd(sv, gd, "decoder.hierarchical_decoder", nl, dx, dxa, nq, Gp, N, None, zmem=sv.z_act,
                                     dzmem=dz32, lab=sv.lab_d, dlab=dlab_d, lab_rpg=1)
                ops.rows_embed_bwd(dx, None, gd["decoder.hierarchical_embedding.PE.pos_embed.weight"], N, Gp, d,
                                   self._drop(sv, "dec.pe2", 0.1))
            if cfg.label_condition:
                ops.scatter_rows(dlab_d, sv.label, N, cfg.dim_label, gd["decoder.label_embedding.label_embedding.weight"])
        return dict(flat=flat, gd=gd, dz32=dz32, dmu_ext=dmu_ext, dls_ext=dls_ext, fused=fused, handle=handle)

    def _backward_b(self, sv, st):
        """Encoder half of the backward pass: latent block, E2, E1, embedding."""
        cfg = self.cfg
        d, dz = cfg.d_model, cfg.dim_z
        two = cfg.encode_stages == 2
        pl = self.planes
        P = self._param
        gd, dz32, dmu_ext, dls_ext, fused, handle = st["gd"], st["dz32"], st["dmu_ext"], st["dls_ext"], st["fused"], st["handle"]
        dev = dz32.device
        N = sv.N
        if sv.has_encoder:
            # ---- latent (model.py:361-367) ----
            dzin = torch.zeros(N, d, device=dev)        # grad w.r.t. the ResNet output
            if cfg.use_vae:
                dmu, dls = torch.empty(N, dz, device=dev), torch.empty(N, dz, device=dev)
                kl_coef = handle.scales[3:4] if fused else None
                ops.vae_bwd(sv.mu, sv.ls, sv.eps, dz32, kl_coef, handle.loss_out if fused else None,
                            1.0 / (N * dz * getattr(handle, "world", 1)) if fused else 0.0, dmu, dls, N * dz)
                if dmu_ext is not None:
                    dmu += dmu_ext.reshape(N, dz)
                if dls_ext is not None:
                    dls += dls_ext.reshape(N, dz)
                for nm, g32 in (("vae.enc_mu_fcn", dmu), ("vae.enc_sigma_fcn", dls)):
                    ga = Act(N, dz, pl, dev)
                    ops.cast_act(g32, N, dz, out=ga)
                    self._head_bwd(gd, nm, [(ga, None)], sv.lat_in, N, dz, d, dzin)
            else:
                ga = Act(N, dz, pl, dev)
                ops.cast_act(dz32, N, dz, out=ga)
                self._head_bwd(gd, "bottleneck.bottleneck", [(ga, None)], sv.lat_in, N, dz, d, dzin)
            if cfg.use_resnet:
                for i in range(4, 0, -1):
                    za, ra = sv.res[i - 1]
                    dr = Act(N, d, pl, dev)
                    ops.cast_act(dzin, N, d, out=dr, mask=ra, mask_scale=1.0)
                    self._head_bwd(gd, "resnet.linear%d.0" % i, [(dr, None)], za, N, d, d, dzin)
            # ---- encoder ----
            G, L = sv.G, sv.L
            nseq, M1 = N * G, N * G * L
            nl = cfg.n_layers
            dlab_e = torch.zeros(N, cfg.dim_label, device=dev) if cfg.label_condition else None
            if two:
                dx, dxa = torch.empty(nseq, d, device=dev), Act(nseq, d, pl, dev)
                ops.ln_bwd(sv.e2_x, sv.e2_mean, sv.e2_rstd, P("encoder.hierarchical_encoder.norm.weight"), nseq, d,
                           dz=dzin, valid=sv.visible, inv_cnt=sv.e2_icnt, L=G, dx_out=dx, dact=dxa,
                           drop=self._drop(sv, "encoder.hierarchical_encoder.layers.%d.drop2" % (nl - 1)),
                           dgamma=gd["encoder.hierarchical_encoder.norm.weight"],
                           dbeta=gd["encoder.hierarchical_encoder.norm.bias"])
                dx = self._stack_bwd(sv, gd, "encoder.hierarchical_encoder", nl, dx, dxa, nseq, G, N, sv.visible,
                                     lab=sv.lab_e, dlab=dlab_e, lab_rows_per_group=G)
                if self.self_match:
                    dzp = dx
                else:
                    dzp = torch.empty(nseq, d, device=dev)
                    ops.rows_embed_bwd(dx, dzp, gd["encoder.hierarchical_PE.pos_embed.weight"], N, G, d,
                                       self._drop(sv, "enc.pe2", 0.1))
            else:
                dzp = dzin
            dx, dxa = torch.empty(M1, d, device=dev), Act(M1, d, pl, dev)
            ops.ln_bwd(sv.e1_x, sv.e1_mean, sv.e1_rstd, P("encoder.encoder.norm.weight"), M1, d, dz=dzp,
                       valid=sv.key_valid, inv_cnt=sv.e1_icnt, L=L, dx_out=dx, dact=dxa,
                       drop=self._drop(sv, "encoder.encoder.layers.%d.drop2" % (nl - 1)),
                       dgamma=gd["encoder.encoder.norm.weight"], dbeta=gd["encoder.encoder.norm.bias"])
            dlab_e1 = dlab_e
            if cfg.label_condition and G > 1:
                dlab_e1 = torch.zeros(nseq, cfg.dim_label, device=dev)
            dx = self._stack_bwd(sv, gd, "encoder.encoder", nl, dx, dxa, M1, L, nseq, sv.key_valid, lab=sv.lab_e1,
                                 dlab=dlab_e1, lab_rows_per_group=L)
            if cfg.label_condition and G > 1:
                ops.scatter_rows(dlab_e1, sv.label_e1, nseq, cfg.dim_label, gd["encoder.label_embedding.label_embedding.weight"])
            V, na = cfg.args_dim + 1, cfg.n_args
            scratch = torch.empty(na * V, d, device=dev)
            ops.embed_bwd(sv.commands, sv.args, sv.grp, dx, P("encoder.embedding.arg_embed.weight"),
                          P("encoder.embedding.embed_fcn.weight"), gd["encoder.embedding.command_embed.weight"],
                          gd["encoder.embedding.pos_encoding.pos_embed.weight"],
                          None if two else gd["encoder.embedding.group_embed.weight"],
                          gd["encoder.embedding.arg_embed.weight"], gd["encoder.embedding.embed_fcn.weight"],
                          gd["encoder.embedding.embed_fcn.bias"], scratch, nseq, L, V, na, d, cfg.max_num_groups + 2,
                          self._drop(sv, "enc.pe", 0.1))
            if cfg.label_condition:
                ops.scatter_rows(dlab_e, sv.label, N, cfg.dim_label, gd["encoder.label_embedding.label_embedding.weight"])

    # =================================================================================================
    # step execution: eager launches, or CUDA-graph replay of the captured launch sequences
    # =================================================================================================
    def _graph_key(self, inp):
        """Input signature a captured graph is valid for, or None when this call is not graphable."""
        if not self.graphs or self.self_match or self.autoregressive or not inp["training"] or not inp.get("need_grad", False) or inp["z"] is not None \
                or inp["encode_mode"] or inp["return_hierarch"] or ops.PROFILE is not None:
            return None
        c, a, lab = inp["commands"], inp["args"], inp["label"]
        if c.dtype != torch.float32 or a.dtype != torch.float32:
            return None
        if self._eps_override is not None:          # injected VAE noise (tests): a caller-owned tensor, not capturable
            return None
        ptrs = tuple(self._param(n).data_ptr() for n in self._pnames)
        return (tuple(c.shape), tuple(a.shape), None if lab is None else tuple(lab.shape), str(c.device), self.planes,
                hash(ptrs))

    def release_graphs(self):
        """Drops the captured step (and its private memory pool: activations of one step), and the decode caches and
        captured decode step of greedy_sample."""
        self._ds = None
        gs, self._gs = self._gs, None
        self._gs_streak = (None, 0)
        if gs is not None:
            gs.release()

    def _refresh_weights(self):
        """Re-cast every cached bf16 weight operand whose fp32 master changed (eager launches, outside the graphs)."""
        for name, dev in list(self._wcache):
            self._pack(name)

    def _run_forward(self, inp):
        key = self._graph_key(inp)
        gs = self._gs
        if key is None:
            return self._forward_impl(inp)
        if gs is not None and gs.key == key:
            return gs.replay_forward(inp)
        last, n = self._gs_streak
        n = n + 1 if last == key else 1
        self._gs_streak = (key, n)
        if n < 3:
            return self._forward_impl(inp)                      # warm-up: eager (also fills the weight-operand cache)
        if gs is not None:
            self._gs = None
            gs.release()
        try:
            gs = _GraphState(self, key, inp)
        except Exception as e:                                   # capture is an optimisation: fall back to eager launches
            import sys
            sys.stderr.write("deepsvg_b200: WARNING: CUDA-graph capture of the forward failed (%r); running eagerly\n" % (e,))
            self.graphs = False
            return self._forward_impl(inp)
        self._gs = gs
        return gs.replay_forward(inp)

    def _run_backward(self, sv, out_grads, g_token, gen):
        gs = getattr(sv, "graph", None)
        if gs is not None and gen != gs.gen:
            raise RuntimeError("deepsvg_b200: backward() of an earlier forward after a later one overwrote the captured "
                               "activations (CUDA-graph mode keeps ONE set of activation buffers); construct "
                               "SVGTransformer(..., graphs=False) for this usage")
        handle = getattr(sv, "handle", None)
        fused_only = (g_token is not None and handle is not None and handle.dl_args is not None
                      and all(g is None for g in out_grads))
        pg = self.process_group
        if gs is not None and fused_only and handle.bufs is gs.loss_bufs and gs.backward_ok:
            return gs.replay_backward(sv, out_grads, g_token)
        st = self._backward_a(sv, out_grads, g_token)
        flat, gd = st["flat"], st["gd"]
        work = None
        if pg is not None:
            import torch.distributed as dist
            split = self._bucket_split()
            # decoder gradients are final: their all-reduce runs on NCCL's stream while the encoder half computes
            work = dist.all_reduce(flat[split:], op=dist.ReduceOp.SUM, group=pg, async_op=True)
        self._backward_b(sv, st)
        if pg is not None:
            dist.all_reduce(flat[:split], op=dist.ReduceOp.SUM, group=pg)
            work.wait()
        if gs is None:
            sv.layers.clear()
            sv.__dict__.clear()     # release all saved activations now (the autograd node may outlive this call)
            return [gd[n] for n in self._pnames]
        return [g.clone() for g in (gd[n] for n in self._pnames)]


class _GraphState:
    """One captured train step: static input buffers, the forward graph, the two backward graphs (decoder half / encoder
    half, so that the gradient all-reduce of the decoder half overlaps the encoder half), and the saved-activation record
    whose tensors live in the graphs' private memory pool.  Outputs and activations are overwritten by every replay."""

    def __init__(self, model, key, inp):
        self.model, self.key = model, key
        self.gen = 0
        c, a, lab = inp["commands"], inp["args"], inp["label"]
        dev = c.device
        self.cmd, self.args = c.detach().clone().contiguous(), a.detach().clone().contiguous()
        self.label = lab.detach().clone() if lab is not None else None
        self.seed_dev = torch.zeros(1, dtype=torch.int64, device=dev)     # redrawn before every replay
        self.pool = torch.cuda.graph_pool_handle()
        self.bwd_a = self.bwd_b = None
        self.backward_ok = True
        self.bst = None
        model._refresh_weights()
        static = dict(inp, commands=self.cmd, args=self.args, label=self.label)
        torch.cuda.synchronize(dev)
        self.fwd = torch.cuda.CUDAGraph()
        from . import _lib
        n0 = _lib.launch_count()
        with torch.cuda.graph(self.fwd, pool=self.pool):
            outs, sv = model._forward_impl(static, seed_dev=self.seed_dev)
        self.n_fwd, self.n_bwd = _lib.launch_count() - n0, 0      # kernel nodes per replay
        self.outs, self.sv = outs, sv
        sv.graph = self
        # static buffers SVGLoss writes its outputs into (the backward graphs read them)
        cfg = model.cfg
        two = cfg.decode_stages == 2
        Md, nseq_d = sv.Md, sv.nseq_d
        na_out, nc = cfg.n_args * model.args_dim, cfg.n_commands
        pl = model.planes
        self.loss_bufs = dict(dl_args=Act(Md, na_out, pl, dev, ld=_r8(na_out)), dl_cmd=Act(Md, nc, pl, dev, ld=8),
                              dl_vis=Act(nseq_d, 2, pl, dev, ld=8) if two else None,
                              scales=torch.zeros(4, device=dev), loss_out=torch.zeros(8, device=dev))
        sv.loss_bufs = self.loss_bufs

    def release(self):
        self.fwd = self.bwd_a = self.bwd_b = None
        self.outs = self.sv = self.bst = self.loss_bufs = None

    def replay_forward(self, inp):
        m = self.model
        self.cmd.copy_(inp["commands"], non_blocking=True)
        self.args.copy_(inp["args"], non_blocking=True)
        if self.label is not None:
            self.label.copy_(inp["label"], non_blocking=True)
        self.seed_dev.random_()
        m._refresh_weights()
        self.fwd.replay()
        m.graph_kernel_launches += self.n_fwd
        self.gen += 1
        self.sv.gen = self.gen
        m._last_saved = self.sv
        return [t.detach() for t in self.outs], self.sv

    def replay_backward(self, sv, out_grads, g_token):
        m = self.model
        if self.bwd_a is None:
            try:
                torch.cuda.synchronize()
                ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                from . import _lib
                n0 = _lib.launch_count()
                with torch.cuda.graph(ga, pool=self.pool):
                    st = m._backward_a(sv, out_grads, g_token)
                with torch.cuda.graph(gb, pool=self.pool):
                    m._backward_b(sv, st)
                self.n_bwd = _lib.launch_count() - n0
                self.bwd_a, self.bwd_b, self.bst = ga, gb, st
            except Exception as e:
                import sys
                sys.stderr.write("deepsvg_b200: WARNING: CUDA-graph capture of the backward failed (%r); the backward runs "
                                 "eagerly\n" % (e,))
                self.backward_ok = False
                return m._run_backward(sv, out_grads, g_token, self.gen)
        flat, gd = self.bst["flat"], self.bst["gd"]
        pg = m.process_group
        self.bwd_a.replay()
        m.graph_kernel_launches += self.n_bwd
        work = None
        if pg is not None:
            import torch.distributed as dist
            split = m._bucket_split()
            work = dist.all_reduce(flat[split:], op=dist.ReduceOp.SUM, group=pg, async_op=True)
        self.bwd_b.replay()
        if pg is not None:
            dist.all_reduce(flat[:split], op=dist.ReduceOp.SUM, group=pg)
            work.wait()
        out = flat.clone()          # p.grad must not alias the buffer the next replay overwrites
        res, off = [], 0
        for n in m._pnames:
            p = m._param(n)
            res.append(out[off:off + p.numel()].view(p.shape))
            off += p.numel()
        return res


class _DecodeState:
    """Static buffers of cached decoding for one (N, precision, device, parameter storage): per-layer key/value caches, the
    step counter, token and bookkeeping buffers, the per-call refreshed inputs (folded embedding table, row vectors,
    temperature, seed), the head logits, and the captured decode step with its private memory pool."""

    def __init__(self, model, key, N, dev):
        cfg = model.cfg
        T, d, H, pl = cfg.max_total_len, cfg.d_model, cfg.n_heads, model.planes
        na, V = cfg.n_args, model.args_dim
        self.key, self.N, self.dev = key, N, dev
        self.sv = _Saved()
        self.sv.training = False
        self.step = torch.zeros(2, dtype=torch.int32, device=dev)            # t, block ticket
        self.cmd_in = torch.zeros(N, dtype=torch.int32, device=dev)
        self.args_in = torch.zeros(N, na, dtype=torch.int32, device=dev)
        self.grp = torch.zeros(N, dtype=torch.int32, device=dev)
        self.key_valid = torch.zeros(N, T, dtype=torch.uint8, device=dev)
        self.out_cmd = torch.zeros(N, T, dtype=torch.int64, device=dev)
        self.out_args = torch.zeros(N, T, na, dtype=torch.int64, device=dev)
        self.k_cache = [ops.decode_cache(N, H, d // H, T, pl, dev) for _ in range(cfg.n_layers_decode)]
        self.v_cache = [ops.decode_cache(N, H, d // H, T, pl, dev) for _ in range(cfg.n_layers_decode)]
        self.table = torch.empty(na * V, d, device=dev)
        self.base = torch.empty(d, device=dev)
        self.rowvec = [torch.empty(N, d, device=dev) for _ in range(cfg.n_layers_decode)]
        self.temperature = torch.zeros(1, device=dev)
        self.seed = torch.zeros(1, dtype=torch.int64, device=dev)
        self.cmd_logits = torch.empty(N, cfg.n_commands, device=dev)
        self.args_logits = torch.empty(N, na * V, device=dev)
        self.weights = ["decoder.fcn.command_fcn.weight", "decoder.fcn.args_fcn.weight"]
        for i in range(cfg.n_layers_decode):
            lp = "decoder.decoder.layers.%d." % i
            self.weights += [lp + n for n in ("self_attn.in_proj_weight", "self_attn.out_proj.weight", "linear1.weight",
                                              "linear2.weight", "linear_global.weight")]
            if cfg.label_condition:
                self.weights.append(lp + "linear_global2.weight")
        self.pool = torch.cuda.graph_pool_handle()
        self.graph, self.graph_failed, self.n_launches = None, False, 0
