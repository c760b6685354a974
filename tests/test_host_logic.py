"""CPU: host-side logic of the drop-in modules (no kernels): parameter inventory, state_dict compatibility with the
reference (via the golden fixtures' parameter names), config mirror, rejection of unsupported variants, init rules."""
import pytest
import torch

from oracle import svg_oracle as O
from tests.golden_cases import CASES, load_case


def _mk(kind, over):
    from deepsvg_b200 import SVGTransformer
    from deepsvg_b200.config import _DefaultConfig
    o = O.make_cfg(kind, **over)
    return SVGTransformer(_DefaultConfig(**vars(o))), o


@pytest.mark.parametrize("kind,over", [("hierarchical", dict(use_vae=False)),
                                       ("hierarchical", dict(use_vae=False, self_match=True)),
                                       ("hierarchical", dict(label_condition=True, n_labels=62, dim_z=128)),
                                       ("one_stage", dict(label_condition=True, n_labels=52, max_total_len=50))])
def test_parameter_inventory_matches_oracle_and_reference_names(kind, over):
    model, o = _mk(kind, over)
    mine = {k: tuple(v.shape) for k, v in model.named_parameters()}
    assert mine == O.param_shapes(o) and list(mine) == list(O.param_shapes(o))


def test_state_dict_keys_match_reference_golden():
    cfg, fx, _ = load_case("hier_cfg1")          # param_names were read from the real reference module
    from deepsvg_b200 import SVGTransformer
    from deepsvg_b200.config import _DefaultConfig
    model = SVGTransformer(_DefaultConfig(**vars(cfg)))
    assert sorted(k for k, _ in model.named_parameters()) == list(fx["param_names"])
    sd = model.state_dict()
    assert len(sd) == 247 and sum(p.numel() for p in model.parameters()) == 10304596   # SURVEY.md 8b [probe]
    assert sd["cmd_args_mask"].dtype == torch.int64 and tuple(sd["cmd_args_mask"].shape) == (7, 11)
    assert tuple(sd["encoder.embedding.pos_encoding.position"].shape) == (32, 1)
    assert tuple(sd["decoder.embedding.PE.position"].shape) == (31, 1)


def test_layers_of_a_stack_start_identical_and_vae_init():
    model, _ = _mk("hierarchical", dict(use_vae=True))
    sd = model.state_dict()
    for stack in ("encoder.encoder", "decoder.decoder"):
        for leaf in ("self_attn.in_proj_weight", "linear1.weight", "linear2.bias"):
            assert torch.equal(sd["%s.layers.0.%s" % (stack, leaf)], sd["%s.layers.3.%s" % (stack, leaf)])
    assert sd["vae.enc_mu_fcn.weight"].std().item() < 2e-3 and sd["vae.enc_mu_fcn.bias"].abs().max().item() == 0
    assert sd["encoder.encoder.layers.0.self_attn.in_proj_bias"].abs().max().item() == 0


def test_config_mirror_and_model_args():
    from deepsvg_b200 import Hierarchical, OneStageOneShot
    h = Hierarchical()
    assert (h.encode_stages, h.decode_stages, h.max_total_len, h.num_groups_proposal) == (2, 2, 240, 8)
    assert h.get_model_args() == ["commands", "args", "commands", "args"]
    o = OneStageOneShot(label_condition=True)
    assert o.get_model_args() == ["commands_grouped", "args_grouped", "commands_grouped", "args_grouped", "label"]


@pytest.mark.parametrize("over", [dict(model_type="lstm"), dict(pred_mode="autoregressive"),   # (two-stage autoregressive)
                                  dict(self_match=True, num_groups_proposal=20, max_num_groups=20), dict(d_model=192),
                                  dict(encode_stages=2, decode_stages=1)])
def test_unsupported_variants_raise_at_construction(over):
    from deepsvg_b200 import Hierarchical, SVGTransformer
    with pytest.raises(NotImplementedError):
        SVGTransformer(Hierarchical(**over))


def test_attention_length_limit_matches_the_shared_memory_formula():
    """The longest sequence per head_dim is the largest L whose SIMT-backward tiles (Q, K, V, dO: L x hd; P, dS: L x (L | 1),
    fp32) fit the 227 KB opt-in shared memory; one more position raises at construction, and the message quotes the
    limits in tokens (two positions fewer: SOS and EOS)."""
    import re
    from deepsvg_b200 import OneStageOneShot, SVGTransformer
    from deepsvg_b200.config import check_supported
    from tests.test_kernels_gpu import ATTN_MAX_L

    def fits(L, hd):
        return 4 * (4 * L * hd + 2 * L * (L | 1) + 3) <= 227 * 1024

    for hd, L in ATTN_MAX_L.items():
        assert fits(L, hd) and not fits(L + 1, hd), hd
        check_supported(OneStageOneShot(d_model=128, n_heads=128 // hd, max_total_len=L - 2))
        with pytest.raises(NotImplementedError) as e:
            SVGTransformer(OneStageOneShot(d_model=128, n_heads=128 // hd, max_total_len=L - 1))
        quoted = re.search(r"limits: (\d+) / (\d+) / (\d+) tokens for head_dim 16 / 32 / 64", str(e.value))
        assert quoted and [int(t) for t in quoted.groups()] == [ATTN_MAX_L[h] - 2 for h in (16, 32, 64)], str(e.value)


def test_self_matching_variant_is_constructible_and_has_no_path_positional_code():
    """model/config.py:101-108, model.py:114-115."""
    from deepsvg_b200 import HierarchicalSelfMatching, OneStageOneShot, SVGTransformer
    m = SVGTransformer(HierarchicalSelfMatching(use_vae=False))
    names = dict(m.named_parameters())
    assert "encoder.hierarchical_PE.pos_embed.weight" not in names and "decoder.hierarchical_embedding.PE.pos_embed.weight" in names
    cfg, fx, _ = load_case("selfmatch_d128")
    from deepsvg_b200.config import _DefaultConfig
    m2 = SVGTransformer(_DefaultConfig(**vars(cfg)))
    assert sorted(k for k, _ in m2.named_parameters()) == list(fx["param_names"])     # names read from the real reference
    with pytest.raises(NotImplementedError):
        SVGTransformer(OneStageOneShot(self_match=True, max_total_len=50))


def test_sketchformer_variant_matches_reference_parameter_names():
    """model/config.py:74-80: autoregressive decoder with its own SVGEmbedding, 2 * args_dim classes (rel_targets)."""
    from deepsvg_b200 import Sketchformer, SVGTransformer
    from deepsvg_b200.config import _DefaultConfig
    cfg, fx, _ = load_case("sketchformer_d128")
    m = SVGTransformer(_DefaultConfig(**vars(cfg)))
    assert sorted(k for k, _ in m.named_parameters()) == list(fx["param_names"])     # names read from the real reference
    sd = m.state_dict()
    assert tuple(sd["decoder.embedding.arg_embed.weight"].shape) == (512, 64)
    assert tuple(sd["decoder.fcn.args_fcn.weight"].shape) == (11 * 512, 128)
    assert tuple(sd["decoder.square_subsequent_mask"].shape) == (31, 31) and sd["decoder.square_subsequent_mask"][0, 1] == float("-inf")
    assert Sketchformer(max_total_len=50).get_model_args() == ["commands_grouped", "args_grouped", "commands_grouped",
                                                                "args_rel_grouped"]
    with pytest.raises(NotImplementedError):     # default Sketchformer: 240-token sequences exceed the attention tile
        SVGTransformer(Sketchformer())


def test_golden_cases_cover_all_reference_branches():
    kinds = {(c[0], c[1].get("use_vae", True), c[1].get("label_condition", False)) for c in CASES.values()}
    assert ("hierarchical", False, False) in kinds and ("hierarchical", True, True) in kinds
    assert ("one_stage", True, True) in kinds
