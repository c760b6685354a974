"""ctypes signatures of every symbol declared in include/dsvg_b200.h (kept in the same order as the header).

tests/test_abi.py parses the header and checks that this table and the built library export exactly those names.
"""
import ctypes as C

P = C.c_void_p
I = C.c_int
F = C.c_float
Z = C.c_size_t
U32 = C.c_uint32
U64 = C.c_uint64
DROP = [F, U32, U64]

#: must equal dsvg_abi_version() of the loaded library (checked in _lib.load())
ABI_VERSION = 6

SIGNATURES = {
    "dsvg_abi_version": (I, []),
    "dsvg_linear": (I, [P, Z, I, P, Z, I, I, I, I, P, P]),
    "dsvg_outer": (I, [P, Z, I, P, Z, I, I, I, I, F, P, P, I, P, P]),
    "dsvg_outer_group": (I, [I, P, I, P]),
    "dsvg_linear_ln_fusable": (I, [I, I, I]),
    "dsvg_linear_ln_fwd": (I, [P, Z, I, P, Z, I, I, I, I, P, P, P, P, P, P, P]),
    "dsvg_pack_icons": (I, [P, P, I, I, I, I, P, P]),
    "dsvg_unpack_batch": (I, [P, P, P, P, Z, I, P]),
    "dsvg_match_assign": (I, [P, I, P, I, I, I, P, P, P, I, I, I, I, P, P, P, P, P, P]),
    "dsvg_permute_groups": (I, [P, P, P, I, I, Z, I, P]),
    "dsvg_seq_prep": (I, [P, I, I, P, P, P, P, P, P]),
    "dsvg_embed_fold": (I, [P, P, P, P, P, I, I, I, P]),
    "dsvg_embed_fwd": (I, [P, P, P, P, P, P, P, P, P, I, I, I, I, I] + DROP + [P]),
    "dsvg_embed_bwd": (I, [P, P, P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, I] + DROP + [P]),
    "dsvg_rows_embed_fwd": (I, [P, P, P, I, I, I] + DROP + [P]),
    "dsvg_rows_embed_bwd": (I, [P, P, P, I, I, I] + DROP + [P]),
    "dsvg_ln_fwd": (I, [P, P, P, P, Z, P, P, I, I, P]),
    "dsvg_ln_pool_fwd": (I, [P, P, P, P, P, P, P, P, I, I, I, P]),
    "dsvg_ln_bwd": (I, [P, P, P, P, P, Z, P, P, P, I, P, P, P, Z] + DROP + [P, P, I, I, P]),
    "dsvg_attn_fwd": (I, [P, Z, P, P, Z, I, I, I, I, I] + DROP + [P]),
    "dsvg_attn_bwd": (I, [P, Z, P, P, Z, P, Z, I, I, I, I, I, F] + DROP + [P]),
    "dsvg_decode_embed": (I, [P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, P]),
    "dsvg_decode_attn": (I, [P, P, Z, P, P, Z, P, P, Z, I, I, I, I, P]),
    "dsvg_decode_sample": (I, [P, P, I, P, I, P, P, P, P, P, P, I, I, I, I, I, P]),
    "dsvg_ce_args": (I, [P, I, P, P, P, P, Z, I, P, I, I, I, I, P]),
    "dsvg_ce_cmd": (I, [P, P, P, P, P, P, Z, I, P, I, I, I, P]),
    "dsvg_ce_vis": (I, [P, P, P, Z, I, P, I, F, P]),
    "dsvg_kl_sum": (I, [P, P, P, I, P]),
    "dsvg_loss_finalize": (I, [P, P, P, F, F, F, F, F, F, F, I, I, P]),
    "dsvg_vae_fwd": (I, [P, P, P, P, I, P]),
    "dsvg_vae_bwd": (I, [P, P, P, P, P, P, F, P, P, I, P]),
    "dsvg_cast_act": (I, [P, I, I, I, P, Z, I, P, Z, I, P, Z, I, F] + DROP + [P]),
    "dsvg_colsum": (I, [P, Z, I, I, I, P, P, P]),
    "dsvg_seg_sum": (I, [P, I, I, I, P, Z, P] + DROP + [P]),
    "dsvg_gather_rows": (I, [P, P, I, I, I, P, Z, P]),
    "dsvg_scatter_rows": (I, [P, P, I, I, I, P, P]),
    "dsvg_add_f32": (I, [P, P, P, Z, P]),
    "dsvg_grad_sqnorm": (I, [P, I, I, P, P]),
    "dsvg_adamw_step": (I, [P, I, I, F, F, F, F, F, F, F, F, P, P]),
}
