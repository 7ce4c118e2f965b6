"""CPU tests of the C entry points themselves, through ctypes, without a GPU.

Called with all-zero arguments (null pointers, 0, 0.0), every entry point must stop at its own argument check, before
it touches CUDA, and report its own status and message.  A wrong pairing of entry point and body, or arguments shifted
by one, changes the pair.  The table was recorded from the library as built before the entry points moved next to
their kernels.
"""
import ctypes

from tfimm.backend import lib, ops

ZERO_CALL = {
    "gemm_bf16": (1, "gemm: M, N, K must be positive (got 0 0 0)"),
    "conv_bf16": (1, "conv: C must be a multiple of 64 (got 0)"),
    "gemm_f32": (1, "gemm_f32: M, N, K must be positive"),
    "gemm_tf32": (1, "gemm_tf32: M, N, K must be positive (got 0 0 0)"),
    "conv_tf32": (1, "conv: C must be a multiple of 32 (got 0)"),
    "attention_tf32": (1, "attention_tf32: bad shape B=0 N=0 H=0"),
    "layernorm": (1, "layernorm: need rows>0 and C%8==0 (rows=0 C=0)"),
    "layernorm_patch2x2": (1, "layernorm_patch2x2: need even H, W and C%8==0 (H=0 W=0 C=0)"),
    "patch_merge_ln": (1, "patch_merge_ln: need even H, W and C%8==0 (H=0 W=0 C=0)"),
    "attention_bf16": (1, "attention: bad shape B=0 N=0 H=0"),
    "attention_cls_bf16": (1, "attention_cls: bad shape"),
    "attention_f32": (1, "attention_f32: bad shape"),
    "window_attention_bf16": (1, "window_attention: bad shape"),
    "window_attention_tc_bf16": (1, "window_attention: bad shape"),
    "gemm_bf16_gated": (1, "gemm_gated: need K % 8 == 0 (got M=0 N=0 K=0)"),
    "mlp_bf16": (3, "mlp_fused: needs C in {96, 128, 192, 256} and hidden % 128 == 0, >= 256 (got C=0 hidden=0)"),
    "patchify": (1, "patchify: H, W must be multiples of the patch size (H=0 W=0 p=0)"),
    "assemble_tokens": (1, "assemble_tokens: bad shape"),
    "cast": (1, "cast: n must be positive"),
    "dwconv_ln": (1, "dwconv_ln: need C%4==0 (C=0)"),
    "dwconv_bias_act": (1, "dwconv: need C%4==0 (C=0)"),
    "global_avg_pool": (1, "global_avg_pool: need C%4==0"),
    "im2col": (1, "im2col: bad geometry"),
    "im2col_u8": (1, "im2col: bad geometry"),
    "group_norm": (1, "group_norm: need C%groups==0 and C%8==0 (C=0 groups=0)"),
    "blur_pool": (1, "blur_pool: need H,W>1 and C%8==0 (C=0)"),
    "se_gate": (1, "se_gate: bad shape"),
    "scale_channels": (1, "scale_channels: need C%8==0 (C=0)"),
    "pool2d": (1, "pool2d: need C%8==0 (C=0)"),
    "grouped_conv": (1, "grouped_conv: bad channel grouping (C=0 cg=0)"),
    "eca_gate": (1, "eca_gate: need an odd kernel size"),
    "scale_add_act": (1, "scale_add_act: need C%8==0 (C=0)"),
    "relpos_attention_bf16": (1, "relpos_attention: bad shape B=0 grid=0x0 H=0 dh=0 window=0"),
    "relpos_attention_f32": (1, "relpos_attention: bad shape B=0 grid=0x0 H=0 dh=0 window=0"),
    "token_gemm_bf16": (1, "token_gemm: empty shape (imgs 0 M 0 N 0 K 0)"),
    "token_gemm_f32": (1, "token_gemm_f32: bad shape (imgs 0 M 0 N 0 K 0)"),
    "gemm_glu_bf16": (1, "gemm_glu: need K % 8 == 0 and an even N (got M=0 N=0 K=0)"),
    "gemm_glu_f32": (1, "gemm_glu_f32: need N % 16 == 0 and n_out <= N / 2 (got N 0, n_out 0)"),
    "affine": (1, "affine: bad shape"),
}

# entry points whose launches bench.py's roofline (and tools/ncu_traffic.py) count under another kernel family
OTHER_FAMILY = {
    "conv_bf16": "gemm_bf16",
    "gemm_bf16_gated": "gemm_bf16",
    "window_attention_tc_bf16": "window_attention_bf16",
    "im2col_u8": "im2col",
}

PREFIX = "tfimm_b200_"


def test_every_entry_point_rejects_all_zero_arguments_with_its_own_message():
    handle = lib.load()
    assert {PREFIX + n for n in ZERO_CALL} == set(lib.SIGNATURES)
    got = {}
    for name, argtypes in lib.SIGNATURES.items():
        args = [None if t is ctypes.c_void_p else 0.0 if t is ctypes.c_float else 0 for t in argtypes]
        status = getattr(handle, name)(*args)
        got[name[len(PREFIX):]] = (status, handle.tfimm_b200_last_error().decode())
    assert got == ZERO_CALL


def test_trace_family_of_every_entry_point():
    want = {PREFIX + n: OTHER_FAMILY.get(n, n) for n in ZERO_CALL}
    assert ops.TRACE_FAMILY == want
