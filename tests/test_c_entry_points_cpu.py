"""CPU tests of the C entry points themselves, through ctypes, without a GPU.

``lib.SIGNATURES`` types every entry point of every ``include/tfimm_b200*.h``: the headers must declare exactly what
the table and the built library hold, each parameter of the kind ctypes passes.

Called with all-zero arguments (null pointers, 0, 0.0), every entry point must stop at its own argument check, before
it touches CUDA, and report its own status and message.  A wrong pairing of entry point and body, or arguments shifted
by one, changes the pair.  The core entries were recorded from the library as built before the entry points moved next
to their kernels, each family's from the library that added it.
"""
import ctypes
import re
import subprocess
from pathlib import Path

from tfimm.backend import lib, ops

ROOT = Path(__file__).resolve().parent.parent

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
    # include/tfimm_b200_poolformer.h
    "gn1_partials": (1, "gn1_partials: need B, H, W > 0 and C % 4 == 0 (B=0 H=0 W=0 C=0)"),
    "poolformer_mixer": (1, "poolformer_mixer: need B, H, W > 0 and C % 4 == 0 (B=0 H=0 W=0 C=0)"),
    "gn1_apply": (1, "gn1_apply: need B, H, W > 0 and C % 4 == 0 (B=0 H=0 W=0 C=0)"),
    # include/tfimm_b200_pit.h
    "pit_attention_bf16": (1, "pit_attention_bf16: bad shape B=0 T=0 H=0"),
    "pit_pool": (1, "pit_pool: need B, H, W > 0, C % 4 == 0 and nb_tokens >= 0 (B=0 H=0 W=0 C=0 nb_tokens=0)"),
    # include/tfimm_b200_convmixer.h
    "convmixer_dwconv": (1, "convmixer_dwconv: need B, H, W, C > 0 (B=0 H=0 W=0 C=0)"),
    # include/tfimm_b200_pvt.h
    "pvt_sr_attention_bf16": (1, "pvt_sr_attention_bf16: bad shape B=0 N=0 Nk=0 H=0"),
    "pvt_sr_attention_f32": (1, "pvt_sr_attention_f32: bad shape B=0 N=0 Nk=0 H=0"),
    "pvt_embed_norm": (1, "pvt_embed_norm: need B, P > 0, ntok 0 or 1, C % 4 == 0 and C <= 1024 "
                          "(B=0 P=0 ntok=0 C=0)"),
    # include/tfimm_b200_pvt_v2.h
    "pvt_v2_conv_mlp_bf16": (3, "pvt_v2_conv_mlp_bf16: needs C in {32, 64, 128} and hidden % 64 == 0 "
                                "(got C=0 hidden=0)"),
    "pvt_v2_sr_attention_bf16": (1, "pvt_v2_sr_attention_bf16: bad shape B=0 N=0 Nk=0 H=0"),
    "pvt_v2_sr_attention_f32": (1, "pvt_v2_sr_attention_f32: bad shape B=0 N=0 Nk=0 H=0"),
    # include/tfimm_b200_cait.h
    "cait_talking_heads_bf16": (1, "cait_talking_heads_bf16: bad shape B=0 N=0 H=0"),
    "cait_talking_heads_f32": (1, "cait_talking_heads_f32: bad shape B=0 N=0 H=0"),
    "cait_class_attention": (1, "cait_class_attention: bad shape B=0 T=0 H=0"),
    "cait_add_pos": (1, "cait_add_pos: need B, N > 0 and D % 4 == 0 (B=0 N=0 D=0)"),
}

# entry points whose launches bench.py's roofline (and tools/ncu_traffic.py) count under another kernel family
OTHER_FAMILY = {
    "conv_bf16": "gemm_bf16",
    "gemm_bf16_gated": "gemm_bf16",
    "window_attention_tc_bf16": "window_attention_bf16",
    "im2col_u8": "im2col",
}

PREFIX = "tfimm_b200_"
# the declaration of each entry point: "int" (a status) or "const char*" (version, last_error) at the start of a line
DECLARATION = r"^(?:int|const char\*) ({})\("


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


def _argtype(param):
    """The ctypes type of a C parameter: a float passed as int, or a 64-bit stride passed as int, would be silent
    garbage through ctypes."""
    return ctypes.c_void_p if "*" in param else ctypes.c_float if param.startswith("float") else \
        ctypes.c_long if param.startswith("long") else ctypes.c_int


def test_headers_declare_exactly_the_ctypes_table_and_the_library_exports_it():
    """The .so loads without a GPU.  Across include/tfimm_b200*.h every name is declared once, the declarations are
    exactly ``lib.exported_symbols()`` (which also catches a name repeated in ``lib.SIGNATURES``'s literal, where the
    later row silently replaces the earlier), the library exports each of them, and every parameter is of the kind its
    ctypes argtype passes."""
    handle = lib.load()
    header = "\n".join(p.read_text() for p in sorted((ROOT / "include").glob("tfimm_b200*.h")))
    declared = re.findall(DECLARATION.format(r"tfimm_b200_\w+"), header, re.M)
    assert len(declared) == len(set(declared)), sorted(n for n in set(declared) if declared.count(n) > 1)
    assert set(declared) == set(lib.exported_symbols()), set(declared) ^ set(lib.exported_symbols())
    nm = subprocess.run(["nm", "-D", "--defined-only", str(lib.LIB_PATH)], capture_output=True, text=True).stdout
    exported = set(re.findall(r"\sT\s+(tfimm_b200_\w+)", nm))
    assert set(declared) <= exported, set(declared) - exported
    for name, argtypes in lib.SIGNATURES.items():
        params = re.search(DECLARATION.format(name) + r"([^;]*?)\)\s*;", header, re.M | re.S).group(2).split(",")
        assert [_argtype(p.strip()) for p in params] == argtypes, name
    assert handle.tfimm_b200_version().decode().startswith("tfimm_b200")
