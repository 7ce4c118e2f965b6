"""ctypes binding of ``libtfimm_b200.so`` (C ABI declared in ``include/tfimm_b200.h`` and the family headers
``include/tfimm_b200_<family>.h``).

The shared object is built in-tree by ``tensorflow-image-models_b200/build.py``.  Loading it
does not need a GPU (cudart is linked statically and the driver entry points are resolved
lazily), so the CPU test-suite can check that every declared symbol is exported.  There is
no CPU fallback: if the library is missing, every kernel call raises.
"""
import contextvars
import ctypes
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libtfimm_b200.so"

# dtype / activation codes (mirror include/tfimm_b200.h)
F32, BF16, U8 = 0, 1, 2
ACT = {
    None: 0, "": 0, "linear": 0, "none": 0,
    "gelu": 1, "swish": 2, "silu": 2, "relu": 3, "relu6": 4, "tanh": 5, "sigmoid": 6,
}

_c = ctypes
_P = _c.c_void_p
_I = _c.c_int
_L = _c.c_long
_F = _c.c_float

# name -> argtypes; restype is int (status) unless listed in _SPECIAL
SIGNATURES = {
    # include/tfimm_b200.h
    "tfimm_b200_gemm_bf16": [_P, _I, _P, _I, _P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_conv_bf16": [_P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_gemm_f32": [_P, _I, _P, _I, _P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_gemm_tf32": [_P, _I, _P, _I, _P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_conv_tf32": [_P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_attention_tf32": [_P, _P, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_layernorm": [_P, _I, _L, _P, _P, _P, _I, _L, _L, _I, _F, _P],
    "tfimm_b200_layernorm_patch2x2": [_P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_patch_merge_ln": [_P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_attention_bf16": [_P, _P, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_attention_cls_bf16": [_P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_attention_f32": [_P, _P, _P, _P, _I, _L, _I, _I, _I, _F, _P, _P, _I, _P],
    "tfimm_b200_window_attention_bf16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_window_attention_tc_bf16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_gemm_bf16_gated": [_P, _I, _P, _I, _I, _P, _I, _P, _P, _I, _P, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_mlp_bf16": [_P, _I, _P, _I, _P, _P, _I, _P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_patchify": [_P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _F, _P, _P, _P],
    "tfimm_b200_assemble_tokens": [_P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_cast": [_P, _I, _P, _I, _L, _P],
    "tfimm_b200_dwconv_ln": [_P, _I, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_dwconv_bias_act": [_P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_global_avg_pool": [_P, _I, _P, _I, _I, _I, _P],
    "tfimm_b200_im2col": [_P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_im2col_u8": [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P, _P, _P],
    "tfimm_b200_group_norm": [_P, _I, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _I, _P],
    "tfimm_b200_blur_pool": [_P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_se_gate": [_P, _F, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_scale_channels": [_P, _I, _P, _I, _I, _I, _P],
    "tfimm_b200_pool2d": [_P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_grouped_conv": [_P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_eca_gate": [_P, _P, _P, _I, _I, _I, _P],
    "tfimm_b200_scale_add_act": [_P, _I, _P, _P, _I, _I, _I, _I, _P],
    "tfimm_b200_relpos_attention_bf16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_relpos_attention_f32": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_token_gemm_bf16": [_P, _I, _P, _L, _L, _P, _P, _P, _L, _L, _P, _L, _L, _P, _L, _L, _I, _I, _I, _I,
                                   _I, _I, _I, _I, _I, _P],
    "tfimm_b200_token_gemm_f32": [_P, _I, _P, _L, _L, _P, _P, _P, _L, _L, _P, _L, _L, _P, _L, _L, _I, _I, _I, _I,
                                  _I, _I, _I, _P],
    "tfimm_b200_gemm_glu_bf16": [_P, _I, _P, _I, _P, _P, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_gemm_glu_f32": [_P, _I, _P, _I, _P, _P, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_affine": [_P, _L, _P, _P, _P, _I, _L, _L, _I, _P],
    # include/tfimm_b200_poolformer.h
    "tfimm_b200_gn1_partials": [_P, _P, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_poolformer_mixer": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_gn1_apply": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P],
    # include/tfimm_b200_pit.h
    "tfimm_b200_pit_attention_bf16": [_P, _P, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_pit_pool": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    # include/tfimm_b200_convmixer.h
    "tfimm_b200_convmixer_dwconv": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P],
    # include/tfimm_b200_pvt.h
    "tfimm_b200_pvt_sr_attention_bf16": [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_pvt_sr_attention_f32": [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_pvt_embed_norm": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P],
    # include/tfimm_b200_pvt_v2.h
    "tfimm_b200_pvt_v2_conv_mlp_bf16": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P],
    "tfimm_b200_pvt_v2_sr_attention_bf16": [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_pvt_v2_sr_attention_f32": [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    # include/tfimm_b200_cait.h
    "tfimm_b200_cait_talking_heads_bf16": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "tfimm_b200_cait_talking_heads_f32": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "tfimm_b200_cait_class_attention": [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "tfimm_b200_cait_add_pos": [_P, _P, _I, _I, _I, _P],
}
_SPECIAL = {
    "tfimm_b200_version": ([], _c.c_char_p),
    "tfimm_b200_last_error": ([], _c.c_char_p),
    "tfimm_b200_sm_count": ([], _I),
}

_lib = None

# precision="tf32": while set, the fp32 launchers of ``tfimm.backend.ops`` whose contraction has a TF32 tensor-core kernel
# (gemm, conv_gemm, ViT attention) run it instead of the fp32 SIMT kernel.  A model's public forward entry points
# (``call``, ``forward_features``: see ``Model.__init_subclass__``) set it to whether the model is a tf32 model and reset
# it afterwards; a context variable, so threads and asyncio tasks each see their own.
tf32_mode = contextvars.ContextVar("tfimm_tf32_mode", default=False)


def round_tf32(t):
    """fp32 tensor -> the nearest TF32 value (10 explicit mantissa bits, low 13 bits zero), ties away from zero: what
    ``cvt.rna.tf32.f32`` computes inside the TF32 kernels.  Finite values at the top of the range round to +-inf;
    inf and NaN pass through.  Used for GEMM weights, which are rounded once when the plan is built."""
    import torch

    assert t.dtype == torch.float32, t.dtype
    bits = t.contiguous().view(torch.int32)
    finite = (bits & 0x7F800000) != 0x7F800000
    # adding half a TF32 ulp to the magnitude bits and truncating rounds the magnitude half away from zero; a carry
    # out of the mantissa correctly bumps the exponent (and the largest binade into inf)
    rounded = (bits + 0x1000) & ~0x1FFF
    return torch.where(finite, rounded, bits).view(torch.float32)


class KernelLibraryError(RuntimeError):
    pass


def exported_symbols():
    """All symbol names the headers declare (used by the CPU test-suite)."""
    return sorted(list(SIGNATURES) + list(_SPECIAL))


def load():
    """Loads the shared library (building it first if the build tree is writable and it is
    missing).  Raises ``KernelLibraryError`` -- never falls back to another implementation."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("TFIMM_B200_LIB", LIB_PATH))
    if not path.exists():
        raise KernelLibraryError(
            f"{path} not found. Build it with `python tensorflow-image-models_b200/build.py` "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). "
            "tfimm_b200 has no CPU / eager fallback."
        )
    lib = ctypes.CDLL(str(path))
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = _I
    for name, (argtypes, restype) in _SPECIAL.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = restype
    _lib = lib
    return lib


def check(status: int, what: str):
    if status != 0:
        msg = load().tfimm_b200_last_error().decode("utf-8", "replace")
        raise KernelLibraryError(f"{what} failed (status {status}): {msg}")
