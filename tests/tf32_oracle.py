"""TEST INFRASTRUCTURE ONLY -- precision="tf32" on top of oracle/emulate_bf16.py and oracle/shadow.py.

A tf32 model stores everything in fp32, like an fp32 model; only its contractions differ: ``ops.gemm``,
``ops.conv_gemm`` and the plain ViT ``ops.attention`` (head_dim 64; no bias / mask / probs / row map) run TF32 tensor-core
kernels whose operands are rounded to TF32 (round to nearest, ties away from zero) and whose products accumulate in
fp32.  Inside ``tf32_oracle()``:

* the emulation's statements of those three launchers round their operands the same way -- both GEMM / convolution
  operands (the weights already are), q, k and v, and the softmax numerator P before P V -- and then compute exactly as
  before (float64);
* the shadow harness's rules for them bound the kernel against that emulation: the fp32 accumulation of exact TF32
  products (``shadow._UT`` per term, the tensor core truncates), no storage ulp (outputs are fp32), and for attention
  ``shadow._blocked_softmax_err`` with TF32's spacing of P -- the statement runs the kernel's online softmax over 64-key
  blocks.

Both take the tf32 branch only while a tf32 model's forward pass runs (``tfimm.backend.lib.tf32_mode``) and the operands
are fp32; every other call is the unchanged statement and rule.  Enter it outside ``emulated_ops()`` /
``shadowed_ops()``, which capture the statements and rules on entry.
"""
from contextlib import contextmanager

import torch

from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64


def round_tf32(t):
    from tfimm.backend.lib import round_tf32 as r

    return r(t)


def round_p_tf32(p):
    """P as the TF32 P V product sees it (``cvt.rna`` of the fp32 value), kept in p's dtype."""
    return round_tf32(p.float()).to(p.dtype)


def _tf32_on(*tensors):
    from tfimm.backend.lib import tf32_mode

    return tf32_mode.get() and all(t.dtype == torch.float32 for t in tensors)


def _plain_attention(qkv, dh, bias, mask, probs, row_map):
    return _tf32_on(qkv) and dh == 64 and bias is None and mask is None and probs is None and row_map is None


# --------------------------------------------------------------------------------------------------- the emulation
def _emu_gemm(base):
    def gemm(a, w, bias=None, act=None, gamma=None, residual=None, out=None, out_dtype=None, block_n=0,
             act_after_residual=False):
        if _tf32_on(a, w):
            a, w = round_tf32(a), round_tf32(w)
        return base(a, w, bias=bias, act=act, gamma=gamma, residual=residual, out=out, out_dtype=out_dtype,
                    block_n=block_n, act_after_residual=act_after_residual)
    return gemm


def _emu_conv_gemm(base):
    def conv_gemm(x, w, bias=None, ks=3, stride=1, pad=1, act=None, residual=None, act_after_residual=False,
                  out_dtype=None):
        if _tf32_on(x, w):
            x, w = round_tf32(x), round_tf32(w)
        return base(x, w, bias=bias, ks=ks, stride=stride, pad=pad, act=act, residual=residual,
                    act_after_residual=act_after_residual, out_dtype=out_dtype)
    return conv_gemm


def _emu_attention(base):
    def attention(qkv, B, N, H, dh, scale, bias=None, mask=None, probs=None, row_map=None, nw_img=0):
        if not _plain_attention(qkv, dh, bias, mask, probs, row_map):
            return base(qkv, B, N, H, dh, scale, bias=bias, mask=mask, probs=probs, row_map=row_map, nw_img=nw_img)
        q, k, v = round_tf32(qkv).to(emu._HP).view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
        # the kernel's online softmax: P rounded to TF32 per 64-key block, the row sum of the unrounded P
        o = torch.cat([emu._softmax_pv(scale * (q[c] @ k[c].transpose(-1, -2)), v[c], round_p_tf32, emu.KEY_BLOCK)[0]
                       for c in emu.image_chunks(B, H, N)])
        return o.permute(0, 2, 1, 3).reshape(B * N, H * dh).contiguous().to(qkv.dtype)
    return attention


# ------------------------------------------------------------------------------------------------------ the rules
def _rule_gemm(base):
    def rule(A):
        a, w = A["a"], A["w"]
        if not _tf32_on(a, w):
            return base(A)
        S = round_tf32(a).abs().to(_F64) @ round_tf32(w).abs().to(_F64).t()
        if A["bias"] is not None:
            S = S + shadow._a(A["bias"])
        # TF32 x TF32 products are exact in fp32 (11 x 11 significant bits); the tensor core adds them with truncation
        return [("out", shadow._ret, shadow._bounded(
            shadow._epilogue(S, a.shape[1] + 1, shadow._UT, A["act"], A["gamma"], A["residual"])))]
    return rule


def _rule_conv_gemm(base):
    def rule(A):
        x, w = A["x"], A["w"]
        if not _tf32_on(x, w):
            return base(A)
        S = emu.conv_gemm(round_tf32(x).abs().to(_F64), round_tf32(w).abs().to(_F64), bias=shadow._a(A["bias"]),
                          ks=A["ks"], stride=A["stride"], pad=A["pad"], out_dtype=_F64)
        n = A["ks"] * A["ks"] * x.shape[-1] + 1
        return [("out", shadow._ret, shadow._bounded(shadow._epilogue(S, n, shadow._UT, A["act"], None, A["residual"])))]
    return rule


def _rule_attention(base):
    def rule(A):
        qkv, B, N, H, dh = A["qkv"], A["B"], A["N"], A["H"], A["dh"]
        if not _plain_attention(qkv, dh, A["bias"], A["mask"], A["probs"], A["row_map"]):
            return base(A)
        # The bf16 branch's bound with P rounded to TF32 (its spacing 2^(e-11)) and q, k, v rounded on both sides; the
        # output is fp32: its own rounding is the final product's, part of the bound.
        bound = shadow._blocked_attention_bound(round_tf32(qkv), B, N, H, dh, A["scale"], round_p_tf32)
        return [("out", shadow._ret, shadow._bounded(bound))]
    return rule


_EMU = {"gemm": _emu_gemm, "conv_gemm": _emu_conv_gemm, "attention": _emu_attention}
_RULE = {"gemm": _rule_gemm, "conv_gemm": _rule_conv_gemm, "attention": _rule_attention}


@contextmanager
def tf32_oracle():
    saved_emu = {n: getattr(emu, n) for n in _EMU}
    saved_rules = {n: shadow._RULES[n] for n in _RULE}
    for n, make in _EMU.items():
        setattr(emu, n, make(saved_emu[n]))
    for n, make in _RULE.items():
        shadow._RULES[n] = make(saved_rules[n])
    try:
        yield
    finally:
        for n, f in saved_emu.items():
            setattr(emu, n, f)
        shadow._RULES.update(saved_rules)
