"""TEST INFRASTRUCTURE ONLY -- the PVT launchers (``tfimm.backend.pvt_ops``) on top of oracle/emulate_bf16.py and
oracle/shadow.py.

Each launcher gets
* a statement at the kernels' storage points, in the emulation's arithmetic (float64 by default):
  - ``pvt_sr_attention_bf16``: the bf16 q and kv as stored, kv read as (B, N', 2, H, dh); softmax(scale q k^T) v with
    P rounded to bf16 per 64-key block of an online softmax (``emulate_bf16._softmax_pv(.., round_bf16, 64)``, the
    tensor-core kernels' algorithm), one rounding of the output to bf16.  With q and kv cut from one packed qkv this is
    ``emulate_bf16.attention`` itself;
  - ``pvt_sr_attention_f32``: softmax(scale q k^T) v of the fp32 q and kv, exactly, one rounding to fp32;
  - ``pvt_embed_norm``: the reference's LayerNorm of the patch rows plus the position rows, the class row cls + pos[0],
    one rounding to fp32.
* a derived error bound for the op-by-op shadow harness (``_rule_*``):
  - bf16 attention: the tensor-core kernels' bound (``shadow._blocked_attention_bound``) restated for separate q and
    kv: scores accumulated in the tensor cores (gamma_{dh+3} with truncating adds), then
    ``shadow._blocked_softmax_err`` over 64-key blocks with P rounded to bf16, the output's own bf16 rounding and the
    flip criterion;
  - fp32 attention: ``shadow._softmax_err``'s terms for the kernel's online form: each score is a 64-fma dot product
    of the pre-scaled q (gamma_{dh+2}), then ``_blocked_softmax_err`` over its 32-key blocks with no rounding of P
    (its tie term, twice the error of p, only loosens the bound), expf within 2 ulp;
  - embed_norm: the LayerNorm rule (``shadow._ln_err`` / ``_ln_out``) plus the rounding of one fp32 add.

``emulated_pvt_ops()`` / ``shadowed_pvt_ops()`` are ``emulated_ops()`` / ``shadowed_ops()`` with these launchers
added; ``pvt_registered()`` imports the family for the PVT test files and restores the registry afterwards.
"""
import importlib
import sys
from contextlib import contextmanager
from copy import deepcopy

import torch

from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64


@contextmanager
def pvt_registered():
    """Registers the PVT models (importing or reloading ``tfimm.architectures.pvt``) and yields the module; restores
    the registry afterwards, so that the exact ``list_models()`` / ``list_modules()`` of the other suites hold in any
    test order."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.pvt"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])
KEY_BLOCK_F32 = 32   # keys per block of the fp32 kernel's online softmax (csrc/pvt.cu)


def split_heads(q, kv, B, N, Nk, H, dh, dtype):
    """(q, k, v) as (B, H, N | N', dh) in dtype: kv read as (B, N', 2, H, dh)."""
    qh = q.to(dtype).view(B, N, H, dh).permute(0, 2, 1, 3)
    k, v = kv.to(dtype).view(B, Nk, 2, H, dh).permute(2, 0, 3, 1, 4)
    return qh, k, v


def _merge_heads(o, B, N, H, dh):
    return o.permute(0, 2, 1, 3).reshape(B * N, H * dh)


def sr_attention_statement(q, kv, B, N, Nk, H, dh, scale, round_p, key_block):
    """softmax(scale q k^T) v in emu._HP, per image (so that large batches do not hold every score at once)."""
    qh, k, v = split_heads(q, kv, B, N, Nk, H, dh, emu._HP)
    out = []
    for b in range(B):
        s = scale * (qh[b:b + 1] @ k[b:b + 1].transpose(-1, -2))
        out.append(emu._softmax_pv(s, v[b:b + 1], round_p, key_block)[0])
    return _merge_heads(torch.cat(out), B, N, H, dh)


def pvt_sr_attention_bf16(q, kv, B, N, Nk, H, dh, scale):
    o = sr_attention_statement(q, kv, B, N, Nk, H, dh, scale, emu.round_bf16, emu.KEY_BLOCK)
    return o.contiguous().to(torch.bfloat16)


def pvt_sr_attention_f32(q, kv, B, N, Nk, H, dh, scale):
    return sr_attention_statement(q, kv, B, N, Nk, H, dh, scale, None, None).contiguous().to(torch.float32)


def pvt_embed_norm(tok, gamma, beta, pos, cls, B, P, eps):
    C = tok.shape[1]
    ntok = 0 if cls is None else 1
    y = emu._ln(tok.view(B, P, C), gamma, beta, eps)
    if cls is not None:
        y = torch.cat((cls.to(emu._HP).view(1, 1, C).expand(B, 1, C), y), dim=1)
    y = y + pos.to(emu._HP)[None]
    return y.reshape(B * (ntok + P), C).contiguous().to(torch.float32)


# ------------------------------------------------------------------------------------------------------ the bounds
def sr_attention_bound(q, kv, B, N, Nk, H, dh, scale, key_block, round_p, u_dot, n_dot, u_acc):
    """Per-element bound of a spatial-reduction attention kernel against its statement (before the output's own
    rounding for bf16 outputs; fp32 outputs include it), per image."""
    qh, k, v = split_heads(q, kv, B, N, Nk, H, dh, _F64)
    out = []
    for b in range(B):
        s = scale * (qh[b:b + 1] @ k[b:b + 1].transpose(-1, -2))
        ds = shadow._gamma(n_dot, u_dot) * scale * (qh[b:b + 1].abs() @ k[b:b + 1].abs().transpose(-1, -2))
        out.append(shadow._blocked_softmax_err(s, ds, v[b:b + 1], key_block, round_p, u_acc))
    return _merge_heads(torch.cat(out), B, N, H, dh)


def _rule_pvt_sr_attention_bf16(A):
    bound = sr_attention_bound(A["q"], A["kv"], A["B"], A["N"], A["Nk"], A["H"], A["dh"], A["scale"], emu.KEY_BLOCK,
                               emu.round_bf16, shadow._UT, A["dh"] + 3, shadow._UT)
    return [("out", shadow._ret, shadow._bounded(bound))]


def _rule_pvt_sr_attention_f32(A):
    bound = sr_attention_bound(A["q"], A["kv"], A["B"], A["N"], A["Nk"], A["H"], A["dh"], A["scale"], KEY_BLOCK_F32,
                               lambda p: p, shadow._U, A["dh"] + 2, shadow._U)
    return [("out", shadow._ret, shadow._bounded(bound))]


def embed_norm_bound(tok, gamma, beta, pos, cls, B, P, eps):
    """The patch rows: the LayerNorm's bound, then one rounding of y + pos (|y| <= gamma |n| + |beta|, plus its own
    error); the class row: one rounding of cls + pos[0]."""
    C = tok.shape[1]
    ntok = 0 if cls is None else 1
    n, dn = shadow._ln_err(tok.view(B, P, C), eps)
    g, be, p = shadow._a(gamma), shadow._a(beta), shadow._a(pos)
    ln = shadow._ln_out(n, dn, gamma, beta)
    rows = ln + shadow._U * (g * n.abs() + be + ln + p[None, ntok:])
    if cls is not None:
        first = shadow._U * (shadow._a(cls) + p[0])
        rows = torch.cat((first.view(1, 1, C).expand(B, 1, C), rows), dim=1)
    return rows.reshape(-1, C)


def _rule_pvt_embed_norm(A):
    arith = embed_norm_bound(A["tok"], A["gamma"], A["beta"], A["pos"], A["cls"], A["B"], A["P"], A["eps"])
    return [("out", shadow._ret, shadow._bounded(arith))]


_PVT = {"pvt_sr_attention_bf16": (pvt_sr_attention_bf16, _rule_pvt_sr_attention_bf16),
        "pvt_sr_attention_f32": (pvt_sr_attention_f32, _rule_pvt_sr_attention_f32),
        "pvt_embed_norm": (pvt_embed_norm, _rule_pvt_embed_norm)}


@contextmanager
def emulated_pvt_ops(arithmetic=torch.float64):
    """``emulate_bf16.emulated_ops()`` plus the statements of the ``pvt_ops`` launchers."""
    from tfimm.backend import pvt_ops

    saved = {n: getattr(pvt_ops, n) for n in _PVT}
    with emu.emulated_ops(arithmetic):
        for n, (f, _) in _PVT.items():
            setattr(pvt_ops, n, f)
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(pvt_ops, n, f)


@contextmanager
def shadowed_pvt_ops():
    """``shadow.shadowed_ops()`` plus every ``pvt_ops`` launcher checked against its statement within its bound; yields
    the shared ``Census``.  Whatever ``pvt_ops.<name>`` is on entry is "the kernel"."""
    from tfimm.backend import pvt_ops

    saved = {n: getattr(pvt_ops, n) for n in _PVT}
    for n, (f, rule) in _PVT.items():
        setattr(emu, n, f)
        shadow._RULES[n] = rule
    try:
        with shadow.shadowed_ops() as census:
            for n in _PVT:
                setattr(pvt_ops, n, shadow._shadow(n, saved[n], census))
            yield census
    finally:
        for n, f in saved.items():
            setattr(pvt_ops, n, f)
            delattr(emu, n)
            del shadow._RULES[n]
