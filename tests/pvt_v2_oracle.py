"""TEST INFRASTRUCTURE ONLY -- the PVT v2 launchers (``tfimm.backend.pvt_v2_ops``) on top of oracle/emulate_bf16.py,
oracle/shadow.py and tests/pvt_oracle.py.

Each launcher gets
* a statement at the kernels' storage points, in the emulation's arithmetic (float64 by default):
  - ``pvt_v2_conv_mlp_bf16``: hid = bf16(h W1^T + b1); a = bf16(act(dwconv3x3(hid) + b_dw)) with zero padding;
    out = residual + a W2^T + b2, one rounding to fp32.  These are the storage points of the unfused chain (fc1 GEMM
    with a bf16 output, ``dwconv_bias_act``, fc2 GEMM + residual), so one statement covers both paths;
  - ``pvt_v2_sr_attention_{bf16,f32}``: the head-dim-64 statements of tests/pvt_oracle.py, which are generic in dh.
* a derived error bound for the op-by-op shadow harness (``_rule_*``):
  - ConvFFN: the error is carried through the three steps element by element.  fc1 is a tensor-core dot product of
    C terms plus the bias (gamma_{C+1} with truncating adds); where that interval around the exact value straddles a
    bf16 rounding boundary the stored hidden value may be the neighbour, so the hidden error is the distance between
    the roundings of the interval's ends (0 almost everywhere).  The depthwise sum adds the taps' weighted hidden
    errors and its own fp32 evaluation (gamma_10 of the absolute sum); the activation its slope times that plus its
    own error (``shadow._act_err``); the second bf16 rounding the same interval argument; fc2 the weighted operand
    errors, gamma_{hidden+1} of its absolute sum (truncating adds), and the two fp32 roundings of the bias and
    residual adds;
  - attention: ``pvt_oracle.sr_attention_bound`` at dh 32.
"""
import importlib
import sys
from contextlib import contextmanager
from copy import deepcopy

import torch

import pvt_oracle as po
from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64
_PADS = (1, 1, 1, 1)   # the depthwise convolution's zero padding (left, right, top, bottom)


@contextmanager
def pvt_v2_registered():
    """Registers the PVT v2 models (importing or reloading ``tfimm.architectures.pvt_v2``) and yields the module;
    restores the registry afterwards, so that the exact ``list_models()`` / ``list_modules()`` of the other suites
    hold in any test order."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.pvt_v2"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


# ------------------------------------------------------------------------------------------------------ statements
def conv_mlp_statement(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act):
    """(hid, z, a, y): the exact fc1 output before its rounding, the exact depthwise output (from the rounded hidden),
    the rounded activation and the exact output, all in emu._HP."""
    hp = emu._HP
    hidden = w1.shape[0]
    y1 = h.to(hp) @ w1.to(hp).t() + b1.to(hp)
    hid = y1.to(torch.bfloat16).to(hp)
    z = emu._dw(hid.view(B, gh, gw, hidden), wdw, bdw, 3, 1, _PADS).reshape(-1, hidden)
    a = emu._act(z, act).to(torch.bfloat16).to(hp)
    y = residual.to(hp) + (a @ w2.to(hp).t() + b2.to(hp))
    return y1, z, a, y


def pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act, out=None):
    y = conv_mlp_statement(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act)[3].to(torch.float32)
    if out is not None:
        out.copy_(y)
        return out
    return y


def pvt_v2_sr_attention_bf16(q, kv, B, N, Nk, H, dh, scale):
    return po.pvt_sr_attention_bf16(q, kv, B, N, Nk, H, dh, scale)


def pvt_v2_sr_attention_f32(q, kv, B, N, Nk, H, dh, scale):
    return po.pvt_sr_attention_f32(q, kv, B, N, Nk, H, dh, scale)


# ------------------------------------------------------------------------------------------------------ the bounds
def _rounding_spread(x, e):
    """|bf16(x + e) - bf16(x - e)|: how far apart two bf16 roundings of values within e of x can be."""
    return ((x + e).to(torch.bfloat16).to(_F64) - (x - e).to(torch.bfloat16).to(_F64)).abs()


def conv_mlp_bound(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act):
    """Per-element bound of the ConvFFN (fused kernel or unfused chain) against its statement (fp32 output: its own
    rounding included)."""
    saved, emu._HP = emu._HP, _F64
    try:
        y1, z, a, _ = conv_mlp_statement(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act)
    finally:
        emu._HP = saved
    C, hidden = h.shape[1], w1.shape[0]
    S1 = shadow._a(h) @ shadow._a(w1).t() + shadow._a(b1)
    d_hid = _rounding_spread(y1, shadow._gamma(C + 1, shadow._UT) * S1)
    hid = y1.to(torch.bfloat16).to(_F64)
    img = (B, gh, gw, hidden)
    aw = shadow._a(wdw)
    Mz = emu._dw((hid.abs() + d_hid).view(img), aw, shadow._a(bdw), 3, 1, _PADS).reshape(-1, hidden)
    e_z = emu._dw(d_hid.view(img), aw, None, 3, 1, _PADS).reshape(-1, hidden) + shadow._gamma(10) * Mz
    g = emu._act(z, act)
    e_g = shadow._LIP.get(act, 1.0) * e_z + shadow._act_err(act, z.abs() + e_z)
    d_a = _rounding_spread(g, e_g)
    S2 = (a.abs() + d_a) @ shadow._a(w2).t() + shadow._a(b2)
    extra = d_a @ shadow._a(w2).t()
    return extra + shadow._gamma(hidden + 1, shadow._UT) * S2 + 2 * shadow._U * (S2 + shadow._a(residual))


def _rule_pvt_v2_conv_mlp_bf16(A):
    bound = conv_mlp_bound(A["h"], A["w1"], A["b1"], A["wdw"], A["bdw"], A["w2"], A["b2"], A["residual"], A["B"],
                           A["gh"], A["gw"], A["act"])
    return [("out", shadow._ret, shadow._bounded(bound))]


def _rule_pvt_v2_sr_attention_bf16(A):
    return po._rule_pvt_sr_attention_bf16(A)


def _rule_pvt_v2_sr_attention_f32(A):
    return po._rule_pvt_sr_attention_f32(A)


_PVT_V2 = {"pvt_v2_conv_mlp_bf16": (pvt_v2_conv_mlp_bf16, _rule_pvt_v2_conv_mlp_bf16),
           "pvt_v2_sr_attention_bf16": (pvt_v2_sr_attention_bf16, _rule_pvt_v2_sr_attention_bf16),
           "pvt_v2_sr_attention_f32": (pvt_v2_sr_attention_f32, _rule_pvt_v2_sr_attention_f32)}


@contextmanager
def emulated_pvt_v2_ops(arithmetic=torch.float64):
    """``pvt_oracle.emulated_pvt_ops()`` plus the statements of the ``pvt_v2_ops`` launchers."""
    from tfimm.backend import pvt_v2_ops

    saved = {n: getattr(pvt_v2_ops, n) for n in _PVT_V2}
    with po.emulated_pvt_ops(arithmetic):
        for n, (f, _) in _PVT_V2.items():
            setattr(pvt_v2_ops, n, f)
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(pvt_v2_ops, n, f)


@contextmanager
def shadowed_pvt_v2_ops():
    """``pvt_oracle.shadowed_pvt_ops()`` plus every ``pvt_v2_ops`` launcher checked against its statement within its
    bound; yields the shared ``Census``.  Whatever ``pvt_v2_ops.<name>`` is on entry is "the kernel"."""
    from tfimm.backend import pvt_v2_ops

    saved = {n: getattr(pvt_v2_ops, n) for n in _PVT_V2}
    for n, (f, rule) in _PVT_V2.items():
        setattr(emu, n, f)
        shadow._RULES[n] = rule
    try:
        with po.shadowed_pvt_ops() as census:
            for n in _PVT_V2:
                setattr(pvt_v2_ops, n, shadow._shadow(n, saved[n], census))
            yield census
    finally:
        for n, f in saved.items():
            setattr(pvt_v2_ops, n, f)
            delattr(emu, n)
            del shadow._RULES[n]
