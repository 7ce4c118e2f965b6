"""TEST INFRASTRUCTURE ONLY -- the ConvMixer launcher (``tfimm.backend.convmixer_ops``) on top of
oracle/emulate_bf16.py and oracle/shadow.py.

``dwconv`` gets
* a statement in the REFERENCE's form, not the kernel's folded one: the previous BatchNorm applied to the stored fp32
  activation, x = s_in a + t_in; x zero-padded for the "same" depthwise convolution; + bias; the activation; BN1 as
  s1 act + t1; the residual x added; one rounding to the output's storage type at the end.  Arithmetic in the
  emulation's precision (float64 by default);
* a derived error bound for the op-by-op shadow harness (``_rule_dwconv``): x = fmaf(s_in, a, t_in) rounds once
  (|dx| <= u |x|), the k^2 fma taps and the bias add are an fp32 sum of k^2 + 1 terms, and x's error passes through the
  taps, so with Z = sum |w| |x| + |b|, z is off by <= gamma_{k^2 + 2} Z; the activation multiplies that by its slope and
  adds its own error (shadow._act_err); |act(z)| <= Z for relu and gelu.  Then fmaf(s1, act, t1) rounds once, the
  residual add once and the statement's own fp32 store once more.

``kernel_form`` is a float32 model of the kernel's algorithm (folded BN, position mask, fma taps in (ky, kx) order) for
the CPU rehearsals.  ``emulated_convmixer_ops()`` / ``shadowed_convmixer_ops()`` are ``emulated_ops()`` /
``shadowed_ops()`` with ``convmixer_ops.dwconv`` and ``mixer_ops.affine`` (the features and the head's BN) added.
"""
from contextlib import contextmanager

import torch
import torch.nn.functional as F

import mixer_oracle
from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64


def _k(taps):
    return int(round(taps.shape[0] ** 0.5))


def _depthwise_same(x, taps, bias):
    """DepthwiseConv2D(k, "same") of NHWC x (zero-padded) with taps (k * k, C) in x's dtype."""
    k, C = _k(taps), x.shape[-1]
    p = (k - 1) // 2
    wt = taps.to(x.dtype).t().reshape(C, 1, k, k)
    y = F.conv2d(F.pad(x.permute(0, 3, 1, 2), (p, p, p, p)), wt, None if bias is None else bias.to(x.dtype), groups=C)
    return y.permute(0, 2, 3, 1)


def dwconv(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
    hp = emu._HP
    x = s_in.to(hp) * a.to(hp) + t_in.to(hp)
    z = _depthwise_same(x, taps.to(hp), bias.to(hp))
    y = s1.to(hp) * emu._act(z, act) + t1.to(hp) + x
    return y.to(out_dtype).contiguous()


def kernel_form(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
    """What the kernel computes, in float32: x = fmaf(s_in, a, t_in) inside the image and 0 in the padding, each output
    summed tap by tap in (ky, kx) order from 0 with fma roundings, + bias, act, x + fmaf(s1, act, t1)."""
    B, H, W, C = a.shape
    k = _k(taps)
    p = (k - 1) // 2
    x = (s_in.double() * a.double() + t_in.double()).float()
    xp = F.pad(x, (0, 0, p, p, p, p))
    acc = torch.zeros_like(a)
    for ky in range(k):
        for kx in range(k):
            acc = (acc.double() + xp[:, ky:ky + H, kx:kx + W].double() * taps[ky * k + kx].double()).float()
    z = emu._act(acc + bias, act).float()
    y = x + (s1.double() * z.double() + t1.double()).float()
    return y.to(out_dtype).contiguous()


@contextmanager
def kernel_forms():
    """``convmixer_ops.dwconv`` replaced by the float32 model of its kernel (CPU rehearsals)."""
    from tfimm.backend import convmixer_ops

    saved = convmixer_ops.dwconv
    convmixer_ops.dwconv = kernel_form
    try:
        yield
    finally:
        convmixer_ops.dwconv = saved


# ------------------------------------------------------------------------------------------------------ the bounds
_U = shadow._U


def dwconv_bound(a, s_in, t_in, taps, bias, s1, t1, act):
    """Bound on |fp32 kernel - float64 statement| before the output's rounding to bf16 (module docstring)."""
    k = _k(taps)
    x = (s_in.to(_F64) * a.to(_F64) + t_in.to(_F64)).abs()
    Z = _depthwise_same(x, taps.to(_F64).abs(), bias.to(_F64).abs())
    s1a, t1a = s1.to(_F64).abs(), t1.to(_F64).abs()
    dz = shadow._gamma(k * k + 2) * Z
    e_act = shadow._LIP.get(act, 1.0) * dz + shadow._act_err(act, Z)
    return s1a * e_act + _U * (s1a * Z + t1a) + _U * x + 2 * _U * (x + s1a * Z + t1a)


def _rule_dwconv(A):
    return [("out", shadow._ret, shadow._bounded(dwconv_bound(A["a"], A["s_in"], A["t_in"], A["taps"], A["bias"],
                                                             A["s1"], A["t1"], A["act"])))]


_CONVMIXER = {"dwconv": (dwconv, _rule_dwconv)}
_AFFINE = {"affine": mixer_oracle._MIXER["affine"]}


@contextmanager
def emulated_convmixer_ops(arithmetic=torch.float64):
    """``emulate_bf16.emulated_ops()`` plus the statements of ``convmixer_ops.dwconv`` and ``mixer_ops.affine``."""
    from tfimm.backend import convmixer_ops, mixer_ops

    saved = (convmixer_ops.dwconv, mixer_ops.affine)
    with emu.emulated_ops(arithmetic):
        convmixer_ops.dwconv, mixer_ops.affine = dwconv, _AFFINE["affine"][0]
        try:
            yield
        finally:
            convmixer_ops.dwconv, mixer_ops.affine = saved


@contextmanager
def shadowed_convmixer_ops():
    """``shadow.shadowed_ops()`` plus ``convmixer_ops.dwconv`` and ``mixer_ops.affine`` checked against their
    statements within their bounds; yields the shared ``Census``.  Whatever the launchers are on entry is "the
    kernel"."""
    from tfimm.backend import convmixer_ops, mixer_ops

    mods = {"dwconv": convmixer_ops, "affine": mixer_ops}
    table = {**_CONVMIXER, **_AFFINE}
    saved = {n: getattr(mods[n], n) for n in table}
    for n, (f, rule) in table.items():
        setattr(emu, n, f)
        shadow._RULES[n] = rule
    try:
        with shadow.shadowed_ops() as census:
            for n in table:
                setattr(mods[n], n, shadow._shadow(n, saved[n], census))
            yield census
    finally:
        for n, f in saved.items():
            setattr(mods[n], n, f)
            delattr(emu, n)
            del shadow._RULES[n]
