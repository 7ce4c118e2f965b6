"""TEST INFRASTRUCTURE ONLY -- the MLP-Mixer launchers (``tfimm.backend.mixer_ops``) on top of oracle/emulate_bf16.py and
oracle/shadow.py.

Each launcher gets

* a statement with the kernels' storage points (``token_gemm``, ``gemm_glu``, ``affine``): the stored operands (bf16 or
  fp32) as they are, the contraction, bias, activation / GLU, gamma, multiplier and residual in the emulation's
  arithmetic (float64 by default), one rounding to the output's storage type at the end -- what the kernels do in fp32;
* a derived error bound for the op-by-op shadow harness (``_rule_*``).

``emulated_mixer_ops()`` / ``shadowed_mixer_ops()`` are ``emulated_ops()`` / ``shadowed_ops()`` with these launchers added.
"""
from contextlib import contextmanager

import torch

from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64


def _glu_rows(acc, act):
    """acc (..., M, C) with rows in groups of 16 (8 values, then their 8 gates) -> value * act(gate), (..., M / 2, C)."""
    *lead, M, C = acc.shape
    a = acc.reshape(*lead, M // 16, 2, 8, C)
    return (a[..., 0, :, :] * emu._act(a[..., 1, :, :], act)).reshape(*lead, M // 2, C)


def token_gemm(wt, x, bias=None, act=None, gamma=None, residual=None, mul=None, out=None, m_out=None, glu=False,
               out_dtype=None, block_n=0):
    hp = emu._HP
    M = wt.shape[0]
    y = torch.einsum("mk,bkc->bmc", wt.to(hp), x.to(hp))
    if bias is not None:
        y = y + bias.to(hp)[:, None]
    y = _glu_rows(y, act) if glu else emu._act(y, act)
    m_out = m_out if m_out is not None else (M // 2 if glu else M)
    y = y[:, :m_out]
    if gamma is not None:
        y = y * gamma.to(hp)
    if mul is not None:
        y = y * mul.to(hp)
    if residual is not None:
        y = y + residual.to(hp)
    dt = out_dtype or (residual.dtype if residual is not None else x.dtype)
    return emu._store(y.contiguous(), out, dt)


def _glu_cols(acc, act, pairwise):
    if pairwise:
        return acc[:, 0::2] * emu._act(acc[:, 1::2], act)
    return _glu_rows(acc.t(), act).t()


def gemm_glu(a, w, bias, n_out, act, block_n=0):
    hp = emu._HP
    y = a.to(hp) @ w.to(hp).t() + bias.to(hp)
    return _glu_cols(y, act, a.dtype == torch.bfloat16)[:, :n_out].contiguous().to(a.dtype)


def affine(x, alpha, beta, out_dtype):
    return (alpha.to(emu._HP) * x.to(emu._HP) + beta.to(emu._HP)).to(out_dtype)


# ------------------------------------------------------------------------------------------------------ the bounds
def _glu_err(S, n, u, act, glu):
    """(bound on the pre-epilogue value's error, bound on its magnitude) from S = sum of |terms| of every accumulator
    (rows or columns as the kernel holds them).  Plain: the contraction (gamma_n S), the activation's slope and own error
    (shadow._epilogue's terms).  GLU: value v and gate g each off by gamma_n S; v act(g) is off by
    e_v |act(g)| + |v| (L e_g + e_act) + one rounding, with |act(g)| <= |g| <= S_g (GELU / swish)."""
    L = shadow._LIP.get(act, 1.0)
    e = shadow._gamma(n, u)
    if glu is None:
        return L * e * S + shadow._act_err(act, S), S
    sv, sg = glu
    err = e * sv * sg + sv * (L * e * sg + shadow._act_err(act, sg)) + shadow._U * sv * sg
    return err, sv * sg


def _tail(err, mag, gamma, mul, residual):
    """gamma, multiplier and residual after the activation: each product scales the error and adds one fp32 rounding,
    the residual add one more, and the statement's own rounding to fp32 storage one more (as shadow._epilogue's two
    roundings of the residual add)."""
    for f in (gamma, mul):
        if f is not None:
            fa = f.abs().to(_F64)
            err, mag = err * fa, mag * fa
            err = err + shadow._U * mag
    r = residual.abs().to(_F64) if residual is not None else 0.0
    return err + 2 * shadow._U * (mag + r)


def _rule_token_gemm(A):
    wt, x, glu, act = A["wt"], A["x"], A["glu"], A["act"]
    M = wt.shape[0]
    S = torch.einsum("mk,bkc->bmc", wt.abs().to(_F64), x.abs().to(_F64))
    if A["bias"] is not None:
        S = S + A["bias"].abs().to(_F64)[:, None]
    u = shadow._UT if x.dtype == torch.bfloat16 else shadow._U
    m_out = A["m_out"] if A["m_out"] is not None else (M // 2 if glu else M)
    if glu:
        s = S.reshape(S.shape[0], M // 16, 2, 8, -1)
        err, mag = _glu_err(None, x.shape[1] + 1, u, act,
                            (s[:, :, 0].reshape(S.shape[0], M // 2, -1), s[:, :, 1].reshape(S.shape[0], M // 2, -1)))
    else:
        err, mag = _glu_err(S, x.shape[1] + 1, u, act, None)
    err, mag = err[:, :m_out], mag[:, :m_out]
    err = _tail(err, mag, A["gamma"], A["mul"], A["residual"])
    return [("out", shadow._ret, shadow._bounded(err))]


def _rule_gemm_glu(A):
    a, w = A["a"], A["w"]
    S = a.abs().to(_F64) @ w.abs().to(_F64).t() + A["bias"].abs().to(_F64)
    u = shadow._UT if a.dtype == torch.bfloat16 else shadow._U
    if a.dtype == torch.bfloat16:
        sv, sg = S[:, 0::2], S[:, 1::2]
    else:
        M, F = S.shape
        s = S.t().reshape(F // 16, 2, 8, M)
        sv, sg = s[:, 0].reshape(F // 2, M).t(), s[:, 1].reshape(F // 2, M).t()
    err, mag = _glu_err(None, a.shape[1] + 1, u, A["act"], (sv, sg))
    err = err + shadow._U * mag    # the statement's own rounding to the storage type (fp32 outputs)
    return [("out", shadow._ret, shadow._bounded(err[:, :A["n_out"]]))]


def _rule_affine(A):
    # the kernel's fma rounds once, a product and a sum (the float32 stand-in) twice, and the statement's own rounding
    # to fp32 storage once more: 3 u (|alpha x| + |beta|)
    mag = (A["alpha"].abs().to(_F64) * A["x"].abs().to(_F64) + A["beta"].abs().to(_F64))
    return [("out", shadow._ret, shadow._bounded(3 * shadow._U * mag))]


_MIXER = {"token_gemm": (token_gemm, _rule_token_gemm), "gemm_glu": (gemm_glu, _rule_gemm_glu),
          "affine": (affine, _rule_affine)}


@contextmanager
def emulated_mixer_ops(arithmetic=torch.float64):
    """``emulate_bf16.emulated_ops()`` plus the statements of the ``mixer_ops`` launchers."""
    from tfimm.backend import mixer_ops

    saved = {n: getattr(mixer_ops, n) for n in _MIXER}
    with emu.emulated_ops(arithmetic):
        for n, (f, _) in _MIXER.items():
            setattr(mixer_ops, n, f)
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(mixer_ops, n, f)


@contextmanager
def shadowed_mixer_ops():
    """``shadow.shadowed_ops()`` plus every ``mixer_ops`` launcher checked against its statement within its bound;
    yields the shared ``Census``.  Whatever ``mixer_ops.<name>`` is on entry is "the kernel"."""
    from tfimm.backend import mixer_ops

    saved = {n: getattr(mixer_ops, n) for n in _MIXER}
    for n, (f, rule) in _MIXER.items():
        setattr(emu, n, f)
        shadow._RULES[n] = rule
    try:
        with shadow.shadowed_ops() as census:
            for n in _MIXER:
                setattr(mixer_ops, n, shadow._shadow(n, saved[n], census))
            yield census
    finally:
        for n, f in saved.items():
            setattr(mixer_ops, n, f)
            delattr(emu, n)
            del shadow._RULES[n]
