"""TEST INFRASTRUCTURE ONLY -- the CaiT launchers (``tfimm.backend.cait_ops``) on top of oracle/emulate_bf16.py and
oracle/shadow.py.

Each launcher gets
* a statement at the kernels' storage points, in the emulation's arithmetic (float64 by default):
  - ``talking_heads_bf16``: the bf16 qkv and the fp32 mixing weights as stored; S_h = q_h k_h^T,
    L_g = sum_h wl[h, g] S_h + bl[g] (log2 units), P_g = 2^(L_g - max) / sum 2^(L_g - max) over keys,
    P'_f = sum_g P_g ww[g, f] + bw[f] rounded once to bf16, O_f = P'_f V_f rounded once to bf16;
  - ``talking_heads_f32``: the same with P' unrounded and one rounding of O to fp32;
  - ``class_attention``: softmax(scale q k^T) v for one query per (image, head), one rounding to the output dtype;
  - ``add_pos``: x + pos, one rounding to fp32.
* a derived error bound for the op-by-op shadow harness (``_rule_*``), ``talking_heads_bound`` and
  ``class_attention_bound``:
  - S: dh products accumulated in fp32 (the tensor cores' truncating adds in bf16), gamma_dh |q| |k|;
  - L: the fp32 fma chain of H terms onto the bias, with the weighted errors of S: |wl| dS + gamma_{H+1} (|wl| |S| +
    |bl|);
  - P: the argument L - m is off by dL + max dL (the maximum is one of the computed L) + its own rounding; ex2 adds
    2^-21 relatively; the row sum is off relatively by the P-weighted argument errors, gamma_{N+8} of its fp32 sums,
    and 2^-21 per rescale of a running state (at most one per key a thread visits plus the merges); the division
    one rounding; results below fp32's normal range flush (2^-126);
  - P': |ww| dP + gamma_{H+1} (|ww| P + |bw|); in bf16 the kernel rounds a value within dP' of the statement's P', so
    where that interval straddles a rounding boundary the two roundings differ by one spacing (the flip criterion):
    the spread of the interval's roundings, carried through |V|;
  - O: that operand term plus gamma_N of the P' V accumulation (truncating in the tensor cores); the output's own
    bf16 rounding is the harness's ulp term.
  - class attention: as ``shadow._softmax_err`` for one query, with the 128 per-thread states' rescales and merge.

``emulated_cait_ops()`` / ``shadowed_cait_ops()`` are ``emulated_ops()`` / ``shadowed_ops()`` with these launchers
added.
"""
import importlib
import math
import sys
from contextlib import contextmanager
from copy import deepcopy

import torch

from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64
_LN2 = math.log(2.0)
_EX2 = 2.0 ** -21     # relative error bound of ex2.approx / exp2f, with room
_THREADS_PER_ROW = {True: 4, False: 16}   # fewest mixing threads per query row: bf16 kernel, fp32 kernel
_CLS_THREADS = 128


@contextmanager
def cait_registered():
    """Registers the CaiT models (importing or reloading ``tfimm.architectures.cait``) and yields the module; restores
    the registry afterwards, so that the exact ``list_models()`` / ``list_modules()`` of the other suites hold in any
    test order."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.cait"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


def randomise(w, seed):
    """Weights away from their initial values: non-symmetric (H, H) mixes with entries up to 1.2 in magnitude and
    non-zero biases, gamma_1 != gamma_2 of order 0.5 so that every layer shows in the output, a non-zero class token
    and position table."""
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in w.items():
        v = torch.as_tensor(v).float()
        if k.endswith(("proj_l/kernel", "proj_w/kernel")):
            v = torch.rand(v.shape, generator=gen) * 2.4 - 1.2
        elif k.endswith(("gamma_1", "gamma_2")):
            v = 0.3 + 0.5 * torch.rand(v.shape, generator=gen)
        elif k.endswith("bias") or k in ("cls_token", "pos_embed"):
            v = 0.3 * torch.randn(v.shape, generator=gen)
        out[k] = v
    return out


# ------------------------------------------------------------------------------------------------------ statements
def _heads(qkv, b, N, H, dh, hp):
    """q, k, v of image b: (H, N, dh) each."""
    return qkv[b * N:(b + 1) * N].to(hp).view(N, 3, H, dh).permute(1, 2, 0, 3)


def talking_heads_statement(qkv, wl, bl, ww, bw, B, N, H, dh, round_p, out_dtype):
    hp = emu._HP
    wl, bl, ww, bw = (t.to(hp) for t in (wl, bl, ww, bw))
    out = []
    for b in range(B):
        q, k, v = _heads(qkv, b, N, H, dh, hp)
        L = torch.einsum("hqk,hg->gqk", q @ k.transpose(-1, -2), wl) + bl[:, None, None]
        P = torch.softmax(L * _LN2, dim=-1)
        Pp = torch.einsum("gqk,gf->fqk", P, ww) + bw[:, None, None]
        if round_p:
            Pp = Pp.to(torch.bfloat16).to(hp)
        out.append((Pp @ v).permute(1, 0, 2).reshape(N, H * dh))
    return torch.cat(out).to(out_dtype)


def talking_heads_bf16(qkv, wl, bl, ww, bw, B, N, H, dh):
    return talking_heads_statement(qkv, wl, bl, ww, bw, B, N, H, dh, True, torch.bfloat16)


def talking_heads_f32(qkv, wl, bl, ww, bw, B, N, H, dh):
    return talking_heads_statement(qkv, wl, bl, ww, bw, B, N, H, dh, False, torch.float32)


def class_attention(q, kv, B, T, H, dh, scale):
    hp = emu._HP
    qh = q.to(hp).view(B, H, 1, dh)
    k, v = kv.to(hp).view(B, T, 2, H, dh).permute(2, 0, 3, 1, 4)
    p = torch.softmax(scale * (qh @ k.transpose(-1, -2)), dim=-1)
    return (p @ v).reshape(B, H * dh).to(q.dtype)


def add_pos(x, pos, B, N):
    D = x.shape[1]
    y = (x.to(emu._HP).view(B, N, D) + pos.to(emu._HP)[None]).view(B * N, D).to(torch.float32)
    x.copy_(y)
    return x


# ------------------------------------------------------------------------------------------------------ the bounds
def _spread(x, e):
    return ((x + e).to(torch.bfloat16).to(_F64) - (x - e).to(torch.bfloat16).to(_F64)).abs()


def talking_heads_bound(qkv, wl, bl, ww, bw, B, N, H, dh, bf16):
    """Per-element bound of the talking-heads kernel (bf16: mma.sync, P' rounded; else the fp32 SIMT kernel) against
    its statement, before the output's own bf16 rounding (included for the fp32 output)."""
    U, us = shadow._U, (shadow._UT if bf16 else shadow._U)
    g = shadow._gamma
    wl, bl, ww, bw = (t.to(_F64) for t in (wl, bl, ww, bw))
    awl, abl, aww, abw = wl.abs(), bl.abs(), ww.abs(), bw.abs()
    rescales = -(-N // _THREADS_PER_ROW[bf16]) + 8
    out = []
    for b in range(B):
        q, k, v = _heads(qkv, b, N, H, dh, _F64)
        S = q @ k.transpose(-1, -2)
        dS = g(dh, us) * (q.abs() @ k.abs().transpose(-1, -2))
        L = torch.einsum("hqk,hg->gqk", S, wl) + bl[:, None, None]
        dL = torch.einsum("hqk,hg->gqk", dS, awl) + g(H + 1) * (torch.einsum("hqk,hg->gqk", S.abs(), awl)
                                                                + abl[:, None, None])
        del S, dS
        m = L.amax(-1, keepdim=True)
        eps = _LN2 * (dL + dL.amax(-1, keepdim=True) + U * (L - m).abs()) + _EX2
        P = torch.softmax(L * _LN2, dim=-1)
        del L, dL
        lam = (P * eps).sum(-1, keepdim=True) + rescales * _EX2 + g(N + 8)
        dP = P * (eps + lam + 2 * U) + 2.0 ** -126
        del eps
        Pp = torch.einsum("gqk,gf->fqk", P, ww) + bw[:, None, None]
        dPp = torch.einsum("gqk,gf->fqk", dP, aww) + g(H + 1) * (torch.einsum("gqk,gf->fqk", P, aww)
                                                                 + abw[:, None, None])
        del P, dP
        av = v.abs()
        if bf16:
            do = _spread(Pp, dPp) @ av + g(N, shadow._UT) * (Pp.to(torch.bfloat16).to(_F64).abs() @ av)
        else:
            do = dPp @ av + g(N + 1) * (Pp.abs() @ av)
        out.append(do.permute(1, 0, 2).reshape(N, H * dh))
    return torch.cat(out)


def class_attention_bound(q, kv, B, T, H, dh, scale):
    U, g = shadow._U, shadow._gamma
    qh = q.to(_F64).view(B, H, 1, dh)
    k, v = kv.to(_F64).view(B, T, 2, H, dh).permute(2, 0, 3, 1, 4)
    s = scale * (qh @ k.transpose(-1, -2))
    ds = g(dh + 3) * scale * (qh.abs() @ k.abs().transpose(-1, -2))
    m = s.amax(-1, keepdim=True)
    p = torch.softmax(s, dim=-1)
    rescales = -(-T // _CLS_THREADS) + 8
    dp = p * (2 * ds.amax(-1, keepdim=True) + U * (s.abs() + (s - m).abs()) + rescales * _EX2
              + g(T + 8 + _CLS_THREADS))
    pv = p @ v.abs()
    do = dp @ v.abs() + g(T + 2 + _CLS_THREADS) * pv
    return do.reshape(B, H * dh)


def _rule_talking_heads(bf16):
    def rule(A):
        bound = talking_heads_bound(A["qkv"], A["wl"], A["bl"], A["ww"], A["bw"], A["B"], A["N"], A["H"], A["dh"],
                                    bf16)
        return [("out", shadow._ret, shadow._bounded(bound))]
    return rule


def _rule_class_attention(A):
    bound = class_attention_bound(A["q"], A["kv"], A["B"], A["T"], A["H"], A["dh"], A["scale"])
    return [("out", shadow._ret, shadow._bounded(bound))]


def _rule_add_pos(A):
    B, N = A["B"], A["N"]
    D = A["x"].shape[1]
    mag = (A["x"].to(_F64).abs().view(B, N, D) + A["pos"].to(_F64).abs()[None]).view(B * N, D)
    return [("x", shadow._ret, shadow._bounded(shadow._U * mag, flips=False))]


_CAIT = {"talking_heads_bf16": (talking_heads_bf16, _rule_talking_heads(True)),
         "talking_heads_f32": (talking_heads_f32, _rule_talking_heads(False)),
         "class_attention": (class_attention, _rule_class_attention),
         "add_pos": (add_pos, _rule_add_pos)}


@contextmanager
def emulated_cait_ops(arithmetic=torch.float64):
    """``emulate_bf16.emulated_ops()`` plus the statements of the ``cait_ops`` launchers."""
    from tfimm.backend import cait_ops

    saved = {n: getattr(cait_ops, n) for n in _CAIT}
    with emu.emulated_ops(arithmetic):
        for n, (f, _) in _CAIT.items():
            setattr(cait_ops, n, f)
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(cait_ops, n, f)


@contextmanager
def shadowed_cait_ops():
    """``shadow.shadowed_ops()`` plus every ``cait_ops`` launcher checked against its statement within its bound;
    yields the shared ``Census``.  Whatever ``cait_ops.<name>`` is on entry is "the kernel"."""
    from tfimm.backend import cait_ops

    saved = {n: getattr(cait_ops, n) for n in _CAIT}
    for n, (f, rule) in _CAIT.items():
        setattr(emu, n, f)
        shadow._RULES[n] = rule
    try:
        with shadow.shadowed_ops() as census:
            for n in _CAIT:
                setattr(cait_ops, n, shadow._shadow(n, saved[n], census))
            yield census
    finally:
        for n, f in saved.items():
            setattr(cait_ops, n, f)
            delattr(emu, n)
            del shadow._RULES[n]
