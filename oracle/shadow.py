"""TEST INFRASTRUCTURE ONLY -- every kernel launch of a forward pass checked against its float64 statement, op by op.

Logit-level comparisons cannot separate a wrong kernel from bf16 storage noise: one flipped rounding spreads through the
layers, and the comparison floor is ~2-3e-3 (tests/test_parity_budget_gpu.py).  Here each launch is checked where it
happens instead.  Inside ``shadowed_ops()`` every launcher of ``tfimm.backend.ops`` that ``oracle/emulate_bf16.py``
restates (the shape predicates excepted)

1. clones every tensor argument -- ``out``, ``residual``, ``pool_sum`` and ``probs`` included, aliasing preserved (the
   engine calls in place: ``out`` is often ``residual``);
2. computes the arithmetic error bound of each output from those pristine inputs (``_RULES``), and runs the
   ``emulate_bf16`` function on the clones in float64 -- the engine's storage points with exact arithmetic;
3. runs the real launcher on the original arguments and synchronises;
4. compares the returned tensor, every output written in place, ``probs`` and the *increase* of ``pool_sum`` (an atomic
   accumulator) with ``check``; every other tensor argument must come back bit-identical;
5. records op, call site (``tfimm/architectures/*.py:line`` and the index of the launch in the pass), arguments, the
   worst error in units of the bound and the flip fraction in the ``Census`` it yields.

The forward pass continues on the kernel's results, so every op is checked on exactly the inputs the engine produced:
errors do not build up from layer to layer, and the bounds are a few bf16 ulps rather than 1e-2 on the logits.  The
references are computed on the tensors' device one op at a time and freed after the comparison.

Usage (tests only)::

    with shadow.shadowed_ops() as census:
        model(x)                      # eager forward; CUDA-graph capture is refused
    print(census.table())
    census.assert_ok()
"""
import inspect
import math
import os
import sys
from contextlib import contextmanager

import torch
import torch.nn.functional as F

from . import emulate_bf16 as emu

_F64 = torch.float64
# Unit roundoff of fp32 round-to-nearest (SIMT arithmetic, epilogues).
_U = 2.0 ** -24
# fp32 accumulation inside the tensor cores: the aligned products are truncated, not rounded, so each addition is
# bounded by one full fp32 ulp.
_UT = 2.0 ** -23


def _gamma(n, u=_U):
    """Classic bound on an n-term fp32 sum / dot product: |fl(sum) - sum| <= gamma_n * sum |terms| (Higham, ch. 3)."""
    return n * u / (1.0 - n * u)


# Largest slope of each activation: an error of its argument grows by at most this factor.  GELU' peaks at 1.129
# (x ~ 1.5), swish' at 1.0998 (x ~ 2.4), sigmoid' at 1/4; relu / relu6 / tanh / identity have slope <= 1.
_LIP = {"gelu": 1.13, "swish": 1.1, "silu": 1.1, "sigmoid": 0.25}
# Activations the kernels evaluate approximately (common.cuh): the erf-GELU fit is good to 3.6e-6 absolute
# (tools/fit_gelu.py), tanhf to 2 ulp, and sigmoid = rcp.approx(1 + ex2.approx(.)) to ~2^-21 relative.  Bound: 5e-6
# absolute -- the floor ``faithful`` uses for the same reason -- plus 8 fp32 ulps of the argument's magnitude.
_SMOOTH = ("gelu", "swish", "silu", "tanh", "sigmoid")
_ACT_ABS = 5e-6

FLIP_LIMIT = 2e-2


def faithful(out, ref):
    """(fraction of outputs with |ref| >= 0.05 that are not the correctly rounded bf16 value, worst error in units of
    max(one bf16 spacing at that magnitude, 5e-6)).  Below ~1e-3 in magnitude an output's own ulp is smaller than the
    4e-6 absolute accuracy of the activation polynomials -- and irrelevant to the next layer's sums."""
    want = ref.to(torch.bfloat16)
    big = ref.abs() >= 0.05
    flips = ((out != want) & big).float().sum().item() / max(big.float().sum().item(), 1.0)
    unit = torch.maximum(ref.abs() * 2.0 ** -7, torch.full_like(ref, 5e-6))
    worst = ((out.double() - ref).abs() / unit).max().item()
    return flips, worst


def ulp_bf16(r):
    """Spacing of the bf16 numbers at |r|: 2^(e-8) for |r| in [2^(e-1), 2^e); below the smallest normal, its spacing."""
    _, e = torch.frexp(r.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(r), e - 8)


# ---------------------------------------------------------------------------------------------------------- the rule
def check(op, kernel_out, ref, ctx):
    """Acceptance rule of one shadowed output, in one place.  Returns (ok, worst error / bound, flip fraction).

    ctx["rule"]:
      "exact"    pure data movement: bit-identical.
      "bounded"  |kernel - ref| <= ctx["arith"] (+ one bf16 ulp of ref when the output is stored in bf16): the float64
                 value, rounded once to the storage type by an implementation whose arithmetic error is at most the
                 derived fp32 term -- i.e. the correctly rounded value or its neighbour.  fp32-stored outputs get no
                 ulp term (their own rounding is part of ``arith``).
      "cited"    the one known exception, the fused MLP (its bf16 hidden tensor never leaves the SM): the total bound
                 ``ctx["bound"]`` (and ``ctx["rms"]`` on the rms error) that the named test of
                 tests/test_kernels_gpu.py argues for (``ctx["cite"]``).
    ctx["flips"] (bf16 outputs): the share of elements with |ref| >= 0.05 that are not the correctly rounded value must
    stay under ``FLIP_LIMIT`` (2 %).  An exact-arithmetic kernel flips ~arith/ulp of them (well under 1 %); a
    systematic defect -- a tanh-form GELU, a biased rounding -- flips far more while staying inside one ulp."""
    flips = 0.0
    if ctx["rule"] == "exact":
        ok = kernel_out.shape == ref.shape and kernel_out.dtype == ref.dtype and torch.equal(kernel_out, ref)
        return ok, (0.0 if ok else math.inf), flips
    k, r = kernel_out.double(), ref.double()
    err = torch.nan_to_num((k - r).abs(), nan=math.inf)
    if ctx["rule"] == "cited":
        worst = err.max().item() / ctx["bound"]
        ok = worst <= 1.0
        if "rms" in ctx:
            ok = ok and (k - r).pow(2).mean().sqrt().item() <= ctx["rms"]
    else:
        bound = ctx["arith"]
        bound = bound.expand_as(r) if torch.is_tensor(bound) else torch.full_like(r, bound)
        if kernel_out.dtype == torch.bfloat16:
            bound = bound + ulp_bf16(r)
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)   # err > 0 against a zero bound: inf
        worst = ratio.max().item() if ratio.numel() else 0.0
        ok = worst <= 1.0
    if ctx.get("flips") and kernel_out.dtype == torch.bfloat16:
        flips, _ = faithful(kernel_out, r)
        ok = ok and flips < FLIP_LIMIT
    return ok, worst, flips


def _bounded(arith, flips=True):
    return {"rule": "bounded", "arith": arith, "flips": flips}


def _exact():
    return {"rule": "exact"}


# ------------------------------------------------------------------------------------ arithmetic terms, op by op
def _a(t):
    return None if t is None else t.abs().to(_F64)


def _act_err(act, zmag):
    """Error the activation adds on top of its slope times the argument's error (see _SMOOTH)."""
    return _ACT_ABS + 8 * _U * zmag if act in _SMOOTH else 0.0


def _epilogue(S, n, u, act, gamma, residual, extra=0.0):
    """out = [act](gamma * act(y) + residual) with y = sum of n terms whose magnitudes sum to S: the contraction
    (gamma_n * S), ``extra`` (an operand difference), the activation (its slope L and own error), the gamma product and
    the residual add (two fp32 roundings of magnitude <= L (|gamma| S + |residual|))."""
    g = _a(gamma) if gamma is not None else 1.0
    r = _a(residual) if residual is not None else 0.0
    L = _LIP.get(act, 1.0)
    e_y = _gamma(n, u) * S + extra
    gmax = torch.clamp(g, min=1.0) if torch.is_tensor(g) else 1.0
    return L * (g * e_y + 2 * _U * (g * S + r)) + gmax * _act_err(act, g * S + r)


def _rule_gemm(A):
    a, w = A["a"], A["w"]
    S = _a(a) @ _a(w).t()
    if A["bias"] is not None:
        S = S + _a(A["bias"])
    u = _UT if a.dtype == torch.bfloat16 else _U
    return [("out", _ret, _bounded(_epilogue(S, a.shape[1] + 1, u, A["act"], A["gamma"], A["residual"])))]


def _rule_gemm_gated(A):
    a, gate, rows, w = A["a"], A["gate"], A["rows_per_image"], A["w"]
    img = torch.arange(a.shape[0], device=a.device) // rows
    prod = a.to(_F64) * gate.to(_F64)[img]                  # exact: 8 x 24 significant bits
    # The kernel multiplies in fp32 and rounds that to bf16 (as a separate scale_channels_ pass would); the reference
    # rounds the exact product once.  Where the fp32 product lands on a bf16 tie the two operands differ by one bf16
    # ulp: that exact operand difference, carried through |W|, is added to the bound.
    d_op = (prod.float().to(torch.bfloat16).to(_F64) - prod.to(torch.bfloat16).to(_F64)).abs()
    S = prod.to(torch.bfloat16).to(_F64).abs() @ _a(w).t()
    if A["bias"] is not None:
        S = S + _a(A["bias"])
    extra = d_op @ _a(w).t() if bool((d_op != 0).any()) else 0.0
    return [("out", _ret, _bounded(_epilogue(S, a.shape[1] + 1, _UT, A["act"], None, A["residual"], extra)))]


def _rule_mlp_fused(A):
    # Known exception (tests/test_kernels_gpu.py::test_mlp_fused_equals_two_gemms): the bf16 hidden tensor never leaves
    # the SM, so a flipped hidden rounding cannot be seen in isolation; the output is held to 3e-3 of max|ref| and its
    # rms error to 2e-4 of it, as there.
    def ctx(kern, ref):
        scale = ref.ret.abs().max().item()
        return {"rule": "cited", "bound": 3e-3 * scale + 1e-30, "rms": 2e-4 * scale,
                "cite": "test_mlp_fused_equals_two_gemms"}
    return [("out", _ret, ctx)]


def _rule_conv_gemm(A):
    x, w = A["x"], A["w"]
    S = emu.conv_gemm(_a(x), _a(w), bias=_a(A["bias"]), ks=A["ks"], stride=A["stride"], pad=A["pad"], out_dtype=_F64)
    n = A["ks"] * A["ks"] * x.shape[-1] + 1
    return [("out", _ret, _bounded(_epilogue(S, n, _UT, A["act"], None, A["residual"])))]


def _ln_err(x, eps, dx=None):
    """(normalised value n, bound on its error) of an fp32 LayerNorm over the last axis.  The mean (C terms) is off by
    <= gamma_C mean|x|; the variance -- mean((x-mean)^2) or mean(x^2) - mean^2, either form -- by <= gamma_{C+2}
    mean(x^2); rsqrtf by 2 ulp; the subtraction and product by one rounding each.  ``dx`` bounds errors already in x
    (the fused convolution's): it moves the mean by <= max dx and the variance by <= 2 max(dx) sd + max(dx)^2."""
    x = x.to(_F64)
    C = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    var = (x - mu).pow(2).mean(-1, keepdim=True) + eps
    sd = var.sqrt()
    n = (x - mu) / sd
    d_mu = _gamma(C) * x.abs().mean(-1, keepdim=True)
    d_var = _gamma(C + 2) * x.pow(2).mean(-1, keepdim=True)
    d_x = 0.0
    if dx is not None:
        D = dx.amax(-1, keepdim=True)
        d_mu, d_var, d_x = d_mu + D, d_var + 2 * D * sd + D * D, dx
    dn = (d_x + d_mu) / sd + n.abs() * (d_var / (2 * var) + 6 * _U)
    return n, dn


def _ln_out(n, dn, gamma, beta):
    g, b = _a(gamma), _a(beta)
    return g * dn + 2 * _U * (g * n.abs() + b)


def _rule_layernorm(A):
    n, dn = _ln_err(A["x"], A["eps"])
    arith = _ln_out(n, dn, A["gamma"], A["beta"])
    return [("out", _ret, _bounded(arith))]


def _rule_layernorm_patch2x2(A):
    B, H, W, C = A["x"].shape
    n, dn = _ln_err(A["x"], A["eps"])
    arith = _ln_out(n, dn, A["gamma"], A["beta"])
    arith = arith.view(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4 * C)
    return [("out", _ret, _bounded(arith))]


def _rule_patch_merge_ln(A):
    x = A["x"]
    cat = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], dim=-1)
    n, dn = _ln_err(cat, A["eps"])
    return [("out", _ret, _bounded(_ln_out(n, dn, A["gamma"], A["beta"]).reshape(-1, cat.shape[-1])))]


def _rule_dwconv_ln(A):
    x, wgt, bias = A["x"], A["wgt"], A["bias"]
    C = x.shape[-1]
    ks = int(round(wgt.shape[0] ** 0.5))
    pads = (ks // 2,) * 4
    y = emu._dw(x, wgt, bias, ks, 1, pads)                                      # exact convolution
    dy = _gamma(ks * ks + 1) * emu._dw(_a(x), _a(wgt), _a(bias), ks, 1, pads)  # its fp32 (fma) evaluation
    n, dn = _ln_err(y, A["eps"], dx=dy)
    return [("out", _ret, _bounded(_ln_out(n, dn, A["gamma"], A["beta"]).reshape(-1, C)))]


def _rule_dwconv_bias_act(A):
    x, ks, stride = A["x"], A["ks"], A["stride"]
    _, _, pads = emu._pads(x.shape[1], x.shape[2], ks, stride, A["padding"])
    M = emu._dw(_a(x), _a(A["wgt"]), _a(A["bias"]), ks, stride, pads)
    arith = _LIP.get(A["act"], 1.0) * _gamma(ks * ks + 1) * M + _act_err(A["act"], M)
    outs = [("out", _ret, _bounded(arith))]
    if A["pool_sum"] is not None:
        pool0 = A["pool_sum"].clone()

        def inc(s):
            return s.args["pool_sum"].to(_F64) - pool0.to(_F64)

        def vs_ref(kern, ref):
            # the stored outputs may differ from the reference's by their bound each; the kernel sums its own in fp32
            y = ref.ret.to(_F64)
            b = arith + (ulp_bf16(y) if ref.ret.dtype == torch.bfloat16 else 2 * _U * y.abs())
            hw = y.shape[1] * y.shape[2]
            return _bounded(b.sum(dim=(1, 2)) + _gamma(hw + 1) * (y.abs() + b).sum(dim=(1, 2)), flips=False)

        def vs_own(kern, ref):
            # the squeeze must see what the next layer reads: the fp32 (atomic) sum of the kernel's own stored output
            y = kern.ret.to(_F64)
            return _bounded(_gamma(y.shape[1] * y.shape[2] + 1) * y.abs().sum(dim=(1, 2)), flips=False)

        outs.append(("pool_sum increase", lambda s: inc(s), vs_ref))
        outs.append(("pool_sum increase = sum of own out", (lambda s: inc(s), lambda s: s.ret.to(_F64).sum((1, 2))),
                     vs_own))
    return outs


def _rule_global_avg_pool(A):
    x = A["x"]
    B, C = x.shape[0], x.shape[-1]
    hw = x.numel() // (B * C)
    m = _a(x).reshape(B, -1, C).mean(dim=1)
    return [("out", _ret, _bounded(_gamma(hw + 2) * m))]


def _softmax_err(qkv, B, N, H, dh, scale, bias=None, mask=None, row_map=None, nw_img=0, u=_U, rows=None):
    """Bounds on the errors of P = softmax(scale q k^T + bias + mask) and O = P V for an fp32 evaluation (exp / exp2,
    fp32 sums; ``u`` the unit of the q k^T accumulation): each score is off by <= gamma_{dh+3} (scale |q||k| + |bias| +
    |mask|); softmax only sees score differences, so p_j moves by <= p_j (2 max_j ds + u (|s_j| + |s_j - max|), the
    scaling and the exponent's argument, + 2 ulp of the exponential + the row sum and the division); O then by
    (dP |V|) + gamma_{N+2} (P |V|).  Also returns P |V|.  ``rows``: only the first ``rows`` queries (attention_cls)."""
    x = qkv.to(_F64)
    if row_map is not None:
        tok = nw_img * N
        idx = (torch.arange(B // nw_img, device=x.device)[:, None] * tok + row_map.long()[None, :]).reshape(-1)
        x = x[idx]
    q, k, v = x.view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    if rows is not None:
        q = q[:, :, :rows]
    s = scale * (q @ k.transpose(-1, -2))
    ds = scale * (q.abs() @ k.abs().transpose(-1, -2))
    if bias is not None:
        s, ds = s + bias.to(_F64)[None], ds + bias.to(_F64).abs()[None]
    if mask is not None:
        nm = mask.shape[0]
        shp = s.shape
        s = (s.view(B // nm, nm, H, N, N) + mask.to(_F64)[None, :, None]).view(shp)
        ds = (ds.view(B // nm, nm, H, N, N) + mask.to(_F64).abs()[None, :, None]).view(shp)
    ds = _gamma(dh + 3, u) * ds
    m = s.amax(-1, keepdim=True)
    p = torch.softmax(s, dim=-1)
    dp = p * (2 * ds.amax(-1, keepdim=True) + _U * (s.abs() + (s - m).abs()) + _gamma(N + 8))
    pv = p @ v.abs()
    do = dp @ v.abs() + _gamma(N + 2) * pv
    return do, dp, pv, idx if row_map is not None else None


def _blocked_softmax_err(s, ds, v, key_block, round_p, u_acc, u_arg=_U):
    """Bound on |kernel - statement| of O = softmax(s) V for a tensor-core kernel running the online softmax of
    ``emulate_bf16._softmax_pv`` over ``key_block``-key blocks, with P rounded by ``round_p`` (bf16 or TF32) before
    P V; before the output's own rounding.  ``s`` (..., Nq, N): the exact scores, ``ds`` the bound on the kernel's
    error of each, ``v`` (..., N, dh); ``u_acc`` the unit of the P V accumulation, ``u_arg`` that of the roundings of
    the exponent's argument (its scaling and the subtraction of the running max).  Per query row, with m_b the running
    max of key j's block, M the row max, c_j = exp(m_b - M) and Z = sum exp(s - M):

    * p_j = exp(s_j - m_b) is off by <= dp_j = p_j (2 max ds + u_arg (|s_j| + |s_j - m_b|) + 2 ulp of exp2) +
      2^-126 (results below fp32's normal range are flushed): the running maxima only shift the scores, so their
      error is one more max ds;
    * tie term: the kernel rounds a value within dp_j of p_j; where round_p(p_j - dp_j) != round_p(p_j + dp_j) that
      rounding may differ from the statement's by their difference (one spacing of P: ``ulp_bf16``, or TF32's
      2^(e-11)): (c tie / Z) @ |V|;
    * the rescale of block b to the row max, c_j, is off by <= eta_j = 2 max ds (the maxima at both ends; between them
      the alphas' exponents telescope) + u_arg (M - m_b) (their argument roundings) + 6u per rescale (exp2's 2 ulp,
      the products alpha O and alpha l);
    * O's numerator: (R eta) @ |V| + gamma_{N + 2 nblocks}(u_acc) R @ |V| with R = c round_p(p) / Z, the statement's P;
    * the row sum: relative error lam <= sum_j P_j (eta_j + dp_j / p_j) + gamma_{N + 2 nblocks + 3}(u) (its fp32
      sums and the division O / l), which moves O by (|O| + numerator error) lam."""
    N = s.shape[-1]
    nb = -(-N // key_block)
    blk = F.pad(s, (0, nb * key_block - N), value=-math.inf).unflatten(-1, (nb, key_block)).amax(-1)
    mb = torch.cummax(blk, dim=-1).values.repeat_interleave(key_block, dim=-1)[..., :N]
    M = mb[..., -1:]
    dsm = ds.amax(-1, keepdim=True)
    p = torch.exp(s - mb)
    eps = 2 * dsm + u_arg * (s.abs() + (mb - s)) + 4 * _U
    dp = p * eps + 2.0 ** -126
    tie = round_p(p + dp) - round_p((p - dp).clamp_min(0.0))
    c = torch.exp(mb - M)
    Z = torch.exp(s - M).sum(-1, keepdim=True)
    eta = 2 * dsm + u_arg * (M - mb) + 6 * _U * nb
    R = c * round_p(p) / Z
    av = v.abs()
    d_num = (R * eta + c * tie / Z) @ av + _gamma(N + 2 * nb, u_acc) * (R @ av)
    lam = (c * p / Z * (eta + eps)).sum(-1, keepdim=True) + _gamma(N + 2 * nb + 3)
    return d_num + ((R @ v).abs() + d_num) * lam


def _blocked_attention_bound(qkv, B, N, H, dh, scale, round_p):
    """Per-element bound of the ViT / PiT / TF32 tensor-core attention against ``emulate_bf16.attention`` in 64-key
    blocks: scores accumulated in the tensor cores (truncating fp32 adds, gamma_{dh+3}: dh products, the scaling by
    scale log2 e and that constant's rounding), then ``_blocked_softmax_err``.  Computed per chunk of images."""
    q, k, v = qkv.to(_F64).view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    out = []
    for c in emu.image_chunks(B, H, N):
        s = scale * (q[c] @ k[c].transpose(-1, -2))
        ds = _gamma(dh + 3, _UT) * scale * (q[c].abs() @ k[c].abs().transpose(-1, -2))
        out.append(_blocked_softmax_err(s, ds, v[c], emu.KEY_BLOCK, round_p, _UT))
    return _heads_to_rows(torch.cat(out), B, N, H, dh, None)


def _heads_to_rows(o, B, n, H, dh, idx):
    o = o.permute(0, 2, 1, 3).reshape(B * n, H * dh)
    if idx is not None:
        out = torch.empty_like(o)
        out[idx] = o
        o = out
    return o


def _rule_attention(A):
    qkv, B, N, H, dh = A["qkv"], A["B"], A["N"], A["H"], A["dh"]
    if qkv.dtype == torch.bfloat16:
        # The tensor-core kernel: P rounded to bf16 per 64-key block of its online softmax, as the statement does;
        # they differ by fp32 arithmetic and, where a P element lies that close to a rounding boundary, by one bf16
        # spacing of it (_blocked_softmax_err).
        bound = _blocked_attention_bound(qkv, B, N, H, dh, A["scale"], emu.round_bf16)
        return [("out", _ret, _bounded(bound))]
    do, dp, _, idx = _softmax_err(qkv, B, N, H, dh, A["scale"], A["bias"], A["mask"], A["row_map"], A["nw_img"])
    outs = [("out", _ret, _bounded(_heads_to_rows(do, B, N, H, dh, idx)))]
    if A["probs"] is not None:
        outs.append(("probs", lambda s: s.args["probs"], _bounded(dp)))
    return outs


def _rule_attention_cls(A):
    # fp32 SIMT softmax (__expf: ex2.approx of the rounded argument) and one bf16 output rounding.  (The 1.5e-2
    # absolute bound of tests/test_kernels_gpu.py::test_attention_cls_rows_equal_full_attention is below one bf16 ulp
    # for outputs >= 2, which ViT-Base at batch 256 produces.)
    B, T, H, dh, nq = A["B"], A["T"], A["H"], A["dh"], A["nq"]
    do, _, _, _ = _softmax_err(A["qkv"], B, T, H, dh, A["scale"], rows=nq)
    return [("out", _ret, _bounded(_heads_to_rows(do, B, nq, H, dh, None)))]


def _window_attention_bound(qkv, bias, mask, row_map, B, nw_img, N, H, dh, scale):
    """Per-element bound of the mma.sync window-attention kernel (csrc/window_attention.cu) against
    ``emulate_bf16.window_attention{,_tc}``: one block over the whole window (``key_block = N``), P rounded to bf16.
    ``bias`` (H, N, N), ``mask`` (nw_img, N, N) of 0 / -100 or None.  The kernel forms each logit in log2 units as
    fl(fl(fma(q.k, fl(scale), bias) + -100) * fl(log2 e)): the q.k of dh = 32 bf16 products accumulated in the tensor
    cores (gamma_dh with truncating adds), the rounding of scale to fp32, the fma, the mask add (masked pairs only), the
    product and the constant's own rounding -- at most dh + 5 roundings of magnitude <= scale |q||k| + |bias| + |mask|:
    ds = gamma_{dh+5}(2^-23) (scale |q||k| + |bias| + |mask|).  The rest (exp2, the fp32 row sum of the unrounded P,
    bf16 P V, the division) is ``_blocked_softmax_err``'s.  Computed per chunk of windows (``emu.image_chunks``)."""
    Bw = B * nw_img
    idx = (torch.arange(B, device=qkv.device)[:, None] * (nw_img * N) + row_map.long()[None, :]).reshape(-1)
    x = qkv[idx].view(Bw, N, 3, H, dh)
    b = bias.to(_F64)
    out = []
    for c in emu.image_chunks(Bw, H, N):
        q, k, v = x[c].to(_F64).permute(2, 0, 3, 1, 4)
        s = scale * (q @ k.transpose(-1, -2)) + b
        mag = scale * (q.abs() @ k.abs().transpose(-1, -2)) + b.abs()
        if mask is not None:
            mw = mask.to(_F64)[torch.arange(c.start, c.stop, device=qkv.device) % nw_img][:, None]
            s, mag = s + mw, mag + mw.abs()
        ds = _gamma(dh + 5, _UT) * mag
        out.append(_blocked_softmax_err(s, ds, v, N, emu.round_bf16, _UT))
    return _heads_to_rows(torch.cat(out), Bw, N, H, dh, idx)


def _rule_window_attention(A):
    mask = None
    if A["labels"] is not None:
        lab = A["labels"].view(A["nw_img"], A["N"])
        mask = torch.where(lab[:, None, :] != lab[:, :, None], -100.0, 0.0)
    bound = _window_attention_bound(A["qkv"], A["bias"], mask, A["row_map"], A["B"], A["nw_img"], A["N"], A["H"],
                                    A["dh"], A["scale"])
    return [("out", _ret, _bounded(bound))]


def _rule_window_attention_tc(A):
    N, maskbits = A["N"], A["maskbits"]
    mask = None
    if maskbits is not None:   # bit j of (window w, token i): tokens i and j lie in different shift regions
        bits = (maskbits[:, :N, None] >> torch.arange(N, device=maskbits.device)[None, None, :]) & 1
        mask = torch.where(bits.bool(), -100.0, 0.0)
    bound = _window_attention_bound(A["qkv"], A["bias_pad"][:, :N, :N], mask, A["row_map"], A["B"], A["nw_img"], N,
                                    A["H"], A["dh"], A["scale"])
    return [("out", _ret, _bounded(bound))]


def _rule_patchify(A):
    if A["mean"] is None:
        return [("out", _ret, _exact())]
    # (x * scale - mean) * inv_std: at most three fp32 roundings (two with an fma) of magnitude <= the sum of |terms|
    mag = emu.patchify(_a(A["img"]), A["p"], _F64, mean=-_a(A["mean"]), inv_std=_a(A["inv_std"]), scale=A["scale"])
    return [("out", _ret, _bounded(4 * _U * mag))]


def _rule_im2col(A):
    if A["pre"] is None:
        return [("out", lambda s: s.ret[0], _exact())]
    mean, inv_std, scale = A["pre"]
    mag, _, _ = emu.im2col(_a(A["x"]), A["ks"], A["stride"], A["padding"], _F64, groups=A["groups"],
                           pre=(-_a(mean), _a(inv_std), scale))      # the zero padding gets a zero bound: exact
    return [("out", lambda s: s.ret[0], _bounded(4 * _U * mag))]


def _rule_assemble_tokens(A):
    mag = emu.assemble_tokens(_a(A["patches"]), _a(A["cls"]), _a(A["dist"]), _a(A["pos"]), A["B"], A["P"], _F64)
    return [("out", _ret, _bounded(2 * _U * mag))]


def _rule_cast(A):
    return [("out", _ret, _exact())]


def _rule_group_norm(A):
    x, G = A["x"], A["groups"]
    B, H, W, C = x.shape
    cg = C // G
    xg = x.reshape(B, H * W, G, cg).permute(0, 2, 1, 3).reshape(B, G, H * W * cg)
    n, dn = _ln_err(xg, A["eps"])
    back = (lambda t: t.view(B, G, H * W, cg).permute(0, 2, 1, 3).reshape(B, H, W, C))
    n, dn = back(n), back(dn)
    g, b = _a(A["gamma"]), _a(A["beta"])
    r = _a(A["residual"]) if A["residual"] is not None else 0.0
    arith = _LIP.get(A["act"], 1.0) * (g * dn + 3 * _U * (g * n.abs() + b + r)) + _act_err(A["act"], g * n.abs() + b + r)
    return [("out", _ret, _bounded(arith))]


def _rule_blur_pool(A):
    mag = emu.blur_pool(_a(A["x"]), A["stride"])
    return [("out", _ret, _bounded(_gamma(10) * mag))]


def _rule_se_gate(A):
    ps, hw = A["pooled_sum"].to(_F64), float(A["hw"])
    wr, br, we, be = (t.to(_F64) for t in (A["w_reduce"], A["b_reduce"], A["w_expand"], A["b_expand"]))
    m = ps / hw
    C, rd = m.shape[1], wr.shape[0]
    z1 = m @ wr.t() + br
    mag1 = m.abs() @ wr.abs().t() + br.abs()
    h = emu._act(z1, A["act"])
    dh = _LIP.get(A["act"], 1.0) * (_gamma(C + 2) * mag1) + _act_err(A["act"], mag1)
    mag2 = h.abs() @ we.abs() + be.abs()
    dz2 = _gamma(rd + 1) * mag2 + dh @ we.abs()
    L = _LIP.get(A["gate_act"], 1.0)
    return [("out", _ret, _bounded(L * dz2 + _act_err(A["gate_act"], mag2)))]


def _rule_eca_gate(A):
    mean, w = A["mean"], A["w"]
    k = w.numel()
    mag = F.conv1d(F.pad(_a(mean), (k // 2, k // 2))[:, None], _a(w)[None, None])[:, 0]
    return [("out", _ret, _bounded(_LIP["sigmoid"] * _gamma(k) * mag + _act_err("sigmoid", mag)))]


def _gated_mag(x, gate):
    B, C = gate.shape
    return (_a(x).view(B, -1, C) * _a(gate)[:, None, :]).view(x.shape)


def _rule_scale_channels_(A):
    return [("x", lambda s: s.args["x"], _bounded(_U * _gated_mag(A["x"], A["gate"])))]


def _rule_scale_add_act_(A):
    mag = _gated_mag(A["x"], A["gate"]) + _a(A["shortcut"])
    arith = _LIP.get(A["act"], 1.0) * 2 * _U * mag + _act_err(A["act"], mag)
    return [("x", lambda s: s.args["x"], _bounded(arith))]


def _rule_pool2d(A):
    if A["mode"] != "avg":
        return [("out", _ret, _exact())]
    mag = emu.pool2d(_a(A["x"]), A["ks"], A["stride"], A["padding"], "avg")
    return [("out", _ret, _bounded(_gamma(A["ks"] * A["ks"] + 2) * mag))]


def _rule_grouped_conv(A):
    x, cg, ks = A["x"], A["cg"], A["ks"]
    M = emu.grouped_conv(_a(x), _a(A["wgt"]), _a(A["bias"]), cg, ks, A["stride"], A["pad"])
    arith = _LIP.get(A["act"], 1.0) * _gamma(ks * ks * cg + 1) * M + _act_err(A["act"], M)
    return [("out", _ret, _bounded(arith))]


def _ret(s):
    return s.ret


_RULES = {
    "gemm": _rule_gemm, "gemm_gated": _rule_gemm_gated, "mlp_fused": _rule_mlp_fused, "conv_gemm": _rule_conv_gemm,
    "layernorm": _rule_layernorm, "layernorm_patch2x2": _rule_layernorm_patch2x2,
    "patch_merge_ln": _rule_patch_merge_ln, "attention": _rule_attention, "attention_cls": _rule_attention_cls,
    "window_attention": _rule_window_attention, "window_attention_tc": _rule_window_attention_tc,
    "patchify": _rule_patchify, "assemble_tokens": _rule_assemble_tokens, "cast": _rule_cast,
    "dwconv_ln": _rule_dwconv_ln, "dwconv_bias_act": _rule_dwconv_bias_act, "global_avg_pool": _rule_global_avg_pool,
    "im2col": _rule_im2col, "group_norm": _rule_group_norm, "blur_pool": _rule_blur_pool, "se_gate": _rule_se_gate,
    "scale_channels_": _rule_scale_channels_, "pool2d": _rule_pool2d, "grouped_conv": _rule_grouped_conv,
    "eca_gate": _rule_eca_gate, "scale_add_act_": _rule_scale_add_act_,
}
# Launchers of emulate_bf16._EMULATED that are shape predicates, not kernels.
PREDICATES = ("mlp_fused_supported",)
SHADOWED = tuple(n for n in emu._EMULATED if n not in PREDICATES)
assert set(SHADOWED) == set(_RULES), set(SHADOWED) ^ set(_RULES)


# ---------------------------------------------------------------------------------------------------- the harness
class _Launch:
    def __init__(self, args, ret):
        self.args, self.ret = args, ret


class Census:
    """One row per checked output of every shadowed launch, in launch order."""

    def __init__(self):
        self.rows = []
        self.launches = 0

    def ops(self):
        return {r["op"] for r in self.rows}

    def failures(self):
        return [r for r in self.rows if not r["ok"]]

    @staticmethod
    def _fmt(r):
        return (f"{'ok  ' if r['ok'] else 'FAIL'} {r['op']:<20} {r['site']:<18} #{r['index']:<4} {r['output']:<34} "
                f"worst {r['worst']:8.3f} x bound  flips {100 * r['flips']:6.3f} %  {r['args']}")

    def table(self):
        return "\n".join(self._fmt(r) for r in self.rows)

    def assert_ok(self):
        bad = self.failures()
        assert not bad, f"{len(bad)} shadowed output(s) outside their bound:\n" + "\n".join(self._fmt(r) for r in bad)


def _call_site():
    """file:line of the innermost caller in the model code (tfimm/architectures/*.py, or tfimm/models/*.py)."""
    f = sys._getframe(2)
    while f is not None:
        fn = f.f_code.co_filename
        if os.sep + "tfimm" + os.sep in fn and os.sep + "backend" + os.sep not in fn:
            return f"{os.path.basename(fn)}:{f.f_lineno}"
        f = f.f_back
    return "(direct call)"


_DT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.uint8: "u8", torch.int32: "i32", torch.int64: "i64",
       torch.float64: "f64"}


def _describe(args):
    parts = []
    for k, v in args.items():
        if v is None:
            continue
        if torch.is_tensor(v):
            parts.append(f"{k}={_DT.get(v.dtype, v.dtype)}{tuple(v.shape)}")
        elif isinstance(v, (tuple, list)):
            parts.append(f"{k}=({', '.join(_DT.get(t.dtype, '?') + str(tuple(t.shape)) if torch.is_tensor(t) else repr(t) for t in v)})")
        elif isinstance(v, torch.dtype):
            parts.append(f"{k}={_DT.get(v, v)}")
        elif isinstance(v, float):
            parts.append(f"{k}={v:.4g}")
        else:
            parts.append(f"{k}={v}")
    return " ".join(parts)


@contextmanager
def _float64():
    saved, emu._HP = emu._HP, _F64
    try:
        yield
    finally:
        emu._HP = saved


def _tensors(v):
    if torch.is_tensor(v):
        yield v
    elif isinstance(v, (tuple, list)):
        for e in v:
            yield from _tensors(e)


def _shadow(name, kernel, census):
    ref_fn = getattr(emu, name)
    sig = inspect.signature(ref_fn)
    rule = _RULES[name]

    def launcher(*args, **kwargs):
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"oracle.shadow: ops.{name} called during CUDA-graph capture; shadowed launches are "
                               "checked one by one and only run in eager forward passes")
        site, index = _call_site(), census.launches
        census.launches += 1
        memo = {}

        def snap(v):   # clone, keeping aliases aliased (out is residual, x is written in place, ...)
            if torch.is_tensor(v):
                key = (v.data_ptr(), v.dtype, tuple(v.shape), v.stride())
                if key not in memo:
                    memo[key] = v.clone()
                return memo[key]
            if isinstance(v, (tuple, list)):
                return type(v)(snap(e) for e in v)
            return v

        ref_args, ref_kwargs = [snap(a) for a in args], {k: snap(v) for k, v in kwargs.items()}
        rb = sig.bind(*ref_args, **ref_kwargs)
        rb.apply_defaults()
        with torch.no_grad(), _float64():
            outputs = rule(rb.arguments)
            ref = _Launch(rb.arguments, ref_fn(*ref_args, **ref_kwargs))
        kb = sig.bind(*args, **kwargs)
        kb.apply_defaults()
        kern = _Launch(kb.arguments, kernel(*args, **kwargs))
        if any(t.is_cuda for t in _tensors(list(kb.arguments.values()))):
            torch.cuda.synchronize()
        desc = _describe(kb.arguments)
        written = set()
        with torch.no_grad():
            for label, get, ctx in outputs:
                kget, rget = get if isinstance(get, tuple) else (get, get)
                k_t, r_t = kget(kern), rget(ref if not isinstance(get, tuple) else kern)
                if callable(ctx):
                    ctx = ctx(kern, ref)
                ok, worst, flips = check(name, k_t, r_t, ctx)
                census.rows.append(dict(op=name, site=site, index=index, output=label, ok=ok, worst=worst,
                                        flips=flips, args=desc, cite=ctx.get("cite")))
                for t in _tensors(kget(kern)):
                    written.add(t.data_ptr())
            for arg, v in kb.arguments.items():     # inputs come back untouched
                for i, t in enumerate(_tensors(v)):
                    if t.data_ptr() in written or (arg == "pool_sum" and name == "dwconv_bias_act"):
                        continue
                    r_t = list(_tensors(rb.arguments[arg]))[i]
                    ok = torch.equal(t, r_t)
                    if not ok:
                        census.rows.append(dict(op=name, site=site, index=index, output=f"input {arg} unchanged",
                                                ok=False, worst=math.inf, flips=0.0, args=desc, cite=None))
        del ref, rb, ref_args, ref_kwargs, memo
        return kern.ret

    launcher.__name__ = name
    return launcher


@contextmanager
def shadowed_ops():
    """Inside the block every ``tfimm.backend.ops`` launcher of ``SHADOWED`` runs shadowed (see the module docstring);
    yields the ``Census``.  Whatever ``ops.<name>`` is on entry is "the kernel": the real launcher, or -- for a CPU
    rehearsal of this harness -- a stand-in installed before."""
    from tfimm.backend import ops

    census = Census()
    saved = {n: getattr(ops, n) for n in SHADOWED}
    for n in SHADOWED:
        setattr(ops, n, _shadow(n, saved[n], census))
    try:
        with torch.no_grad():
            yield census
    finally:
        for n, f in saved.items():
            setattr(ops, n, f)
