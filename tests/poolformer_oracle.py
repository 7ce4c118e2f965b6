"""TEST INFRASTRUCTURE ONLY -- the PoolFormer launchers (``tfimm.backend.poolformer_ops``) on top of
oracle/emulate_bf16.py and oracle/shadow.py.

Each launcher gets
* a statement at the kernels' storage points: the fp32 stream as stored, the one-group GroupNorm of the reference in
  the emulation's arithmetic (float64 by default) with the image's exact statistics, one rounding to the output's
  storage type at the end.  The token mixer's statement is the reference's form, x + ls1 (pool(GN(x)) - GN(x)) with the
  "same" pool over zero-padded GN(x) and padded cells excluded from the count -- not the kernel's identity, so the
  shadow check of every mixer launch also checks the identity;
* a derived error bound for the op-by-op shadow harness (``_rule_*``).

The statistics error model (``_stats_err``), for an image of N values in S chunks of 4096 held by 256 threads: a chunk
sum is a fixed tree of depth <= 19 (16 values per thread, a warp tree of 5, 8 warp totals in order), so a chunk mean is
off by <= gamma_20 max|x|; the centred M2 is off by gamma_23 (M2 + n d^2) + n d^2 for a mean error d (the sum of
(x - m)^2 about a wrong centre grows by exactly n d^2); Chan's merge of S partials adds <= 4 roundings per step, at most
S + 5 steps deep.  With g = gamma_{24 + 4S}: |d mean| <= g max|x| and |d var| <= g var + 4 g max|x| D + 4 (g max|x|)^2,
D the largest distance of a chunk mean from the image mean (the merge's d^2 n f term carries the chunk means' errors).
rstd = rsqrtf(var + eps) is then off by a relative (d var) / (var + eps) + 4 u.

``emulated_poolformer_ops()`` / ``shadowed_poolformer_ops()`` are ``emulated_ops()`` / ``shadowed_ops()`` with these
launchers added.
"""
from contextlib import contextmanager

import torch
import torch.nn.functional as F

from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64
CHUNK = 4096


def _splits(H, W, C):
    return (H * W * C + CHUNK - 1) // CHUNK


def _chunks(x, dtype):
    """x (B, H, W, C) -> (values (B, S, CHUNK) zero-filled past the image, mask of the real values) in dtype."""
    B, H, W, C = x.shape
    N, S = H * W * C, _splits(H, W, C)
    v = F.pad(x.to(dtype).reshape(B, N), (0, S * CHUNK - N)).view(B, S, CHUNK)
    mask = F.pad(torch.ones((B, N), dtype=dtype, device=x.device), (0, S * CHUNK - N)).view(B, S, CHUNK)
    return v, mask


def partials_of(x, dtype=_F64):
    """(count, mean, M2) of every chunk of x, (B, S, 3) in dtype."""
    v, mask = _chunks(x, dtype)
    n = mask.sum(-1)
    mean = v.sum(-1) / n
    m2 = (((v - mean[..., None]) * mask) ** 2).sum(-1)
    return torch.stack((n, mean, m2), -1)


def _gn(x, gamma, beta, eps):
    """The reference's one-group GroupNorm of x (B, H, W, C) in the emulation's arithmetic, exact image statistics."""
    hp = emu._HP
    xh = x.to(hp)
    mean = xh.mean(dim=(1, 2, 3), keepdim=True)
    var = ((xh - mean) ** 2).mean(dim=(1, 2, 3), keepdim=True)
    return (xh - mean) / torch.sqrt(var + eps) * gamma.to(hp) + beta.to(hp)


def _pool_same(n):
    return F.avg_pool2d(n.permute(0, 3, 1, 2), 3, stride=1, padding=1, count_include_pad=False).permute(0, 2, 3, 1)


def gn1_partials(x):
    return partials_of(x, emu._HP).to(torch.float32)


def poolformer_mixer(x, partials, gamma, beta, ls1, eps):
    n = _gn(x, gamma, beta, eps)
    out = (x.to(emu._HP) + ls1.to(emu._HP) * (_pool_same(n) - n)).to(torch.float32).contiguous()
    return out, gn1_partials(out)


def gn1_apply(x, partials, gamma, beta, eps, out_dtype):
    B, H, W, C = x.shape
    return _gn(x, gamma, beta, eps).reshape(B * H * W, C).to(out_dtype)


# --------------------------------------------------------------------- float32 models of the kernels' algorithms
def merge_partials(partials):
    """(mean, rstd-less variance) per image from (B, S, 3) partials by Chan's formula, in the partials' dtype, s in
    order."""
    n, mean, m2 = (partials[:, 0, i].clone() for i in range(3))
    for s in range(1, partials.shape[1]):
        nb, mb, qb = partials[:, s, 0], partials[:, s, 1], partials[:, s, 2]
        nn = n + nb
        d = mb - mean
        f = nb / nn
        mean = mean + d * f
        m2 = m2 + qb + d * d * n * f
        n = nn
    return mean, m2 / n


def _rstd_of(partials, eps):
    mean, var = merge_partials(partials)
    B = partials.shape[0]
    return mean.view(B, 1, 1, 1), (1.0 / torch.sqrt(var + eps)).view(B, 1, 1, 1)


def gn1_partials_kernel_form(x):
    return partials_of(x, torch.float32)


def poolformer_mixer_kernel_form(x, partials, gamma, beta, ls1, eps):
    """What the kernel computes, in float32: x + ls1 gamma rstd mean_j (x_j - x), rstd from the partials."""
    _, r = _rstd_of(partials, eps)
    B, H, W, C = x.shape
    pad = F.pad(x, (0, 0, 1, 1, 1, 1))
    ok = F.pad(torch.ones((1, H, W, 1), device=x.device), (0, 0, 1, 1, 1, 1))
    acc, cnt = torch.zeros_like(x), torch.zeros((1, H, W, 1), device=x.device)
    for dy in range(3):
        for dx in range(3):
            m = ok[:, dy:dy + H, dx:dx + W]
            acc, cnt = acc + (pad[:, dy:dy + H, dx:dx + W] - x) * m, cnt + m
    out = (x + ls1 * gamma * r * (acc / cnt)).contiguous()
    return out, partials_of(out, torch.float32)


def gn1_apply_kernel_form(x, partials, gamma, beta, eps, out_dtype):
    mean, r = _rstd_of(partials, eps)
    B, H, W, C = x.shape
    return ((x - mean) * (r * gamma) + beta).reshape(B * H * W, C).to(out_dtype)


@contextmanager
def kernel_forms():
    """The ``poolformer_ops`` launchers replaced by the float32 models of their kernels (CPU rehearsals)."""
    from tfimm.backend import poolformer_ops

    forms = {"gn1_partials": gn1_partials_kernel_form, "poolformer_mixer": poolformer_mixer_kernel_form,
             "gn1_apply": gn1_apply_kernel_form}
    saved = {n: getattr(poolformer_ops, n) for n in forms}
    for n, f in forms.items():
        setattr(poolformer_ops, n, f)
    try:
        yield
    finally:
        for n, f in saved.items():
            setattr(poolformer_ops, n, f)


# ------------------------------------------------------------------------------------------------------ the bounds
_U = shadow._U


def _stats_err(x, eps):
    """Per image, shaped (B, 1, 1, 1): exact mean, exact rstd, bound on rstd's relative error, bound on the mean's
    error (module docstring)."""
    B, H, W, C = x.shape
    S = _splits(H, W, C)
    xd = x.to(_F64).reshape(B, -1)
    m = xd.mean(1)
    var = ((xd - m[:, None]) ** 2).mean(1)
    mx = xd.abs().max(1).values
    p = partials_of(x)
    D = (p[..., 1] - m[:, None]).abs().max(1).values
    g = shadow._gamma(24 + 4 * S)
    dvar = g * var + 4 * g * mx * D + 4 * (g * mx) ** 2
    eps_r = dvar / (var + eps) + 4 * _U
    shape = (B, 1, 1, 1)
    return (m.view(shape), (1.0 / torch.sqrt(var + eps)).view(shape), eps_r.view(shape), (g * mx).view(shape))


def _partials_bound(x):
    """Bound on each (count, mean, M2) of x's partials computed in fp32 from x as stored, including the statement's own
    rounding of mean and M2 to fp32; counts are exact."""
    v, mask = _chunks(x, _F64)
    p = partials_of(x)
    n = p[..., 0]
    d = shadow._gamma(20) * (v.abs().sum(-1) / n)
    dm2 = shadow._gamma(23) * (p[..., 2] + n * d * d) + n * d * d
    return torch.stack((torch.zeros_like(n), d + _U * p[..., 1].abs(), dm2 + _U * p[..., 2]), -1)


def _rule_gn1_partials(A):
    return [("out", shadow._ret, shadow._bounded(_partials_bound(A["x"]), flips=False))]


def _neighbour_sums(x):
    """(mean_j (x_j - x_i), mean_j |x_j - x_i|) over the in-bounds 3 x 3 neighbours of every pixel, float64."""
    xd = x.to(_F64)
    B, H, W, C = xd.shape
    pad = F.pad(xd, (0, 0, 1, 1, 1, 1))
    ok = F.pad(torch.ones((1, H, W, 1), dtype=_F64, device=x.device), (0, 0, 1, 1, 1, 1))
    s = torch.zeros_like(xd)
    a = torch.zeros_like(xd)
    cnt = torch.zeros((1, H, W, 1), dtype=_F64, device=x.device)
    for dy in range(3):
        for dx in range(3):
            m = ok[:, dy:dy + H, dx:dx + W]
            diff = (pad[:, dy:dy + H, dx:dx + W] - xd) * m
            s, a, cnt = s + diff, a + diff.abs(), cnt + m
    return s / cnt, a / cnt


def _rule_poolformer_mixer(A):
    """out = x + k rstd mean_j (x_j - x): each difference rounds once and nine of them are summed (gamma_10 of the mean
    of |x_j - x|, the division included), k = ls1 gamma and its product with rstd round twice, and the fma and the
    statement's own store once each."""
    x = A["x"]
    _, r, eps_r, _ = _stats_err(x, A["eps"])
    k = (A["ls1"].to(_F64) * A["gamma"].to(_F64)).abs()
    dmean, dabs = _neighbour_sums(x)
    t = k * r * dmean.abs()
    err = t * (eps_r + 3 * _U) + k * r * (1 + eps_r) * shadow._gamma(10) * dabs + 2 * _U * (x.to(_F64).abs() + t)

    def partials_ctx(kern, ref):
        return shadow._bounded(_partials_bound(kern.ret[0]), flips=False)

    return [("out", lambda s: s.ret[0], shadow._bounded(err)),
            ("out_partials of the stored out", (lambda s: s.ret[1], lambda s: partials_of(s.ret[0])), partials_ctx)]


def _rule_gn1_apply(A):
    """y = (x - mean) (rstd gamma) + beta in one fma: the subtraction and rstd gamma round once each, the fma once, the
    statement's fp32 store once more; the mean's error passes through rstd gamma."""
    x = A["x"]
    B, H, W, C = x.shape
    m, r, eps_r, dm = _stats_err(x, A["eps"])
    g, b = A["gamma"].to(_F64).abs(), A["beta"].to(_F64).abs()
    nrm = (x.to(_F64) - m).abs() * r
    err = g * (nrm * (eps_r + 3 * _U) + r * (1 + eps_r) * dm) + 2 * _U * (g * nrm + b)
    return [("out", shadow._ret, shadow._bounded(err.reshape(B * H * W, C)))]


_POOLFORMER = {"gn1_partials": (gn1_partials, _rule_gn1_partials),
               "poolformer_mixer": (poolformer_mixer, _rule_poolformer_mixer),
               "gn1_apply": (gn1_apply, _rule_gn1_apply)}


@contextmanager
def emulated_poolformer_ops(arithmetic=torch.float64):
    """``emulate_bf16.emulated_ops()`` plus the statements of the ``poolformer_ops`` launchers."""
    from tfimm.backend import poolformer_ops

    saved = {n: getattr(poolformer_ops, n) for n in _POOLFORMER}
    with emu.emulated_ops(arithmetic):
        for n, (f, _) in _POOLFORMER.items():
            setattr(poolformer_ops, n, f)
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(poolformer_ops, n, f)


@contextmanager
def shadowed_poolformer_ops():
    """``shadow.shadowed_ops()`` plus every ``poolformer_ops`` launcher checked against its statement within its bound;
    yields the shared ``Census``.  Whatever ``poolformer_ops.<name>`` is on entry is "the kernel"."""
    from tfimm.backend import poolformer_ops

    saved = {n: getattr(poolformer_ops, n) for n in _POOLFORMER}
    for n, (f, rule) in _POOLFORMER.items():
        setattr(emu, n, f)
        shadow._RULES[n] = rule
    try:
        with shadow.shadowed_ops() as census:
            for n in _POOLFORMER:
                setattr(poolformer_ops, n, shadow._shadow(n, saved[n], census))
            yield census
    finally:
        for n, f in saved.items():
            setattr(poolformer_ops, n, f)
            delattr(emu, n)
            del shadow._RULES[n]
