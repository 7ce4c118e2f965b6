"""TEST INFRASTRUCTURE ONLY -- the Segment Anything attention launcher on top of oracle/emulate_bf16.py and
oracle/shadow.py.

``tfimm.backend.sam_ops.relpos_attention`` (softmax(scale q k^T + rel_h + rel_w) v over global or windowed sequences,
csrc/relpos_attention.cu) gets

* a float64 statement with the kernels' rounding points (``relpos_attention``): q, k, v are the stored qkv values (bf16
  or fp32), the window padding's keys / values are the stored qkv bias, the relative-position terms use the unscaled q
  and the fp32 tables as they are; in bf16, the online softmax of ``emulate_bf16._softmax_pv`` over 64-key blocks, P
  rounded to bf16 per block (relative to the running row max) and the row sum of the unrounded P -- what the
  tensor-core kernel does;
* a derived error bound for the op-by-op shadow harness (``relpos_bound``).

``emulated_sam_ops()`` / ``shadowed_sam_ops()`` are ``emulated_ops()`` / ``shadowed_ops()`` with this launcher added.
"""
from contextlib import contextmanager

import torch

from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64


def seq_index(gh, gw, window, device=None):
    """(nseq, S_h * S_w) grid row of every sequence token (-1: window padding), and (S_h, S_w)."""
    sh, sw = (window, window) if window else (gh, gw)
    nwh, nww = -(-gh // sh), -(-gw // sw)
    y = torch.arange(nwh * sh, device=device)[:, None]
    x = torch.arange(nww * sw, device=device)[None, :]
    idx = torch.where((y < gh) & (x < gw), y * gw + x, torch.full_like(y * x, -1))
    return idx.view(nwh, sh, nww, sw).permute(0, 2, 1, 3).reshape(nwh * nww, sh * sw), sh, sw


def _sequences(qkv, B, gh, gw, H, dh, rel_h, rel_w, window, pad_bias, hp):
    """q, k, v (B, nseq, H, N, dh) in ``hp``; the relative-position terms (B, nseq, H, N, N) of both axes with their
    magnitude sums |q| |R|; and the sequence index."""
    idx, sh, sw = seq_index(gh, gw, window, qkv.device)
    x = qkv.to(hp).view(B, gh * gw, 3, H, dh)
    pad = pad_bias.to(hp).view(3, H, dh) if pad_bias is not None else torch.zeros(3, H, dh, dtype=hp, device=x.device)
    seq = torch.where((idx >= 0)[None, :, :, None, None, None], x[:, idx.clamp(min=0)], pad)
    q, k, v = (t.permute(0, 1, 3, 2, 4) for t in seq.unbind(3))
    N = sh * sw
    j = torch.arange(N, device=qkv.device)
    ty, tx = j // sw, j % sw
    rh = rel_h.to(hp)[ty[:, None] - torch.arange(sh, device=j.device)[None, :] + sh - 1]   # (N, S_h, dh)
    rw = rel_w.to(hp)[tx[:, None] - torch.arange(sw, device=j.device)[None, :] + sw - 1]
    return q, k, v, rh, rw, ty, tx, idx


def _rel(q, rh, rw, ty, tx):
    """rel_h[i, ky(j)] + rel_w[i, kx(j)] for every query i and key j: (..., N, N)."""
    return torch.einsum("...nd,nkd->...nk", q, rh)[..., ty] + torch.einsum("...nd,nkd->...nk", q, rw)[..., tx]


def _to_rows(o, idx, B, T):
    """(B, nseq, H, N, dh) -> (B * T, H * dh), dropping the window padding."""
    Bq, nseq, H, N, dh = o.shape
    o = o.permute(0, 1, 3, 2, 4).reshape(B, nseq * N, H * dh)
    keep = idx.reshape(-1) >= 0
    out = torch.empty((B, T, H * dh), dtype=o.dtype, device=o.device)
    out[:, idx.reshape(-1)[keep]] = o[:, keep]
    return out.reshape(B * T, H * dh)


def relpos_attention(qkv, B, gh, gw, H, dh, scale, rel_h, rel_w, window=0, pad_bias=None):
    hp = emu._HP
    q, k, v, rh, rw, ty, tx, idx = _sequences(qkv, B, gh, gw, H, dh, rel_h, rel_w, window, pad_bias, hp)
    outs = []
    for h in range(H):     # one head at a time: a global (N, N) score matrix at N = 4096 is 128 MB per image
        qh, kh, vh = q[:, :, h], k[:, :, h], v[:, :, h]
        s = scale * (qh @ kh.transpose(-1, -2)) + _rel(qh, rh, rw, ty, tx)
        if qkv.dtype == torch.bfloat16:
            o, _ = emu._softmax_pv(s, vh, emu.round_bf16, emu.KEY_BLOCK)
        else:
            o = torch.softmax(s, dim=-1) @ vh
        outs.append(o)
    return _to_rows(torch.stack(outs, dim=2), idx, B, gh * gw).contiguous().to(qkv.dtype)


def relpos_bound(qkv, B, gh, gw, H, dh, scale, rel_h, rel_w, window=0, pad_bias=None):
    """Bound on |kernel - relpos_attention| per output element (before the output's own bf16 rounding, which the
    shadow rule adds as one ulp).  Derivation, per query row:

    * each logit s = scale q.k + q.R_h + q.R_w is off by ds <= gamma_{dh+3}(u) scale |q||k| + (gamma_{2dh+3}(u) +
      e_R) (|q||R_h| + |q||R_w|): fp32 accumulation of exact products (u = 2^-23 on the tensor cores, which truncate;
      2^-24 in the SIMT kernel) and, in bf16, R carried as a bf16 hi + lo pair (e_R = 2^-17);
    * bf16 (tensor-core kernel, the statement's online softmax over 64-key blocks): ``shadow._blocked_softmax_err``
      with 4u per unit of |s_j| + |s_j - m| for the argument (the table sum, its scaling by log2(e), the fma);
    * fp32 (SIMT kernel, one pass): softmax sees differences of logits only, so p_j moves by <= p_j (2 max ds + 4u
      (|s_j| + |s_j - m|) + gamma_{N+8}): the argument's scaling by log2(e), exp2, the row sum and the division;
      O = P V then moves by (dP |V|) + gamma_{N+2} (P |V|).
    This is the bound of the ViT attention (oracle/shadow.py, _rule_attention) with the relative-position terms in the
    logit error."""
    bf16 = qkv.dtype == torch.bfloat16
    u = shadow._UT if bf16 else shadow._U
    e_r = 2.0 ** -17 if bf16 else 0.0
    q, k, v, rh, rw, ty, tx, idx = _sequences(qkv, B, gh, gw, H, dh, rel_h, rel_w, window, pad_bias, _F64)
    N = q.shape[-2]
    outs = []
    for h in range(H):
        qh, kh, vh = q[:, :, h], k[:, :, h], v[:, :, h]
        s = scale * (qh @ kh.transpose(-1, -2)) + _rel(qh, rh, rw, ty, tx)
        ds = (shadow._gamma(dh + 3, u) * scale * (qh.abs() @ kh.abs().transpose(-1, -2))
              + (shadow._gamma(2 * dh + 3, u) + e_r) * _rel(qh.abs(), rh.abs(), rw.abs(), ty, tx))
        if bf16:
            do = shadow._blocked_softmax_err(s, ds, vh, emu.KEY_BLOCK, emu.round_bf16, u, u_arg=4 * shadow._U)
        else:
            m = s.amax(-1, keepdim=True)
            p = torch.softmax(s, dim=-1)
            dp = p * (2 * ds.amax(-1, keepdim=True) + 4 * shadow._U * (s.abs() + (s - m).abs()) + shadow._gamma(N + 8))
            do = dp @ vh.abs() + shadow._gamma(N + 2) * (p @ vh.abs())
        outs.append(do)
    return _to_rows(torch.stack(outs, dim=2), idx, B, gh * gw)


def _rule_relpos_attention(A):
    bound = relpos_bound(A["qkv"], A["B"], A["gh"], A["gw"], A["H"], A["dh"], A["scale"], A["rel_h"], A["rel_w"],
                         A["window"], A["pad_bias"])
    return [("out", shadow._ret, shadow._bounded(bound))]


@contextmanager
def emulated_sam_ops(arithmetic=torch.float64):
    """``emulate_bf16.emulated_ops()`` plus the float64 statement of ``sam_ops.relpos_attention``."""
    from tfimm.backend import sam_ops

    saved = sam_ops.relpos_attention
    with emu.emulated_ops(arithmetic):
        sam_ops.relpos_attention = relpos_attention
        try:
            yield
        finally:
            sam_ops.relpos_attention = saved


@contextmanager
def shadowed_sam_ops():
    """``shadow.shadowed_ops()`` plus ``sam_ops.relpos_attention`` checked against ``relpos_attention`` within
    ``relpos_bound``; yields the shared ``Census``.  Whatever ``sam_ops.relpos_attention`` is on entry is "the
    kernel"."""
    from tfimm.backend import sam_ops

    saved = sam_ops.relpos_attention
    emu.relpos_attention = relpos_attention
    shadow._RULES["relpos_attention"] = _rule_relpos_attention
    try:
        with shadow.shadowed_ops() as census:
            sam_ops.relpos_attention = shadow._shadow("relpos_attention", saved, census)
            yield census
    finally:
        sam_ops.relpos_attention = saved
        del emu.relpos_attention
        del shadow._RULES["relpos_attention"]
