"""TEST INFRASTRUCTURE ONLY -- bf16-emulating oracle: the engine's graph with EXACT per-op arithmetic.

Why: ``north_star`` asks for logits within 1e-3 of the reference in bf16.  The engine measures 4-7e-3 against the
fp32 oracle.  That number mixes two things: (1) the rounding of tensors the engine STORES in bf16 (GEMM operands,
qkv, the softmax probabilities fed to PV, the MLP hidden tensor, the activation stream of the BN families) -- inherent
to "bf16 operands, fp32 accumulate" -- and (2) whatever the kernels approximate internally (tanh-form GELU,
``tanh.approx`` swish, ``ex2.approx`` softmax, fp16 staging in the depthwise kernel, accumulation order).  This module
separates them: it provides a drop-in replacement for every function of ``tfimm.backend.ops`` written with plain
torch fp32 arithmetic (exact erf / sigmoid / exp, fp32 accumulation), rounding to bf16 ONLY where the engine's kernels
store bf16.  Running the engine's own host orchestration (``tfimm/architectures/*.py``) on top of it gives the logits
an ideal bf16-operand implementation of the same graph would produce; ``engine - emulated`` is then the kernels' own
contribution and is what the GPU tests bound at 1e-3.

That the emulated graph IS the oracle's graph is itself tested: with ``precision="fp32"`` models (no bf16 storage
anywhere) the emulation reproduces ``oracle/*.py`` -- which is pinned to the reference -- to ~1e-6
(tests/test_models_gpu.py::test_emulated_graph_equals_oracle_in_fp32).

Usage (tests only)::

    with emulate_bf16.emulated_ops():
        y_ideal = model(x)          # same model object, same plan tensors, torch arithmetic
    y_engine = model(x)             # CUDA kernels
"""
import math
from contextlib import contextmanager

import torch
import torch.nn.functional as F

# Arithmetic precision of the emulation: float64, so that "exact per-op arithmetic" is not a figure of speech (cuDNN's
# fp32 convolution algorithms -- Winograd / FFT -- are themselves only ~1e-5 accurate).
_HP = torch.float64

ACT_NAMES = (None, "", "linear", "none", "gelu", "swish", "silu", "relu", "relu6", "tanh", "sigmoid")


def _act(x, act):
    if act in (None, "", "linear", "none"):
        return x
    if act == "gelu":  # Keras default: exact erf form (layers/factory.py:6-13 of the reference)
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    if act in ("swish", "silu"):
        return x * torch.sigmoid(x)
    if act == "relu":
        return torch.relu(x)
    if act == "relu6":
        return torch.clamp(x, 0.0, 6.0)
    if act == "tanh":
        return torch.tanh(x)
    if act == "sigmoid":
        return torch.sigmoid(x)
    raise ValueError(f"Unknown activation: {act}.")


def act_code(act):
    if act not in ACT_NAMES:
        raise ValueError(f"Unknown activation: {act}.")
    return 0


def _store(y, out, dtype):
    """Round ``y`` (fp32) to the storage dtype; write into ``out`` (possibly a strided view) if given."""
    if out is not None:
        out.copy_(y.to(out.dtype))
        return out
    return y.to(dtype)


def gemm(a, w, bias=None, act=None, gamma=None, residual=None, out=None, out_dtype=None, block_n=0,
         act_after_residual=False):
    y = a.to(_HP) @ w.to(_HP).t()
    if bias is not None:
        y = y + bias.to(_HP)
    r = residual.to(_HP) if residual is not None else None
    if act_after_residual:
        if gamma is not None:
            y = y * gamma.to(_HP)
        if r is not None:
            y = y + r
        y = _act(y, act)
    else:
        y = _act(y, act)
        if gamma is not None:
            y = y * gamma.to(_HP)
        if r is not None:
            y = y + r
    dt = out_dtype or (residual.dtype if residual is not None else a.dtype)
    return _store(y, out, dt)


def gemm_gated(a, gate, rows_per_image, w, bias=None, act=None, residual=None):
    img = torch.arange(a.shape[0], device=a.device) // rows_per_image
    scaled = (a.to(_HP) * gate.to(_HP)[img]).to(a.dtype)          # the product is rounded to bf16 before the GEMM
    return gemm(scaled, w, bias=bias, act=act, residual=residual)


def mlp_fused_supported(C, hidden):
    return C in (96, 128, 192, 256) and hidden % 128 == 0 and hidden >= 256


def mlp_fused(a, w1, b1, w2, b2, act, gamma=None, residual=None, out=None):
    # the kernel's rounding points are those of the two-GEMM form: bf16 hidden activations, fp32 output
    hid = gemm(a, w1, bias=b1, act=act)
    return gemm(hid, w2, bias=b2, gamma=gamma, residual=residual, out=out, out_dtype=torch.float32)


def conv_gemm(x, w, bias=None, ks=3, stride=1, pad=1, act=None, residual=None, act_after_residual=False,
              out_dtype=None):
    B, H, W, C = x.shape
    N = w.shape[0]
    wt = w.to(_HP).view(N, ks, ks, C).permute(0, 3, 1, 2)
    y = F.conv2d(x.to(_HP).permute(0, 3, 1, 2), wt, None, stride=stride, padding=pad).permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias.to(_HP)
    if act_after_residual:
        if residual is not None:
            y = y + residual.to(_HP)
        y = _act(y, act)
    else:
        y = _act(y, act)
        if residual is not None:
            y = y + residual.to(_HP)
    return y.contiguous().to(out_dtype or (residual.dtype if residual is not None else x.dtype))


def _ln(x, gamma, beta, eps):
    x = x.to(_HP)
    mean = x.mean(dim=-1, keepdim=True)
    var = (x - mean).pow(2).mean(dim=-1, keepdim=True)
    return (x - mean) * torch.rsqrt(var + eps) * gamma.to(_HP) + beta.to(_HP)


def layernorm(x, gamma, beta, eps, out_dtype, out=None):
    return _store(_ln(x, gamma, beta, eps), out, out_dtype)


def layernorm_patch2x2(x, gamma, beta, eps, out_dtype):
    B, H, W, C = x.shape
    y = _ln(x, gamma, beta, eps)
    y = y.view(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * (H // 2) * (W // 2), 4 * C)
    return y.contiguous().to(out_dtype)


def patch_merge_ln(x, gamma, beta, eps, out_dtype):
    cat = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], dim=-1)
    return _ln(cat, gamma, beta, eps).reshape(-1, cat.shape[-1]).contiguous().to(out_dtype)


# Keys per block of the online softmax of the tensor-core attention kernels (csrc/attention.cu, pit.cu,
# relpos_attention.cu).
KEY_BLOCK = 64


def round_bf16(p):
    """P as a bf16 tensor-core operand sees it: rounded to nearest even, kept in p's dtype."""
    return p.to(torch.bfloat16).to(p.dtype)


def _softmax_pv(s, v, round_p=None, key_block=None):
    """softmax(s) @ v the way the tensor-core kernels do it: an online softmax over blocks of ``key_block`` keys from
    key 0 (None: the whole row in one block).  Per block, m = the largest score so far, p = exp(s - m), the row sum
    l = l exp(m_old - m) + sum p of the unrounded p, O = O exp(m_old - m) + round_p(p) V; O / l at the end.
    ``round_p``: the rounding of P for the PV product (``round_bf16``, TF32, or None).  Also returns the normalised
    (rounded) P when the row is one block, else None."""
    N = s.shape[-1]
    kb = N if key_block is None else key_block
    rnd = round_p if round_p is not None else (lambda p: p)
    m = s[..., :kb].amax(dim=-1, keepdim=True)
    p = torch.exp(s[..., :kb] - m)
    l = p.sum(dim=-1, keepdim=True)
    p = rnd(p)
    o = p @ v[..., :kb, :]
    for j0 in range(kb, N, kb):
        sb = s[..., j0:j0 + kb]
        m_new = torch.maximum(m, sb.amax(dim=-1, keepdim=True))
        alpha = torch.exp(m - m_new)
        pb = torch.exp(sb - m_new)
        l = l * alpha + pb.sum(dim=-1, keepdim=True)
        o = o * alpha + rnd(pb) @ v[..., j0:j0 + kb, :]
        m = m_new
    return o / l, (p / l if kb >= N else None)


def image_chunks(B, H, N, budget=2 ** 24):
    """Slices of the image axis whose (images, H, N, N) score tensors hold at most ``budget`` elements (at least one
    image each): the float64 statements and bounds of attention are computed chunk by chunk, so that a benchmark batch
    of ViT-B (256 x 12 x 197^2) does not hold its whole score tensor and its temporaries at once."""
    step = max(1, budget // (H * N * N))
    return [slice(b0, min(B, b0 + step)) for b0 in range(0, B, step)]


def attention(qkv, B, N, H, dh, scale, bias=None, mask=None, probs=None, row_map=None, nw_img=0, key_block=KEY_BLOCK):
    """bf16 qkv: P rounded to bf16 per block of ``key_block`` keys (the tensor-core kernels; the window kernels pass
    None: one block); fp32 qkv: the SIMT kernel's unrounded softmax over the whole row."""
    dt = qkv.dtype
    x = qkv
    if row_map is not None:  # Swin: rows of window w of image b live at row_map[w*N + i] of that image's tokens
        nimg = B // nw_img
        tok = nw_img * N
        idx = (torch.arange(nimg, device=x.device)[:, None] * tok + row_map.long()[None, :]).reshape(-1)
        x = x[idx]
    x = x.view(B, N, 3, H, dh)
    round_p = round_bf16 if dt == torch.bfloat16 else None
    kb = key_block if round_p is not None else None

    def chunk(c):
        """(scores, v) of the images (windows) of slice c, in float64"""
        q, k, v = x[c].to(_HP).permute(2, 0, 3, 1, 4)
        s = scale * (q @ k.transpose(-1, -2))
        if bias is not None:
            s = s + bias.to(_HP)[None]
        if mask is not None:   # image (window) b takes mask[b % nm]
            s = s + mask.to(_HP)[torch.arange(c.start, c.stop, device=s.device) % mask.shape[0]][:, None]
        return s, v

    if probs is None:
        o = torch.cat([_softmax_pv(*chunk(c), round_p, kb)[0] for c in image_chunks(B, H, N)])
    else:
        o, p = _softmax_pv(*chunk(slice(0, B)), round_p, kb)
        probs.copy_(p)
    o = o.permute(0, 2, 1, 3).reshape(B * N, H * dh)
    if row_map is not None:
        out = torch.empty_like(o)
        out[idx] = o
        o = out
    return o.contiguous().to(dt)


def attention_cls(qkv, B, T, H, dh, scale, nq=1):
    q, k, v = qkv.to(_HP).view(B, T, 3, H, dh).permute(2, 0, 3, 1, 4)
    s = scale * (q[:, :, :nq] @ k.transpose(-1, -2))
    o = torch.softmax(s, dim=-1) @ v  # SIMT kernel: fp32 throughout, one bf16 output rounding
    return o.permute(0, 2, 1, 3).reshape(B * nq, H * dh).contiguous().to(qkv.dtype)


def window_attention(qkv, bias, row_map, labels, B, nw_img, N, H, dh, scale):
    mask = None
    if labels is not None:
        lab = labels.view(nw_img, N)
        mask = torch.where(lab[:, None, :] != lab[:, :, None], -100.0, 0.0).to(_HP)
    return attention(qkv, B * nw_img, N, H, dh, scale, bias=bias, mask=mask, row_map=row_map, nw_img=nw_img,
                     key_block=None)   # the window kernels take the whole window in one pass


def window_attention_tc(qkv, bias_pad, row_map, maskbits, B, nw_img, N, H, dh, scale):
    mask = None
    if maskbits is not None:
        bits = (maskbits[:, :N, None] >> torch.arange(N, device=maskbits.device)[None, None, :]) & 1
        mask = torch.where(bits.bool(), -100.0, 0.0).to(_HP)
    return attention(qkv, B * nw_img, N, H, dh, scale, bias=bias_pad[:, :N, :N], mask=mask, row_map=row_map,
                     nw_img=nw_img, key_block=None)


def patchify(img, p, out_dtype, mean=None, inv_std=None, scale=1.0):
    B, H, W, C = img.shape
    x = img.to(_HP)
    if mean is not None:
        x = (x * scale - mean.to(_HP)) * inv_std.to(_HP)
    K = p * p * C
    y = x.view(B, H // p, p, W // p, p, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, K)
    Kpad = (K + 7) // 8 * 8
    if Kpad != K:
        y = F.pad(y, (0, Kpad - K))
    return y.contiguous().to(out_dtype)


def assemble_tokens(patches, cls, dist, pos, B, P, out_dtype):
    D = patches.shape[1]
    toks = [cls.to(_HP).view(1, 1, D).expand(B, 1, D)]
    if dist is not None:
        toks.append(dist.to(_HP).view(1, 1, D).expand(B, 1, D))
    y = torch.cat(toks + [patches.to(_HP).view(B, P, D)], dim=1) + pos.to(_HP)[None]
    return y.reshape(-1, D).contiguous().to(out_dtype)


def cast(x, dtype):
    return x if x.dtype == dtype else x.contiguous().to(dtype)


def _dw(x, wgt, bias, ks, stride, pads):
    C = x.shape[-1]
    wt = wgt.to(_HP).view(ks, ks, C).permute(2, 0, 1)[:, None]
    xin = F.pad(x.to(_HP).permute(0, 3, 1, 2), pads)
    return F.conv2d(xin, wt, bias.to(_HP) if bias is not None else None, stride=stride, groups=C).permute(0, 2, 3, 1)


def dwconv_ln(x, wgt, bias, gamma, beta, eps, out_dtype):
    C = x.shape[-1]
    ks = int(round(wgt.shape[0] ** 0.5))
    y = _dw(x, wgt, bias, ks, 1, (ks // 2,) * 4)
    return _ln(y, gamma, beta, eps).reshape(-1, C).contiguous().to(out_dtype)


def same_pad(size, k, s):
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return out, total // 2


def conv_geometry(H, W, ks, stride, padding):
    if padding == "same":
        Ho, pt = same_pad(H, ks, stride)
        Wo, pl = same_pad(W, ks, stride)
        return Ho, Wo, pt, pl
    if padding == "symmetric":
        pd = ((stride - 1) + (ks - 1)) // 2
    elif padding == "valid":
        pd = 0
    else:
        pd = int(padding)
    return (H + 2 * pd - ks) // stride + 1, (W + 2 * pd - ks) // stride + 1, pd, pd


def _pads(H, W, ks, stride, padding):
    Ho, Wo, pt, pl = conv_geometry(H, W, ks, stride, padding)
    pb = max((Ho - 1) * stride + ks - H - pt, 0)
    pr = max((Wo - 1) * stride + ks - W - pl, 0)
    return Ho, Wo, (pl, pr, pt, pb)


def dwconv_bias_act(x, wgt, bias, ks, stride, padding, act=None, pool_sum=None):
    B, H, W, C = x.shape
    _, _, pads = _pads(H, W, ks, stride, padding)
    y = _act(_dw(x, wgt, bias, ks, stride, pads), act).contiguous().to(x.dtype)
    if pool_sum is not None:
        pool_sum.add_(y.to(_HP).sum(dim=(1, 2)).to(pool_sum.dtype))  # the squeeze sees what the next layer reads
    return y


def global_avg_pool(x):
    B, C = x.shape[0], x.shape[-1]
    return x.to(_HP).reshape(B, -1, C).mean(dim=1)


def im2col(x, ks, stride, padding, out_dtype, groups=1, pre=None):
    B, H, W, C = x.shape
    Ho, Wo, pads = _pads(H, W, ks, stride, padding)
    xh = x.to(_HP)
    if pre is not None:   # raw pixels: create_preprocessing before the (zero) padding
        mean, inv_std, scale = pre
        xh = (xh * scale - mean.to(_HP)) * inv_std.to(_HP)
    xin = F.pad(xh.permute(0, 3, 1, 2), pads)
    cols = F.unfold(xin, ks, stride=stride)  # (B, C*ks*ks, L), rows ordered (c, ky, kx)
    cols = cols.view(B, C, ks * ks, Ho * Wo).permute(0, 3, 2, 1)  # (B, L, (ky,kx), c)
    cg = C // groups
    K = ks * ks * cg
    Kpad = (K + 7) // 8 * 8
    if groups == 1:
        out = cols.reshape(B * Ho * Wo, K)
    else:
        out = cols.reshape(B * Ho * Wo, ks * ks, groups, cg).permute(2, 0, 1, 3).reshape(groups, B * Ho * Wo, K)
    if Kpad != K:
        out = F.pad(out, (0, Kpad - K))
    return out.contiguous().to(out_dtype), Ho, Wo


def group_norm(x, gamma, beta, groups, eps, act=None, residual=None):
    y = F.group_norm(x.to(_HP).permute(0, 3, 1, 2), groups, gamma.to(_HP), beta.to(_HP), eps).permute(0, 2, 3, 1)
    if residual is not None:
        y = y + residual.to(_HP)
    return _act(y, act).contiguous().to(x.dtype)


def blur_pool(x, stride=2):
    C = x.shape[-1]
    xc = F.pad(x.to(_HP).permute(0, 3, 1, 2), (1, 1, 1, 1), mode="reflect")
    k1 = torch.tensor([1.0, 2.0, 1.0], device=x.device, dtype=_HP)
    k = (k1[:, None] * k1[None, :] / 16)[None, None].repeat(C, 1, 1, 1)
    return F.conv2d(xc, k, stride=stride, groups=C).permute(0, 2, 3, 1).contiguous().to(x.dtype)


def se_gate(pooled_sum, hw, w_reduce, b_reduce, w_expand, b_expand, act, gate_act="sigmoid"):
    m = pooled_sum.to(_HP) / float(hw)
    h = _act(m @ w_reduce.to(_HP).t() + b_reduce.to(_HP), act)
    return _act(h @ w_expand.to(_HP) + b_expand.to(_HP), gate_act)


def scale_channels_(x, gate):
    B, C = gate.shape
    y = x.to(_HP).view(B, -1, C) * gate.to(_HP)[:, None, :]
    x.copy_(y.view(x.shape).to(x.dtype))
    return x


def pool2d(x, ks, stride, padding, mode):
    B, H, W, C = x.shape
    _, _, pads = _pads(H, W, ks, stride, padding)
    xin = x.to(_HP).permute(0, 3, 1, 2)
    if mode == "avg":
        num = F.avg_pool2d(F.pad(xin, pads), ks, stride, divisor_override=1)
        cnt = F.avg_pool2d(F.pad(torch.ones_like(xin[:, :1]), pads), ks, stride, divisor_override=1)
        y = num / cnt
    elif mode == "max_zero_pad":
        y = F.max_pool2d(F.pad(xin, pads), ks, stride)
    else:
        y = F.max_pool2d(F.pad(xin, pads, value=float("-inf")), ks, stride)
    return y.permute(0, 2, 3, 1).contiguous().to(x.dtype)


def grouped_conv(x, wgt, bias, cg, ks, stride, pad, act=None):
    C = x.shape[-1]
    w = wgt.to(_HP).view(ks, ks, cg, C).permute(3, 2, 0, 1)
    y = F.conv2d(x.to(_HP).permute(0, 3, 1, 2), w, bias.to(_HP) if bias is not None else None, stride=stride,
                 padding=pad, groups=C // cg).permute(0, 2, 3, 1)
    return _act(y, act).contiguous().to(x.dtype)


def eca_gate(mean, w):
    k = w.numel()
    y = F.conv1d(F.pad(mean.to(_HP), (k // 2, k // 2))[:, None], w.to(_HP)[None, None])[:, 0]
    return torch.sigmoid(y)


def scale_add_act_(x, gate, shortcut, act):
    B, C = gate.shape
    y = x.to(_HP).view(B, -1, C) * gate.to(_HP)[:, None, :] + shortcut.to(_HP).view(B, -1, C)
    x.copy_(_act(y, act).view(x.shape).to(x.dtype))
    return x


_EMULATED = ("gemm", "gemm_gated", "mlp_fused", "mlp_fused_supported", "conv_gemm", "layernorm", "layernorm_patch2x2", "patch_merge_ln", "attention", "attention_cls",
             "window_attention", "window_attention_tc", "patchify", "assemble_tokens", "cast", "dwconv_ln", "dwconv_bias_act",
             "global_avg_pool", "im2col", "group_norm", "blur_pool", "se_gate", "scale_channels_", "pool2d",
             "grouped_conv", "eca_gate", "scale_add_act_")


@contextmanager
def emulated_ops(arithmetic=torch.float64):
    """Inside the block every ``tfimm.backend.ops`` launcher is the exact-arithmetic torch version above.
    ``arithmetic=torch.float32`` evaluates the same graph with the same bf16 storage points in plain fp32: a second,
    equally legitimate "ideal" bf16 implementation whose distance from the float64 one is the DIVERGENCE FLOOR of
    bf16 storage (rounding decisions of ~2 % of the stored elements flip on a 1e-7 perturbation and cascade)."""
    from tfimm.backend import ops

    global _HP
    saved_hp, _HP = _HP, arithmetic

    missing = [n for n in dir(ops) if callable(getattr(ops, n)) and not n.startswith("_") and n not in _EMULATED
               and n not in ("act_code", "same_pad", "conv_geometry", "attention_bf16_supported", "Optional") and
               getattr(getattr(ops, n), "__module__", "") == ops.__name__]
    if missing:
        raise RuntimeError(f"oracle/emulate_bf16.py has no emulation for ops.{missing}")
    saved = {n: getattr(ops, n) for n in _EMULATED}
    for n in _EMULATED:
        setattr(ops, n, globals()[n])
    try:
        with torch.no_grad():
            yield
    finally:
        _HP = saved_hp
        for n, f in saved.items():
            setattr(ops, n, f)
