"""Launchers of the Segment Anything image-encoder kernels (``csrc/relpos_attention.cu``).

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.
"""
import torch

from . import lib as _lib
from . import ops as _ops


def relpos_attention_bf16_supported(dh, sh, sw) -> bool:
    """Shapes the bf16 tensor-core kernel takes (csrc/relpos_attention.cu): head_dim 64 or 80, and a sequence extent
    S_h x S_w whose K / V ring plus per-warp [S_h | S_w] tables fit its 113 KB of shared memory (two CTAs per SM):
    S_h + S_w <= 153 at head_dim 64, <= 137 at 80 -- global blocks up to a 76 x 76 / 68 x 68 token grid."""
    if dh not in (64, 80):
        return False
    rs = max(sh + sw, (dh + 8) // 2) | 1
    return 2 * 2 * 64 * (dh + 8) * 2 + 8 * 16 * rs * 4 <= 113 * 1024


def relpos_attention(qkv, B, gh, gw, H, dh, scale, rel_h, rel_w, window=0, pad_bias=None):
    """Self-attention with decomposed relative-position terms over the packed qkv (B*gh*gw, 3*H*dh) of a gh x gw token
    grid -> (B*gh*gw, H*dh).  window == 0: global; window > 0: window x window windows of the grid padded to a multiple
    of the window, whose padding positions are keys with k / v from ``pad_bias`` (the qkv bias, (3*H*dh,), same dtype
    as qkv; None: zero keys).  rel_h / rel_w: fp32 (2*S - 1, dh) tables of the sequence extent S (window, or gh / gw).
    bf16 qkv: tensor-core kernel (head_dim 64 / 80); fp32 qkv: SIMT kernel."""
    dev = _ops._cuda(qkv, rel_h, rel_w, pad_bias)
    N = gh * gw
    sh, sw = (window, window) if window else (gh, gw)
    assert qkv.shape == (B * N, 3 * H * dh) and qkv.is_contiguous(), (qkv.shape, B, N, H, dh)
    assert rel_h.shape == (2 * sh - 1, dh) and rel_w.shape == (2 * sw - 1, dh), (rel_h.shape, rel_w.shape, sh, sw)
    assert rel_h.dtype == rel_w.dtype == torch.float32 and rel_h.is_contiguous() and rel_w.is_contiguous()
    if pad_bias is not None:
        assert pad_bias.shape == (3 * H * dh,) and pad_bias.dtype == qkv.dtype and pad_bias.is_contiguous()
    out = torch.empty((B * N, H * dh), device=qkv.device, dtype=qkv.dtype)
    nseq = (-(-gh // sh)) * (-(-gw // sw))
    flops = 4.0 * B * nseq * H * (sh * sw) ** 2 * dh
    args = (qkv.data_ptr(), out.data_ptr(), _ops._ptr(pad_bias), rel_h.data_ptr(), rel_w.data_ptr(), B, gh, gw, H, dh,
            int(window), float(scale))
    if qkv.dtype == torch.bfloat16:
        _ops._call("tfimm_b200_relpos_attention_bf16", dev, *args, flops=flops, nbytes=_ops._nbytes(qkv, out))
    elif qkv.dtype == torch.float32:
        _ops._call("tfimm_b200_relpos_attention_f32", dev, *args, flops=flops, nbytes=_ops._nbytes(qkv, out))
    else:
        raise _lib.KernelLibraryError(f"relpos_attention: unsupported dtype {qkv.dtype}")
    return out
