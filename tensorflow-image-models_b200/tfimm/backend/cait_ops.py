"""Launchers of the CaiT family's kernels (``csrc/cait.cu``, C ABI in ``include/tfimm_b200_cait.h``), and CaiT's
attention dispatch.

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.  ``lib.load()`` types their entry points with all the others.
"""
import math

import torch

from . import lib as _lib
from . import ops as _ops

# (H, dh) of the bf16 talking-heads kernel's instantiations: every registered CaiT
BF16_HEADS = (4, 6, 8, 16)
BF16_HEAD_DIM = 48
# the fp32 kernel's range
F32_HEADS = (1, 2, 3, 4, 6, 8, 12, 16)
# head dims of the class-attention kernel
CLS_HEAD_DIMS = (32, 48, 64)

LOG2E = math.log2(math.e)


def f32_supported(H, dh):
    return H in F32_HEADS and 0 < dh <= 64 and dh % 4 == 0


def bf16_supported(H, dh):
    return H in BF16_HEADS and dh == BF16_HEAD_DIM


def fold_premix(wl, bl, dh):
    """The pre-softmax mix in the kernels' log2 units: ``proj_l``'s (H, H) kernel times dh^-0.5 log2 e, its bias times
    log2 e.  The scale multiplies q before the logits are mixed, so it reaches the kernel and not the bias."""
    return ((wl.double() * (dh ** -0.5 * LOG2E)).float().contiguous(), (bl.double() * LOG2E).float().contiguous())


def talking_heads_flops(B, N, H, dh):
    """Per launch: q k^T twice (two passes) and P' V once, 2 FMA-flops each, plus both H x H mixes twice per pair on
    the pre-mix pass and once after."""
    return 2.0 * B * N * N * (3 * H * dh + 3 * H * H)


def talking_heads_nbytes(qkv, out, H):
    return _ops._nbytes(qkv, out) + 4.0 * (2 * H * H + 2 * H)


def _check_mix(wl, bl, ww, bw, H):
    for t in (wl, bl, ww, bw):
        assert t.dtype == torch.float32 and t.is_contiguous(), (t.dtype, t.shape)
    assert wl.shape == ww.shape == (H, H) and bl.shape == bw.shape == (H,), (wl.shape, bl.shape, ww.shape, bw.shape)


def talking_heads_bf16(qkv, wl, bl, ww, bw, B, N, H, dh):
    """Talking-heads attention from the packed bf16 qkv (B * N, 3 * H * dh) -> (B * N, H * dh) bf16.  wl / bl: the
    pre-mix in log2 units (``fold_premix``), ww / bw: the post-mix, all fp32.  dh 48, H in ``BF16_HEADS``, any N."""
    dev = _ops._cuda(qkv, wl, bl, ww, bw)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (B * N, 3 * H * dh), \
        (qkv.dtype, qkv.shape, (B, N, H, dh))
    _check_mix(wl, bl, ww, bw, H)
    out = torch.empty((B * N, H * dh), device=qkv.device, dtype=torch.bfloat16)
    _ops._call("tfimm_b200_cait_talking_heads_bf16", dev, qkv.data_ptr(), out.data_ptr(), wl.data_ptr(), bl.data_ptr(),
               ww.data_ptr(), bw.data_ptr(), B, N, H, dh, flops=talking_heads_flops(B, N, H, dh),
               nbytes=talking_heads_nbytes(qkv, out, H))
    return out


def talking_heads_f32(qkv, wl, bl, ww, bw, B, N, H, dh):
    """The same from fp32 qkv into fp32 out, on the CUDA cores; H in ``F32_HEADS``, dh % 4 == 0 up to 64."""
    dev = _ops._cuda(qkv, wl, bl, ww, bw)
    assert qkv.dtype == torch.float32 and qkv.is_contiguous() and qkv.shape == (B * N, 3 * H * dh), \
        (qkv.dtype, qkv.shape, (B, N, H, dh))
    _check_mix(wl, bl, ww, bw, H)
    out = torch.empty((B * N, H * dh), device=qkv.device, dtype=torch.float32)
    _ops._call("tfimm_b200_cait_talking_heads_f32", dev, qkv.data_ptr(), out.data_ptr(), wl.data_ptr(), bl.data_ptr(),
               ww.data_ptr(), bw.data_ptr(), B, N, H, dh, flops=talking_heads_flops(B, N, H, dh),
               nbytes=talking_heads_nbytes(qkv, out, H))
    return out


def class_attention(q, kv, B, T, H, dh, scale):
    """softmax(scale q k^T) v with one query per (image, head): q (B, H * dh), kv (B * T, 2 * H * dh) = [k | v] of all
    T rows, -> (B, H * dh) in the dtype of q (bf16 or fp32).  Any T; dh in ``CLS_HEAD_DIMS``."""
    dev = _ops._cuda(q, kv)
    D = H * dh
    assert q.dtype == kv.dtype and q.shape == (B, D) and q.stride(1) == 1 and q.stride(0) == D, (q.shape, q.stride())
    assert kv.is_contiguous() and kv.shape == (B * T, 2 * D), (kv.shape, (B, T, D))
    out = torch.empty((B, D), device=q.device, dtype=q.dtype)
    _ops._call("tfimm_b200_cait_class_attention", dev, q.data_ptr(), kv.data_ptr(), out.data_ptr(), _ops._code(q), B, T,
               H, dh, float(scale), flops=4.0 * B * T * D, nbytes=_ops._nbytes(q, kv, out))
    return out


def add_pos(x, pos, B, N):
    """x (B * N, D) fp32 += pos (N, D) fp32 for every image, in place; returns x."""
    dev = _ops._cuda(x, pos)
    D = x.shape[1]
    assert x.dtype == pos.dtype == torch.float32 and x.is_contiguous() and pos.is_contiguous(), (x.dtype, pos.dtype)
    assert x.shape == (B * N, D) and pos.shape == (N, D), (x.shape, pos.shape, (B, N))
    _ops._call("tfimm_b200_cait_add_pos", dev, x.data_ptr(), pos.data_ptr(), B, N, D, flops=float(B * N * D),
               nbytes=4.0 * (2 * B * N * D + N * D))
    return x


def talking_heads(qkv, wl, bl, ww, bw, B, N, H, dh):
    """CaiT self-attention in the precision of ``qkv``: bf16 -> talking_heads_bf16; fp32 (fp32 and tf32 models) ->
    talking_heads_f32.  A shape without a kernel is refused."""
    if qkv.dtype == torch.bfloat16:
        if not bf16_supported(H, dh):
            raise _lib.KernelLibraryError(f"CaiT talking-heads attention: no bf16 kernel for H={H}, head_dim {dh} "
                                          f"(have H in {BF16_HEADS} at head_dim {BF16_HEAD_DIM})")
        return talking_heads_bf16(qkv, wl, bl, ww, bw, B, N, H, dh)
    if not f32_supported(H, dh):
        raise _lib.KernelLibraryError(f"CaiT talking-heads attention: no fp32 kernel for H={H}, head_dim {dh}")
    return talking_heads_f32(qkv, wl, bl, ww, bw, B, N, H, dh)
