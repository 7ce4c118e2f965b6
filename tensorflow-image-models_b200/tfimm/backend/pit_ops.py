"""Launchers of the PiT family's kernels (``csrc/pit.cu``, C ABI in ``include/tfimm_b200_pit.h``), and PiT's attention
dispatch.

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.  ``lib.load()`` types their entry points with all the others.
"""
import torch

from . import lib as _lib
from . import ops as _ops

HEAD_DIMS = (32, 48, 64)


def pool_geometry(H, W):
    """Output grid of ZeroPadding2D(1) + a 3 x 3 / 2 VALID convolution."""
    return (H - 1) // 2 + 1, (W - 1) // 2 + 1


def pit_attention_bf16(qkv, B, T, H, dh, scale):
    """softmax(scale q k^T) v from the packed bf16 qkv (B * T, 3 * H * dh) -> (B * T, H * dh) bf16; any T, dh 32 / 48 /
    64, K and V streamed in 64-key blocks."""
    dev = _ops._cuda(qkv)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (B * T, 3 * H * dh), \
        (qkv.dtype, qkv.shape, (B, T, H, dh))
    out = torch.empty((B * T, H * dh), device=qkv.device, dtype=torch.bfloat16)
    _ops._call("tfimm_b200_pit_attention_bf16", dev, qkv.data_ptr(), out.data_ptr(), B, T, H, dh, float(scale),
               flops=4.0 * B * H * T * T * dh, nbytes=_ops._nbytes(qkv, out))
    return out


def pool_nbytes(B, nb_tokens, H, W, C, tokens_bf16):
    """HBM bytes of pit_pool: one read of the grid rows, one write of the new grid rows, the weights and biases, and the
    token rows read and written in bf16 when asked."""
    Ho, Wo = pool_geometry(H, W)
    tok = B * nb_tokens * C * (4.0 + 2.0) if tokens_bf16 else 0.0
    return 4.0 * (B * H * W * C + B * Ho * Wo * 2 * C + 10 * 2 * C) + tok


def pit_pool(x, w, bias, B, nb_tokens, H, W, tokens_bf16=False):
    """The spatial half of PiT's pooling layer.  x: the fp32 stream (B * (nb_tokens + H * W), C); w: fp32 (9, 2C), the
    (3, 3, 1, 2C) grouped kernel's taps; bias: fp32 (2C).  Returns (out, tokens): out (B * (nb_tokens + Ho * Wo), 2C)
    fp32 with its grid rows written (output channel o reads input channel o // 2) and its token rows left for the
    token Dense; tokens the bf16 (B * nb_tokens, C) copy of x's token rows when ``tokens_bf16``, else None."""
    dev = _ops._cuda(x, w, bias)
    C = x.shape[1]
    assert x.dtype == torch.float32 and x.is_contiguous() and x.shape == (B * (nb_tokens + H * W), C), \
        (x.dtype, x.shape, (B, nb_tokens, H, W))
    assert w.dtype == bias.dtype == torch.float32 and w.is_contiguous() and bias.is_contiguous()
    assert w.shape == (9, 2 * C) and bias.shape == (2 * C,), (w.shape, bias.shape, C)
    Ho, Wo = pool_geometry(H, W)
    out = torch.empty((B * (nb_tokens + Ho * Wo), 2 * C), device=x.device, dtype=torch.float32)
    tokens = torch.empty((B * nb_tokens, C), device=x.device, dtype=torch.bfloat16) if tokens_bf16 else None
    _ops._call("tfimm_b200_pit_pool", dev, x.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(),
               _ops._ptr(tokens), B, nb_tokens, H, W, C, flops=2.0 * 9 * B * Ho * Wo * 2 * C,
               nbytes=pool_nbytes(B, nb_tokens, H, W, C, tokens_bf16))
    return out, tokens


def vit_kernel_preferred(T, dh):
    """bf16 shapes where the ViT kernel (``ops.attention``: K / V resident in shared memory, 128-query tiles up to
    T = 128) was faster than pit_attention_bf16 on the H100 (profiles/pit_h100.md): at T = 65 (pit_b's stage 2) it was;
    at 129 and 257 (pit_b's stage 1) the new kernel was, and at 197 they tied.  Both kernels compute the same algorithm;
    only the time differs."""
    return dh == 64 and T <= 128


def attention(qkv, B, T, H, dh, scale):
    """PiT self-attention in the precision of ``qkv``: bf16 -> pit_attention_bf16 (or the ViT kernel where
    ``vit_kernel_preferred``); fp32 -> ``ops.attention``, i.e. the TF32 kernel at dh 64 in a tf32 model's forward and
    the fp32 SIMT kernel otherwise."""
    if qkv.dtype == torch.bfloat16:
        if dh not in HEAD_DIMS:
            raise _lib.KernelLibraryError(f"PiT attention: no bf16 kernel for head_dim {dh} (have {HEAD_DIMS})")
        if _ops.attention_bf16_supported(T, dh) and vit_kernel_preferred(T, dh):
            return _ops.attention(qkv, B, T, H, dh, scale)
        return pit_attention_bf16(qkv, B, T, H, dh, scale)
    return _ops.attention(qkv, B, T, H, dh, scale)
