"""Launcher of the ConvMixer family's kernel (``csrc/convmixer.cu``, C ABI in ``include/tfimm_b200_convmixer.h``).

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.  ``lib.load()`` types its entry point with all the others.
"""
import torch

from . import ops as _ops

# what the kernel takes (csrc/convmixer.cu): the entry point refuses anything else with TFIMM_ERR_UNSUPPORTED
KERNEL_SIZES = (7, 9)
CHANNEL_MULTIPLE = 32


def supported(C, k) -> bool:
    return k in KERNEL_SIZES and C > 0 and C % CHANNEL_MULTIPLE == 0


def dwconv_nbytes(B, H, W, C, k, out_dtype):
    """HBM bytes the kernel must move: one read of a, one write of y, the taps and the five per-channel vectors.  The
    halo a tile reads beyond its own cells belongs to the tiles beside it and comes from L2."""
    return B * H * W * C * (4.0 + torch.finfo(out_dtype).bits / 8) + 4.0 * C * (k * k + 5)


def dwconv(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
    """ConvMixer's token mixer with the previous BatchNorm folded in, on the fp32 activation a (B, H, W, C):
    x = s_in a + t_in inside the image (0 in the "same" padding), y = x + s1 act(depthwise_k(x) + bias) + t1 -> y
    (B, H, W, C) in out_dtype (bf16 or fp32).  taps: fp32 (k * k, C), the reference's depthwise_kernel (k, k, C, 1)."""
    dev = _ops._cuda(a, s_in, t_in, taps, bias, s1, t1)
    B, H, W, C = a.shape
    assert a.dtype == torch.float32 and a.is_contiguous(), (a.dtype, a.stride())
    k = int(round(taps.shape[0] ** 0.5))
    assert taps.dtype == torch.float32 and taps.is_contiguous() and taps.shape == (k * k, C), (taps.dtype, taps.shape)
    for v in (s_in, t_in, bias, s1, t1):
        assert v.dtype == torch.float32 and v.shape == (C,) and v.is_contiguous(), (v.dtype, v.shape)
    assert out_dtype in (torch.bfloat16, torch.float32), out_dtype
    if not supported(C, k):
        raise ValueError(f"convmixer_dwconv takes kernel sizes {KERNEL_SIZES} and C % {CHANNEL_MULTIPLE} == 0 "
                         f"(got k={k}, C={C})")
    y = torch.empty((B, H, W, C), device=a.device, dtype=out_dtype)
    _ops._call("tfimm_b200_convmixer_dwconv", dev, a.data_ptr(), s_in.data_ptr(), t_in.data_ptr(), taps.data_ptr(),
               bias.data_ptr(), s1.data_ptr(), t1.data_ptr(), y.data_ptr(), _ops._code(y), B, H, W, C, k,
               _ops.act_code(act), flops=2.0 * B * H * W * C * k * k, nbytes=dwconv_nbytes(B, H, W, C, k, out_dtype))
    return y
