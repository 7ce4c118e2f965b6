"""Launchers of the PoolFormer family's kernels (``csrc/poolformer.cu``, C ABI in ``include/tfimm_b200_poolformer.h``).

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.  ``lib.load()`` types their entry points with all the others.

A one-group GroupNorm's statistics travel as partials, fp32 (B, splits(H, W, C), 3) = (count, mean, M2) per chunk of
``CHUNK`` values of an image (see the header).
"""
import torch

from . import ops as _ops

# values per chunk (csrc/poolformer.cu kChunk); the entry points refuse any other chunking
CHUNK = 4096


def splits(H, W, C):
    return (H * W * C + CHUNK - 1) // CHUNK


def _check_stream(x):
    B, H, W, C = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous() and C % 4 == 0, (x.dtype, x.shape, x.stride())
    return B, H, W, C


def _check_partials(partials, B, H, W, C):
    assert partials.dtype == torch.float32 and partials.is_contiguous(), (partials.dtype, partials.stride())
    assert partials.shape == (B, splits(H, W, C), 3), (partials.shape, (B, H, W, C))


def gn1_partials(x):
    """x: (B, H, W, C) fp32 -> its partials (B, splits, 3)."""
    dev = _ops._cuda(x)
    B, H, W, C = _check_stream(x)
    S = splits(H, W, C)
    partials = torch.empty((B, S, 3), device=x.device, dtype=torch.float32)
    _ops._call("tfimm_b200_gn1_partials", dev, x.data_ptr(), partials.data_ptr(), B, H, W, C, S,
               nbytes=_ops._nbytes(x, partials))
    return partials


def mixer_nbytes(B, H, W, C):
    """HBM bytes the token mixer needs: one read of x, one write of out, the partials read and written.  A CTA's halo
    (the pixel rows above and below its chunk) is the chunk of the CTAs beside it, read at the same time, so it comes
    from L1 / L2: counted as HBM traffic it would put the measured rate above the HBM bandwidth
    (profiles/poolformer_h100.md)."""
    N, S = H * W * C, splits(H, W, C)
    return 4.0 * B * (2 * N + 2 * 3 * S)


def apply_nbytes(B, H, W, C, out_dtype):
    """HBM bytes of gn1_apply: one read of x, one write of the output, the partials."""
    N, S = H * W * C, splits(H, W, C)
    return B * (4.0 * N + torch.finfo(out_dtype).bits / 8 * N + 4.0 * 3 * S)


def poolformer_mixer(x, partials, gamma, beta, ls1, eps):
    """x + ls1 * (AvgPool3x3_same(GN(x)) - GN(x)) of the fp32 stream x (B, H, W, C), GN from x's ``partials`` ->
    (out (B, H, W, C) fp32, out's partials).  beta cancels in this form (csrc/poolformer.cu), so only the statement
    the tests check the kernel against reads it."""
    dev = _ops._cuda(x, partials, gamma, beta, ls1)
    B, H, W, C = _check_stream(x)
    _check_partials(partials, B, H, W, C)
    for v in (gamma, beta, ls1):
        assert v.dtype == torch.float32 and v.shape == (C,) and v.is_contiguous()
    out = torch.empty_like(x)
    out_partials = torch.empty_like(partials)
    _ops._call("tfimm_b200_poolformer_mixer", dev, x.data_ptr(), partials.data_ptr(), gamma.data_ptr(), ls1.data_ptr(),
               out.data_ptr(), out_partials.data_ptr(), B, H, W, C, partials.shape[1], float(eps),
               nbytes=mixer_nbytes(B, H, W, C))
    return out, out_partials


def gn1_apply(x, partials, gamma, beta, eps, out_dtype):
    """GN(x) from x's ``partials``: x (B, H, W, C) fp32 -> (B * H * W, C) in out_dtype (bf16 or fp32)."""
    dev = _ops._cuda(x, partials, gamma, beta)
    B, H, W, C = _check_stream(x)
    _check_partials(partials, B, H, W, C)
    for v in (gamma, beta):
        assert v.dtype == torch.float32 and v.shape == (C,) and v.is_contiguous()
    out = torch.empty((B * H * W, C), device=x.device, dtype=out_dtype)
    _ops._call("tfimm_b200_gn1_apply", dev, x.data_ptr(), partials.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
               out.data_ptr(), _ops._code(out), B, H, W, C, partials.shape[1], float(eps),
               nbytes=apply_nbytes(B, H, W, C, out_dtype))
    return out
