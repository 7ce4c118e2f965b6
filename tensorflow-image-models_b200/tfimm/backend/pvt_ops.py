"""Launchers of the PVT family's kernels (``csrc/pvt.cu``, C ABI in ``include/tfimm_b200_pvt.h``).

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.  ``lib.load()`` types their entry points with all the others.
"""
import torch

from . import lib as _lib
from . import ops as _ops

HEAD_DIM = 64


def sr_attention_nbytes(B, N, Nk, H, dh, itemsize):
    """HBM bytes of spatial-reduction attention: q read and out written once, k and v read once."""
    return float(itemsize) * B * H * dh * (2 * N + 2 * Nk)


def _sr_attention(name, dtype, q, kv, B, N, Nk, H, dh, scale):
    dev = _ops._cuda(q, kv)
    assert q.dtype == kv.dtype == dtype and q.is_contiguous() and kv.is_contiguous(), (q.dtype, kv.dtype)
    assert q.shape == (B * N, H * dh) and kv.shape == (B * Nk, 2 * H * dh), (q.shape, kv.shape, (B, N, Nk, H, dh))
    out = torch.empty((B * N, H * dh), device=q.device, dtype=dtype)
    _ops._call(name, dev, q.data_ptr(), kv.data_ptr(), out.data_ptr(), B, N, Nk, H, dh, float(scale),
               flops=4.0 * B * H * N * Nk * dh, nbytes=sr_attention_nbytes(B, N, Nk, H, dh, q.element_size()))
    return out


def pvt_sr_attention_bf16(q, kv, B, N, Nk, H, dh, scale):
    """softmax(scale q k^T) v with queries from q (B * N, H * dh) and keys / values from kv (B * Nk, 2 * H * dh), read
    as (B, Nk, 2, H, dh); bf16 in and out, dh 64, tensor cores."""
    return _sr_attention("tfimm_b200_pvt_sr_attention_bf16", torch.bfloat16, q, kv, B, N, Nk, H, dh, scale)


def pvt_sr_attention_f32(q, kv, B, N, Nk, H, dh, scale):
    """The same on fp32 q / kv, with an fp32 softmax on the CUDA cores."""
    return _sr_attention("tfimm_b200_pvt_sr_attention_f32", torch.float32, q, kv, B, N, Nk, H, dh, scale)


def sr_attention(q, kv, B, N, Nk, H, dh, scale):
    """Spatial-reduction attention in the precision of ``q``: bf16 -> the tensor-core kernel; fp32 (the fp32 and tf32
    precisions) -> the fp32 kernel."""
    if dh != HEAD_DIM:
        raise _lib.KernelLibraryError(f"PVT attention: no kernel for head_dim {dh} (have {HEAD_DIM})")
    if q.dtype == torch.bfloat16:
        return pvt_sr_attention_bf16(q, kv, B, N, Nk, H, dh, scale)
    return pvt_sr_attention_f32(q, kv, B, N, Nk, H, dh, scale)


def embed_norm_nbytes(B, P, ntok, C):
    """HBM bytes of pvt_embed_norm: tok read, the stream written, the position table, gamma, beta and cls."""
    return 4.0 * (B * P * C + B * (P + ntok) * C + (P + ntok) * C + 3 * C)


def pvt_embed_norm(tok, gamma, beta, pos, cls, B, P, eps):
    """The fp32 residual stream (B * (ntok + P), C) of a stage: LayerNorm_eps(tok) * gamma + beta + pos[ntok:] for the
    patch rows and, when ``cls`` is given (ntok = 1), cls + pos[0] for row 0 of every image.  tok: fp32 (B * P, C);
    pos: fp32 (ntok + P, C)."""
    ntok = 0 if cls is None else 1
    dev = _ops._cuda(tok, gamma, beta, pos, cls)
    C = tok.shape[1]
    assert tok.dtype == torch.float32 and tok.is_contiguous() and tok.shape == (B * P, C), (tok.dtype, tok.shape)
    assert pos.dtype == torch.float32 and pos.is_contiguous() and pos.shape == (ntok + P, C), (pos.shape, (P, C))
    for v in (gamma, beta) if cls is None else (gamma, beta, cls):
        assert v.dtype == torch.float32 and v.is_contiguous() and v.shape == (C,), (v.dtype, v.shape, C)
    out = torch.empty((B * (ntok + P), C), device=tok.device, dtype=torch.float32)
    _ops._call("tfimm_b200_pvt_embed_norm", dev, tok.data_ptr(), gamma.data_ptr(), beta.data_ptr(), pos.data_ptr(),
               _ops._ptr(cls), out.data_ptr(), B, P, ntok, C, float(eps), flops=9.0 * B * (P + ntok) * C,
               nbytes=embed_norm_nbytes(B, P, ntok, C))
    return out
