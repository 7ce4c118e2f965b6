"""Launchers of the PVT v2 family's kernels (``csrc/pvt_v2.cu``, C ABI in ``include/tfimm_b200_pvt_v2.h``).

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.  ``lib.load()`` types their entry points with all the others.
"""
import torch

from . import lib as _lib
from . import ops as _ops
from . import pvt_ops as _pvt_ops

HEAD_DIMS = (32, 64)            # 32: the kernels here; 64: pvt_ops' (PVT v1's)
CONV_MLP_CHANNELS = (32, 64, 128)
CONV_MLP_HIDDEN_STEP = 64
# The channel counts at which the model dispatches the fused kernel.  At C = 128 (stage 1 of b1-b5) it is slower than
# the three unfused launches on an H100 (profiles/pvt_v2_h100.md: one CTA per SM at 142 registers), so those blocks run
# the unfused chain.
CONV_MLP_FUSED_CHANNELS = (32, 64)


# ------------------------------------------------------------------------------------------------------ ConvFFN
def conv_mlp_supported(C, hidden):
    """Shapes the fused ConvFFN kernel takes."""
    return C in CONV_MLP_CHANNELS and hidden > 0 and hidden % CONV_MLP_HIDDEN_STEP == 0


def conv_mlp_nbytes(B, gh, gw, C, hidden):
    """HBM bytes of the fused ConvFFN: h read (bf16), the residual read and the output written (fp32), the weights
    once."""
    M = B * gh * gw
    return 2.0 * M * C + 8.0 * M * C + 2.0 * 2 * C * hidden + 4.0 * (11 * hidden + C)


def unfused_conv_mlp_nbytes(B, gh, gw, C, hidden):
    """HBM bytes of the same block as three launches (fc1 GEMM, dwconv_bias_act, fc2 GEMM): the bf16 hidden tensor is
    written by fc1, read and written by the depthwise convolution, and read by fc2."""
    return conv_mlp_nbytes(B, gh, gw, C, hidden) + 4 * 2.0 * B * gh * gw * hidden


def pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act, out=None):
    """out = residual + act(dwconv3x3(bf16(h w1^T + b1)) + bdw) w2^T + b2 in one kernel (in place when ``out`` is
    ``residual``).  h: bf16 (B * gh * gw, C); w1: bf16 (hidden, C); wdw: fp32 (9, hidden); w2: bf16 (C, hidden); b1,
    bdw, b2: fp32; residual: fp32 (B * gh * gw, C).  ValueError for shapes the kernel does not take
    (``conv_mlp_supported``)."""
    C, hidden = h.shape[1], w1.shape[0]
    if not conv_mlp_supported(C, hidden):
        raise ValueError(f"pvt_v2_conv_mlp_bf16: needs C in {CONV_MLP_CHANNELS} and hidden % "
                         f"{CONV_MLP_HIDDEN_STEP} == 0 (got C={C}, hidden={hidden})")
    dev = _ops._cuda(h, w1, b1, wdw, bdw, w2, b2, residual, out)
    M = B * gh * gw
    assert h.dtype == w1.dtype == w2.dtype == torch.bfloat16, (h.dtype, w1.dtype, w2.dtype)
    assert h.shape == (M, C) and w1.shape == (hidden, C) and w2.shape == (C, hidden), (h.shape, w1.shape, w2.shape)
    assert wdw.shape == (9, hidden) and b1.shape == bdw.shape == (hidden,) and b2.shape == (C,)
    assert residual.dtype == torch.float32 and residual.shape == (M, C)
    for t in (h, w1, w2, b1, wdw, bdw, b2, residual):
        assert t.is_contiguous()
    for t in (b1, wdw, bdw, b2):
        assert t.dtype == torch.float32
    if out is None:
        out = torch.empty_like(residual)
    assert out.dtype == torch.float32 and out.shape == (M, C) and out.is_contiguous()
    _ops._call("tfimm_b200_pvt_v2_conv_mlp_bf16", dev, h.data_ptr(), w1.data_ptr(), b1.data_ptr(), wdw.data_ptr(),
               bdw.data_ptr(), w2.data_ptr(), b2.data_ptr(), residual.data_ptr(), out.data_ptr(), B, gh, gw, C, hidden,
               _ops.act_code(act), flops=2.0 * M * hidden * (2 * C + 9),
               nbytes=conv_mlp_nbytes(B, gh, gw, C, hidden))
    return out


def conv_mlp(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act, out=None):
    """The ConvFFN in the precision of ``h``.  bf16 at the shapes of ``conv_mlp_supported`` with C in
    ``CONV_MLP_FUSED_CHANNELS``: the fused kernel; every other shape, and fp32 (the fp32 and tf32 precisions): fc1
    GEMM (+ b1), ``ops.dwconv_bias_act`` (3 x 3, stride 1, one cell of zero padding, + bdw, act), fc2 GEMM (+ b2,
    + residual).  The rounding points are the same on both paths."""
    C, hidden = h.shape[1], w1.shape[0]
    if h.dtype == torch.bfloat16 and C in CONV_MLP_FUSED_CHANNELS and conv_mlp_supported(C, hidden):
        return pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act, out=out)
    hid = _ops.gemm(h, w1, bias=b1)
    hid = _ops.dwconv_bias_act(hid.view(B, gh, gw, hidden), wdw, bdw, 3, 1, "symmetric", act=act)
    return _ops.gemm(hid.view(B * gh * gw, hidden), w2, bias=b2, residual=residual, out=out)


# ------------------------------------------------------------------------------------------------------ attention
def pvt_v2_sr_attention_bf16(q, kv, B, N, Nk, H, dh, scale):
    """softmax(scale q k^T) v with queries from q (B * N, H * dh) and keys / values from kv (B * Nk, 2 * H * dh), read
    as (B, Nk, 2, H, dh); bf16 in and out, dh 32, tensor cores."""
    return _sr_attention("tfimm_b200_pvt_v2_sr_attention_bf16", torch.bfloat16, q, kv, B, N, Nk, H, dh, scale)


def pvt_v2_sr_attention_f32(q, kv, B, N, Nk, H, dh, scale):
    """The same on fp32 q / kv, with an fp32 softmax on the CUDA cores."""
    return _sr_attention("tfimm_b200_pvt_v2_sr_attention_f32", torch.float32, q, kv, B, N, Nk, H, dh, scale)


def _sr_attention(name, dtype, q, kv, B, N, Nk, H, dh, scale):
    dev = _ops._cuda(q, kv)
    assert q.dtype == kv.dtype == dtype and q.is_contiguous() and kv.is_contiguous(), (q.dtype, kv.dtype)
    assert q.shape == (B * N, H * dh) and kv.shape == (B * Nk, 2 * H * dh), (q.shape, kv.shape, (B, N, Nk, H, dh))
    out = torch.empty((B * N, H * dh), device=q.device, dtype=dtype)
    _ops._call(name, dev, q.data_ptr(), kv.data_ptr(), out.data_ptr(), B, N, Nk, H, dh, float(scale),
               flops=4.0 * B * H * N * Nk * dh, nbytes=_pvt_ops.sr_attention_nbytes(B, N, Nk, H, dh, q.element_size()))
    return out


def sr_attention(q, kv, B, N, Nk, H, dh, scale):
    """Spatial-reduction attention in the precision of ``q``: head dim 64 -> ``pvt_ops.sr_attention``; head dim 32 ->
    the kernels here (bf16: tensor cores; fp32, for the fp32 and tf32 precisions: CUDA cores)."""
    if dh == 64:
        return _pvt_ops.sr_attention(q, kv, B, N, Nk, H, dh, scale)
    if dh != 32:
        raise _lib.KernelLibraryError(f"PVT v2 attention: no kernel for head_dim {dh} (have {HEAD_DIMS})")
    if q.dtype == torch.bfloat16:
        return pvt_v2_sr_attention_bf16(q, kv, B, N, Nk, H, dh, scale)
    return pvt_v2_sr_attention_f32(q, kv, B, N, Nk, H, dh, scale)
