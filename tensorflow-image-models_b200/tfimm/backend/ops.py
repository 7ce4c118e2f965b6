"""Tensor-level launchers: torch CUDA tensors in, kernel launches on torch's current stream.

torch is used for device memory and stream handles only; every function here ends in exactly
one call into ``libtfimm_b200.so``.  Nothing falls back to torch ops.
"""
from typing import Optional

import torch

from . import lib as _lib

F32, BF16, U8 = _lib.F32, _lib.BF16, _lib.U8
_DT = {torch.float32: F32, torch.bfloat16: BF16, torch.uint8: U8}

# number of kernels launched through this module (bench.py reports it as gpu_launches)
launch_count = 0


def _code(t: torch.Tensor) -> int:
    try:
        return _DT[t.dtype]
    except KeyError:
        raise TypeError(f"tfimm_b200 kernels take float32 / bfloat16 / uint8 tensors, got {t.dtype}")


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _cuda(*tensors):
    """The device of a launch's operands: all of them CUDA tensors on one device."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.KernelLibraryError(
                "tfimm_b200 kernels only run on CUDA tensors (there is no CPU fallback)."
            )
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise _lib.KernelLibraryError(f"tfimm_b200: operands on different devices ({dev} and {t.device}).")
    return dev


# When set to a list, every launch is bracketed by CUDA events on the launching stream and
# (family, start, end, algorithmic flops, algorithmic bytes) is appended (bench.py roofline pass).
trace = None

# Kernel family of each entry point in ``trace`` (bench.py's roofline rows, tools/ncu_traffic.py): its name without the
# library prefix, except for the entry points that run another family's kernel.
TRACE_FAMILY = {name: name[len("tfimm_b200_"):] for name in _lib.SIGNATURES}
TRACE_FAMILY.update({
    "tfimm_b200_conv_bf16": "gemm_bf16",
    "tfimm_b200_gemm_bf16_gated": "gemm_bf16",
    "tfimm_b200_window_attention_tc_bf16": "window_attention_bf16",
    "tfimm_b200_im2col_u8": "im2col",
})


def _call(name, dev, *args, flops=0.0, nbytes=0.0):
    """Calls entry point ``name`` with ``args`` and the current stream of ``dev`` (every entry point takes its stream
    last), with ``dev`` as the current device: cudaFuncSetAttribute, the launch and the SM count all refer to it."""
    global launch_count
    fn = getattr(_lib.load(), name)
    if dev.index != torch.cuda.current_device():
        with torch.cuda.device(dev):
            return _call(name, dev, *args, flops=flops, nbytes=nbytes)
    args = (*args, torch.cuda.current_stream(dev).cuda_stream)
    if trace is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(fn(*args), name)
        e1.record()
        trace.append((TRACE_FAMILY[name], e0, e1, float(flops), float(nbytes)))
    else:
        _lib.check(fn(*args), name)
    launch_count += 1


def _nbytes(*tensors):
    return float(sum(t.numel() * t.element_size() for t in tensors if t is not None))


def act_code(act) -> int:
    try:
        return _lib.ACT[act]
    except KeyError:
        raise ValueError(f"Unknown activation: {act}.")


def gemm(a, w, bias=None, act=None, gamma=None, residual=None, out=None, out_dtype=None, block_n=0,
         act_after_residual=False):
    """out = residual + gamma * act(a @ w.T + bias)  (act_after_residual: act(residual + gamma*(...))).
    a:(M,K), w:(N,K); bf16 -> wgmma, fp32 -> SIMT, or TF32 wgmma in a tf32 model's forward (``lib.tf32_mode``)."""
    dev = _cuda(a, w, bias, gamma, residual, out)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K, (a.shape, w.shape)
    assert a.stride(1) == 1 and w.stride(1) == 1
    if out is None:
        out_dtype = out_dtype or (residual.dtype if residual is not None else a.dtype)
        ldc = (N + 7) // 8 * 8
        buf = torch.empty((M, ldc), device=a.device, dtype=out_dtype)
        out = buf[:, :N] if ldc != N else buf
    assert out.shape == (M, N) and out.stride(1) == 1
    if residual is not None:
        assert residual.shape == (M, N) and residual.dtype == out.dtype and residual.stride(1) == 1
    ldr = residual.stride(0) if residual is not None else 0
    args = (a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), _ptr(bias), _ptr(gamma), _ptr(residual), ldr,
            out.data_ptr(), out.stride(0), M, N, K, act_code(act), int(bool(act_after_residual)))
    flops, nbytes = 2.0 * M * N * K, _nbytes(a, w, out, residual)
    if a.dtype == torch.bfloat16:
        assert w.dtype == torch.bfloat16
        _call("tfimm_b200_gemm_bf16", dev, *args, _code(out), block_n, flops=flops, nbytes=nbytes)
    elif _lib.tf32_mode.get():
        # precision="tf32": w was rounded to TF32 when the plan was built; the kernel rounds the A tiles
        assert a.dtype == torch.float32 and w.dtype == torch.float32 and out.dtype == torch.float32
        _call("tfimm_b200_gemm_tf32", dev, *args, block_n, flops=flops, nbytes=nbytes)
    else:
        assert a.dtype == torch.float32 and w.dtype == torch.float32 and out.dtype == torch.float32
        _call("tfimm_b200_gemm_f32", dev, *args, flops=flops, nbytes=nbytes)
    return out


def gemm_gated(a, gate, rows_per_image, w, bias=None, act=None, residual=None):
    """act((a * gate[row // rows_per_image]) @ w.T + bias) + residual, bf16: the squeeze-excite gate (B, K) fp32 is applied
    to the A tile in shared memory (rounded to bf16 like ``scale_channels_``), not in a pass over HBM."""
    dev = _cuda(a, gate, w, bias, residual)
    M, K = a.shape
    N = w.shape[0]
    assert a.dtype == w.dtype == torch.bfloat16 and a.stride(1) == 1 and w.stride(1) == 1 and w.shape[1] == K
    assert gate.dtype == torch.float32 and gate.is_contiguous() and gate.shape[1] == K
    assert gate.shape[0] * rows_per_image >= M
    ldc = (N + 7) // 8 * 8
    buf = torch.empty((M, ldc), device=a.device, dtype=torch.bfloat16)
    out = buf[:, :N] if ldc != N else buf
    if residual is not None:
        assert residual.shape == (M, N) and residual.dtype == torch.bfloat16 and residual.stride(1) == 1
    _call("tfimm_b200_gemm_bf16_gated", dev, a.data_ptr(), a.stride(0), gate.data_ptr(), int(rows_per_image),
          gate.shape[0], w.data_ptr(), w.stride(0), _ptr(bias), _ptr(residual),
          residual.stride(0) if residual is not None else 0, out.data_ptr(), out.stride(0), M, N, K, act_code(act),
          flops=2.0 * M * N * K, nbytes=_nbytes(a, w, out, residual))
    return out


def mlp_fused_supported(C, hidden):
    """Shapes of the fused fc1 -> act -> fc2 kernel (csrc/mlp_sm90.cu)."""
    return C in (96, 128, 192, 256) and hidden % 128 == 0 and hidden >= 256


def mlp_fused(a, w1, b1, w2, b2, act, gamma=None, residual=None, out=None):
    """out = residual + gamma * (act(a @ w1.T + b1) @ w2.T + b2) in one kernel; the hidden activations stay on the SM.
    a:(M,C) bf16, w1:(hidden,C), w2:(C,hidden) bf16, residual / out:(M,C) fp32 (may alias)."""
    dev = _cuda(a, w1, b1, w2, b2, gamma, residual, out)
    M, C = a.shape
    Hd = w1.shape[0]
    assert w1.shape == (Hd, C) and w2.shape == (C, Hd), (a.shape, w1.shape, w2.shape)
    assert a.dtype == w1.dtype == w2.dtype == torch.bfloat16
    assert a.stride(1) == 1 and w1.stride(1) == 1 and w2.stride(1) == 1
    if out is None:
        out = torch.empty((M, C), device=a.device, dtype=torch.float32)
    assert out.shape == (M, C) and out.dtype == torch.float32 and out.stride(1) == 1
    if residual is not None:
        assert residual.shape == (M, C) and residual.dtype == torch.float32 and residual.stride(1) == 1
    _call("tfimm_b200_mlp_bf16", dev, a.data_ptr(), a.stride(0), w1.data_ptr(), w1.stride(0), _ptr(b1), w2.data_ptr(),
          w2.stride(0), _ptr(b2), _ptr(gamma), _ptr(residual), residual.stride(0) if residual is not None else 0,
          out.data_ptr(), out.stride(0), M, C, Hd, act_code(act), flops=4.0 * M * C * Hd,
          nbytes=_nbytes(a, w1, w2, out, residual))
    return out


def conv_gemm(x, w, bias=None, ks=3, stride=1, pad=1, act=None, residual=None, act_after_residual=False,
              out_dtype=None):
    """Dense k x k convolution as an implicit GEMM (no im2col matrix).  x: (B,H,W,C) bf16 with C % 64 == 0;
    w: (N, ks*ks*C) bf16 in (ky, kx, c) order; residual / result: (B,Ho,Wo,N).  In a tf32 model's forward
    (``lib.tf32_mode``): x, w, residual and result fp32, C % 32 == 0, TF32 products."""
    dev = _cuda(x, w, bias, residual)
    B, H, W, C = x.shape
    N = w.shape[0]
    tf32 = x.dtype == torch.float32 and _lib.tf32_mode.get()
    assert x.dtype == w.dtype and (x.dtype == torch.bfloat16 or tf32), (x.dtype, w.dtype)
    assert x.is_contiguous() and w.stride(1) == 1
    assert w.shape[1] == ks * ks * C, (w.shape, ks, C)
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    out_dtype = out_dtype or (residual.dtype if residual is not None else x.dtype)
    out = torch.empty((B, Ho, Wo, N), device=x.device, dtype=out_dtype)
    if residual is not None:
        assert residual.shape == out.shape and residual.dtype == out.dtype and residual.is_contiguous()
    if tf32:
        assert out.dtype == torch.float32
        _call("tfimm_b200_conv_tf32", dev, x.data_ptr(), w.data_ptr(), w.stride(0), _ptr(bias), _ptr(residual),
              out.data_ptr(), B, H, W, C, N, ks, stride, pad, act_code(act), int(bool(act_after_residual)),
              flops=2.0 * B * Ho * Wo * N * ks * ks * C, nbytes=_nbytes(x, w, out, residual))
        return out
    _call("tfimm_b200_conv_bf16", dev, x.data_ptr(), w.data_ptr(), w.stride(0), _ptr(bias), _ptr(residual),
          out.data_ptr(), B, H, W, C, N, ks, stride, pad, act_code(act), int(bool(act_after_residual)), _code(out),
          flops=2.0 * B * Ho * Wo * N * ks * ks * C, nbytes=_nbytes(x, w, out, residual))
    return out


def attention_cls(qkv, B, T, H, dh, scale, nq=1):
    """softmax(q K^T) V for the first ``nq`` query tokens of every image only -> (B*nq, H*dh) bf16."""
    dev = _cuda(qkv)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (B * T, 3 * H * dh)
    out = torch.empty((B * nq, H * dh), device=qkv.device, dtype=torch.bfloat16)
    _call("tfimm_b200_attention_cls_bf16", dev, qkv.data_ptr(), out.data_ptr(), B, T, H, dh, nq, float(scale),
          flops=4.0 * B * H * nq * T * dh, nbytes=2.0 * B * T * 2 * H * dh)
    return out


def layernorm(x, gamma, beta, eps, out_dtype, out=None):
    """LayerNorm over the last axis of a 2D (possibly row-strided) tensor."""
    dev = _cuda(x, gamma, beta, out)
    rows, C = x.shape
    assert x.stride(1) == 1
    if out is None:
        out = torch.empty((rows, C), device=x.device, dtype=out_dtype)
    _call("tfimm_b200_layernorm", dev, x.data_ptr(), _code(x), x.stride(0), gamma.data_ptr(), beta.data_ptr(),
          out.data_ptr(), _code(out), out.stride(0), rows, C, float(eps),
          nbytes=rows * C * (x.element_size() + out.element_size()))
    return out


def layernorm_patch2x2(x, gamma, beta, eps, out_dtype):
    """x: (B,H,W,C) contiguous -> (B*H/2*W/2, 4C) LN'd pixels in 2x2/stride-2 im2col order."""
    dev = _cuda(x, gamma, beta)
    B, H, W, C = x.shape
    assert x.is_contiguous()
    out = torch.empty((B * (H // 2) * (W // 2), 4 * C), device=x.device, dtype=out_dtype)
    _call("tfimm_b200_layernorm_patch2x2", dev, x.data_ptr(), _code(x), gamma.data_ptr(), beta.data_ptr(),
          out.data_ptr(), _code(out), B, H, W, C, float(eps), nbytes=_nbytes(x, out))
    return out


def patch_merge_ln(x, gamma, beta, eps, out_dtype):
    """Swin PatchMerging gather + LN.  x: (B,H,W,C) contiguous -> (B*H/2*W/2, 4C)."""
    dev = _cuda(x, gamma, beta)
    B, H, W, C = x.shape
    assert x.is_contiguous()
    out = torch.empty((B * (H // 2) * (W // 2), 4 * C), device=x.device, dtype=out_dtype)
    _call("tfimm_b200_patch_merge_ln", dev, x.data_ptr(), _code(x), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(),
          _code(out), B, H, W, C, float(eps), nbytes=_nbytes(x, out))
    return out


def attention(qkv, B, N, H, dh, scale, bias=None, mask=None, probs=None, row_map=None, nw_img=0):
    """softmax(scale q k^T [+bias +mask]) v from packed qkv (B*N, 3*H*dh) -> (B*N, H*dh).
    row_map/nw_img (fp32 only): Swin window permutation folded into addressing.  In a tf32 model's forward, fp32 qkv
    with head_dim 64 and none of bias / mask / probs / row_map runs the TF32 tensor-core kernel; the rest stays SIMT."""
    dev = _cuda(qkv, bias, mask, probs, row_map)
    assert qkv.shape == (B * N, 3 * H * dh) and qkv.is_contiguous()
    out = torch.empty((B * N, H * dh), device=qkv.device, dtype=qkv.dtype)
    plain = bias is None and mask is None and probs is None and row_map is None
    flops = 4.0 * B * H * N * N * dh
    if qkv.dtype == torch.bfloat16 and plain:
        _call("tfimm_b200_attention_bf16", dev, qkv.data_ptr(), out.data_ptr(), B, N, H, dh, float(scale), flops=flops,
              nbytes=_nbytes(qkv, out))
    elif qkv.dtype == torch.float32 and plain and dh == 64 and _lib.tf32_mode.get():
        _call("tfimm_b200_attention_tf32", dev, qkv.data_ptr(), out.data_ptr(), B, N, H, dh, float(scale), flops=flops,
              nbytes=_nbytes(qkv, out))
    elif qkv.dtype == torch.float32:
        nmask = mask.shape[0] if mask is not None else 1
        _call("tfimm_b200_attention_f32", dev, qkv.data_ptr(), out.data_ptr(), _ptr(bias), _ptr(mask), nmask, B, N, H,
              dh, float(scale), _ptr(probs), _ptr(row_map), nw_img, flops=flops, nbytes=_nbytes(qkv, out, probs))
    else:
        raise _lib.KernelLibraryError("attention: unsupported dtype / option combination")
    return out


def attention_bf16_supported(N, dh) -> bool:
    """Shapes the bf16 tensor-core attention kernels take (csrc/attention.cu: head_dim 64, resident K/V <= 227 KB)."""
    return dh == 64 and N <= 832


def patchify(img, p, out_dtype, mean=None, inv_std=None, scale=1.0):
    """img: (B,H,W,C) -> (B*H/p*W/p, ceil8(p*p*C)); optional fused (x*scale-mean)*inv_std."""
    dev = _cuda(img, mean, inv_std)
    B, H, W, C = img.shape
    assert img.is_contiguous()
    K = p * p * C
    Kpad = (K + 7) // 8 * 8
    out = torch.empty((B * (H // p) * (W // p), Kpad), device=img.device, dtype=out_dtype)
    _call("tfimm_b200_patchify", dev, img.data_ptr(), _code(img), out.data_ptr(), _code(out), B, H, W, C, p, Kpad,
          float(scale), _ptr(mean), _ptr(inv_std), nbytes=_nbytes(img, out))
    return out


def assemble_tokens(patches, cls, dist, pos, B, P, out_dtype):
    dev = _cuda(patches, cls, dist, pos)
    D = patches.shape[1]
    ntok = 2 if dist is not None else 1
    out = torch.empty((B * (P + ntok), D), device=patches.device, dtype=out_dtype)
    _call("tfimm_b200_assemble_tokens", dev, patches.data_ptr(), _code(patches), cls.data_ptr(), _ptr(dist),
          pos.data_ptr(), out.data_ptr(), _code(out), B, P, ntok, D, nbytes=_nbytes(patches, out))
    return out


def cast(x, dtype):
    dev = _cuda(x)
    if x.dtype == dtype:
        return x
    x = x.contiguous()
    out = torch.empty(x.shape, device=x.device, dtype=dtype)
    _call("tfimm_b200_cast", dev, x.data_ptr(), _code(x), out.data_ptr(), _code(out), x.numel(), nbytes=_nbytes(x, out))
    return out


def dwconv_ln(x, wgt, bias, gamma, beta, eps, out_dtype):
    """ConvNeXt block head: depthwise 7x7 (pad 3, bias) + LayerNorm.  x: (B,H,W,C) -> (B*H*W, C)."""
    dev = _cuda(x, wgt, bias, gamma, beta)
    B, H, W, C = x.shape
    assert x.is_contiguous()
    ks = int(round((wgt.shape[0]) ** 0.5))
    out = torch.empty((B * H * W, C), device=x.device, dtype=out_dtype)
    _call("tfimm_b200_dwconv_ln", dev, x.data_ptr(), _code(x), wgt.data_ptr(), bias.data_ptr(), gamma.data_ptr(),
          beta.data_ptr(), out.data_ptr(), _code(out), B, H, W, C, ks, float(eps), flops=2.0 * B * H * W * C * ks * ks,
          nbytes=_nbytes(x, out))
    return out


def same_pad(size, k, s):
    """TF "same": returns (out_size, pad_before)."""
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return out, total // 2


def dwconv_bias_act(x, wgt, bias, ks, stride, padding, act=None, pool_sum=None):
    """Depthwise conv + bias + act.  padding: "same" (TF, asymmetric) | "symmetric" | "valid".
    x: (B,H,W,C) -> (B,Ho,Wo,C); pool_sum: optional (B,C) fp32 zero-initialised accumulator."""
    dev = _cuda(x, wgt, bias, pool_sum)
    B, H, W, C = x.shape
    assert x.is_contiguous()
    if padding == "same":
        Ho, pt = same_pad(H, ks, stride)
        Wo, pl = same_pad(W, ks, stride)
    elif padding == "symmetric":
        pt = pl = ((stride - 1) + (ks - 1)) // 2
        Ho = (H + 2 * pt - ks) // stride + 1
        Wo = (W + 2 * pl - ks) // stride + 1
    elif padding == "valid":
        pt = pl = 0
        Ho = (H - ks) // stride + 1
        Wo = (W - ks) // stride + 1
    else:
        raise ValueError(f"Unknown padding {padding}")
    out = torch.empty((B, Ho, Wo, C), device=x.device, dtype=x.dtype)
    _call("tfimm_b200_dwconv_bias_act", dev, x.data_ptr(), _code(x), wgt.data_ptr(), _ptr(bias), out.data_ptr(),
          _ptr(pool_sum), B, H, W, C, ks, stride, pt, pl, Ho, Wo, act_code(act), flops=2.0 * B * Ho * Wo * C * ks * ks,
          nbytes=_nbytes(x, out))
    return out


def global_avg_pool(x):
    """(B, HW, C) or (B, H, W, C) -> (B, C) fp32 mean over the spatial axes."""
    dev = _cuda(x)
    assert x.is_contiguous()
    B, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * C)
    out = torch.empty((B, C), device=x.device, dtype=torch.float32)
    _call("tfimm_b200_global_avg_pool", dev, x.data_ptr(), _code(x), out.data_ptr(), B, HW, C, nbytes=_nbytes(x, out))
    return out


def window_attention(qkv, bias, row_map, labels, B, nw_img, N, H, dh, scale):
    """Swin (shifted-)window attention on token-ordered qkv (B*nw_img*N, 3*H*dh) -> (B*nw_img*N, H*dh)."""
    dev = _cuda(qkv, bias, row_map, labels)
    assert qkv.shape == (B * nw_img * N, 3 * H * dh) and qkv.is_contiguous() and qkv.dtype == torch.bfloat16
    assert row_map.dtype == torch.int32 and (labels is None or labels.dtype == torch.int32)
    out = torch.empty((B * nw_img * N, H * dh), device=qkv.device, dtype=qkv.dtype)
    _call("tfimm_b200_window_attention_bf16", dev, qkv.data_ptr(), out.data_ptr(), bias.data_ptr(), row_map.data_ptr(),
          _ptr(labels), B, nw_img, N, H, dh, float(scale), flops=4.0 * B * nw_img * H * N * N * dh,
          nbytes=_nbytes(qkv, out))
    return out


def window_attention_tc(qkv, bias_pad, row_map, maskbits, B, nw_img, N, H, dh, scale):
    """Swin (shifted-)window attention for 7 x 7 windows (head_dim 32, N <= 52): token-ordered qkv (B*nw_img*N, 3*H*dh) ->
    (B*nw_img*N, H*dh).  bias_pad: fp32 (H, 64, 64); maskbits: int64 (nw_img, 64) or None (see window_mask_bits)."""
    dev = _cuda(qkv, bias_pad, row_map, maskbits)
    assert qkv.shape == (B * nw_img * N, 3 * H * dh) and qkv.is_contiguous() and qkv.dtype == torch.bfloat16
    assert bias_pad.shape == (H, 64, 64) and bias_pad.dtype == torch.float32 and bias_pad.is_contiguous()
    assert row_map.dtype == torch.int32 and (maskbits is None or (maskbits.dtype == torch.int64
                                                                 and maskbits.shape == (nw_img, 64)))
    out = torch.empty((B * nw_img * N, H * dh), device=qkv.device, dtype=qkv.dtype)
    _call("tfimm_b200_window_attention_tc_bf16", dev, qkv.data_ptr(), out.data_ptr(), bias_pad.data_ptr(),
          row_map.data_ptr(), _ptr(maskbits), B, nw_img, N, H, dh, float(scale),
          flops=4.0 * B * nw_img * H * N * N * dh, nbytes=_nbytes(qkv, out))
    return out


def conv_geometry(H, W, ks, stride, padding):
    """(Ho, Wo, pad_top, pad_left) for "same" (TF, asymmetric) | "symmetric" (PyTorch-style) | "valid" | int."""
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


def im2col(x, ks, stride, padding, out_dtype, groups=1, pre=None):
    """x: (B,H,W,C) -> ((B*Ho*Wo, ceil8(ks*ks*C)), Ho, Wo); groups > 1: ((groups, B*Ho*Wo, ceil8(ks*ks*C/groups)), ...)
    with one im2col matrix per channel group.  uint8 ``x`` (raw pixels) needs ``pre = (mean, inv_std, scale)``: the
    gathered values are (x * scale - mean[c]) * inv_std[c], the padding stays zero."""
    dev = _cuda(x)
    B, H, W, C = x.shape
    assert x.is_contiguous() and C % groups == 0
    Ho, Wo, pt, pl = conv_geometry(H, W, ks, stride, padding)
    Kpad = (ks * ks * (C // groups) + 7) // 8 * 8
    shape = (B * Ho * Wo, Kpad) if groups == 1 else (groups, B * Ho * Wo, Kpad)
    out = torch.empty(shape, device=x.device, dtype=out_dtype)
    if x.dtype == torch.uint8:
        assert pre is not None and groups == 1, "uint8 input: pass pre=(mean, inv_std, scale)"
        mean, inv_std, scale = pre
        dev = _cuda(x, mean, inv_std)
        _call("tfimm_b200_im2col_u8", dev, x.data_ptr(), out.data_ptr(), _code(out), B, H, W, C, ks, stride, pt, pl, Ho,
              Wo, Kpad, float(scale), mean.data_ptr(), inv_std.data_ptr(), nbytes=_nbytes(x, out))
        return out, Ho, Wo
    _call("tfimm_b200_im2col", dev, x.data_ptr(), _code(x), out.data_ptr(), _code(out), B, H, W, C, groups, ks, stride,
          pt, pl, Ho, Wo, Kpad, nbytes=_nbytes(x, out))
    return out, Ho, Wo


def group_norm(x, gamma, beta, groups, eps, act=None, residual=None):
    """GroupNormalization over an NHWC tensor, then optional ``+ residual`` and activation."""
    dev = _cuda(x, gamma, beta, residual)
    B, H, W, C = x.shape
    assert x.is_contiguous() and (residual is None or (residual.shape == x.shape and residual.is_contiguous()
                                                       and residual.dtype == x.dtype))
    out = torch.empty_like(x)
    stats = torch.empty((B, groups, 2), device=x.device, dtype=torch.float32)
    _call("tfimm_b200_group_norm", dev, x.data_ptr(), _code(x), gamma.data_ptr(), beta.data_ptr(), _ptr(residual),
          out.data_ptr(), stats.data_ptr(), B, H * W, C, groups, float(eps), act_code(act),
          nbytes=_nbytes(x, x, out, residual))
    return out


def blur_pool(x, stride=2):
    """BlurPool2D: REFLECT pad 1, 3x3 binomial blur, stride."""
    dev = _cuda(x)
    B, H, W, C = x.shape
    assert x.is_contiguous()
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = torch.empty((B, Ho, Wo, C), device=x.device, dtype=x.dtype)
    _call("tfimm_b200_blur_pool", dev, x.data_ptr(), _code(x), out.data_ptr(), B, H, W, C, stride, Ho, Wo,
          nbytes=_nbytes(x, out))
    return out


def se_gate(pooled_sum, hw, w_reduce, b_reduce, w_expand, b_expand, act, gate_act="sigmoid"):
    """pooled_sum: (B, C) fp32 sums over hw pixels -> gate (B, C) fp32."""
    dev = _cuda(pooled_sum, w_reduce, b_reduce, w_expand, b_expand)
    B, C = pooled_sum.shape
    rd = w_reduce.shape[0]
    gate = torch.empty((B, C), device=pooled_sum.device, dtype=torch.float32)
    _call("tfimm_b200_se_gate", dev, pooled_sum.data_ptr(), 1.0 / float(hw), w_reduce.data_ptr(), b_reduce.data_ptr(),
          w_expand.data_ptr(), b_expand.data_ptr(), gate.data_ptr(), B, C, rd, act_code(act), act_code(gate_act),
          flops=4.0 * B * C * rd, nbytes=_nbytes(pooled_sum, gate))
    return gate


def scale_channels_(x, gate):
    """In place: x[b, ..., c] *= gate[b, c]."""
    dev = _cuda(x, gate)
    assert x.is_contiguous()
    B, C = gate.shape
    HW = x.numel() // (B * C)
    _call("tfimm_b200_scale_channels", dev, x.data_ptr(), _code(x), gate.data_ptr(), B, HW, C, nbytes=2 * _nbytes(x))
    return x


def pool2d(x, ks, stride, padding, mode):
    """mode "max" | "avg" on (B,H,W,C); padding as in conv_geometry."""
    dev = _cuda(x)
    B, H, W, C = x.shape
    assert x.is_contiguous()
    Ho, Wo, pt, pl = conv_geometry(H, W, ks, stride, padding)
    out = torch.empty((B, Ho, Wo, C), device=x.device, dtype=x.dtype)
    _call("tfimm_b200_pool2d", dev, x.data_ptr(), _code(x), out.data_ptr(), B, H, W, C, ks, stride, pt, pl, Ho, Wo,
          {"max": 0, "avg": 1, "max_zero_pad": 2}[mode], nbytes=_nbytes(x, out))
    return out


def grouped_conv(x, wgt, bias, cg, ks, stride, pad, act=None):
    """Grouped k x k conv (cg channels per group, in == out) + bias + act.  wgt: (ks*ks, cg, C) fp32."""
    dev = _cuda(x, wgt, bias)
    B, H, W, C = x.shape
    assert x.is_contiguous()
    Ho, Wo, _, _ = conv_geometry(H, W, ks, stride, pad)
    out = torch.empty((B, Ho, Wo, C), device=x.device, dtype=x.dtype)
    _call("tfimm_b200_grouped_conv", dev, x.data_ptr(), _code(x), wgt.data_ptr(), _ptr(bias), out.data_ptr(), B, H, W,
          C, cg, ks, stride, pad, Ho, Wo, act_code(act), flops=2.0 * B * Ho * Wo * C * cg * ks * ks,
          nbytes=_nbytes(x, out))
    return out


def eca_gate(mean, w):
    """mean: (B, C) fp32, w: (ks,) fp32 -> gate (B, C) fp32."""
    dev = _cuda(mean, w)
    B, C = mean.shape
    gate = torch.empty_like(mean)
    _call("tfimm_b200_eca_gate", dev, mean.data_ptr(), w.data_ptr(), gate.data_ptr(), B, C, w.numel(),
          nbytes=_nbytes(mean, gate))
    return gate


def scale_add_act_(x, gate, shortcut, act):
    """In place: x = act(x * gate[b] + shortcut)."""
    dev = _cuda(x, gate, shortcut)
    assert x.is_contiguous() and shortcut.is_contiguous() and x.shape == shortcut.shape and x.dtype == shortcut.dtype
    B, C = gate.shape
    HW = x.numel() // (B * C)
    _call("tfimm_b200_scale_add_act", dev, x.data_ptr(), _code(x), gate.data_ptr(), shortcut.data_ptr(), B, HW, C,
          act_code(act), nbytes=3 * _nbytes(x))
    return x
