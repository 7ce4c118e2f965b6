"""Launchers of the MLP-Mixer family's kernels (token mixing and channel GLU in ``csrc/gemm_sm90.cu``, their fp32 forms
and the Affine norm in ``csrc/mixer.cu``).

Same conventions as ``tfimm.backend.ops``: torch CUDA tensors in, one library call on the operands' device's current
stream, counted in ``ops.launch_count`` and bracketed by CUDA events when ``ops.trace`` is set.  Nothing falls back to
torch ops.  The token weights are the Dense kernels in the engine layout (``Model._dense_weight``); the GLU layouts come
from ``glu_interleave``.
"""
import torch

from . import lib as _lib
from . import ops as _ops


def _ceil(n, m):
    return (n + m - 1) // m * m


def glu_interleave(w, b, axis_rows):
    """Reorders the output features of a GLU layer's fc1 so that one epilogue thread holds value j and gate j.
    w: (F, K) engine layout (row f = output feature f, the value half first, then the gate half); b: (F,).
    axis_rows=True (token GLU and the fp32 channel GLU): per 16 rows, 8 value rows then their 8 gate rows, with each half
    zero-padded to a multiple of 8 features; axis_rows=False (bf16 channel GLU): rows 2j / 2j + 1 = value / gate j."""
    F = w.shape[0]
    h = F // 2
    xv, xg, bv, bg = w[:h], w[h:], b[:h], b[h:]
    if not axis_rows:
        return (torch.stack((xv, xg), 1).reshape(F, -1).contiguous(), torch.stack((bv, bg), 1).reshape(F).contiguous())
    hp = _ceil(h, 8)
    pad = (0, 0, 0, hp - h)
    xv, xg = torch.nn.functional.pad(xv, pad), torch.nn.functional.pad(xg, pad)
    bv, bg = torch.nn.functional.pad(bv, (0, hp - h)), torch.nn.functional.pad(bg, (0, hp - h))
    wt = torch.stack((xv.reshape(hp // 8, 8, -1), xg.reshape(hp // 8, 8, -1)), 1).reshape(2 * hp, -1)
    bt = torch.stack((bv.reshape(hp // 8, 8), bg.reshape(hp // 8, 8)), 1).reshape(2 * hp)
    return wt.contiguous(), bt.contiguous()


def token_gemm(wt, x, bias=None, act=None, gamma=None, residual=None, mul=None, out=None, m_out=None, glu=False,
               out_dtype=None, block_n=0):
    """Token mixing without transposes: out[b, m, c] = epi(sum_n wt[m, n] x[b, n, c]).

    wt: (M, K), unit column stride, row stride a multiple of 8 (the Dense kernel transposed; a column slice of the
    zero-padded plan tensor); x: (B, K, C) with unit channel stride (any row / image stride, e.g. a column slice).
    Epilogue: + bias[m] -> act (glu: rows in ``glu_interleave`` order, value * act(gate)) -> * gamma[c] -> * mul[b, row,
    c] -> + residual[b, row, c] (may be ``out``).  Rows >= m_out are not stored.  out / residual / mul: (B, m_out, C)
    with unit channel stride.  bf16 x: wgmma (out bf16 or fp32); fp32 x: CUDA cores."""
    dev = _ops._cuda(wt, x, bias, gamma, residual, mul, out)
    B, K, C = x.shape
    M = wt.shape[0]
    ldw = wt.stride(0)
    assert wt.shape[1] == K and wt.stride(1) == 1 and x.stride(2) == 1, (wt.shape, wt.stride(), x.shape)
    assert wt.dtype == x.dtype, (wt.dtype, x.dtype)
    if m_out is None:
        m_out = M // 2 if glu else M
    if out is None:
        out_dtype = out_dtype or (residual.dtype if residual is not None else x.dtype)
        out = torch.empty((B, m_out, C), device=x.device, dtype=out_dtype)
    for t in (out, residual, mul):
        if t is not None:
            assert t.shape == (B, m_out, C) and t.stride(2) == 1 and t.dtype == out.dtype, (t.shape, t.dtype)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.shape == (M,) and bias.is_contiguous()
    if gamma is not None:
        assert gamma.dtype == torch.float32 and gamma.shape == (C,) and gamma.is_contiguous()

    def st(t):
        return (0, 0) if t is None else (t.stride(1), t.stride(0))

    (ldr, img_r), (ldu, img_u), (ldc, img_c) = st(residual), st(mul), st(out)
    flops = 2.0 * B * M * K * C
    nbytes = _ops._nbytes(wt, x, out, residual, mul)
    args = (wt.data_ptr(), ldw, x.data_ptr(), x.stride(1), x.stride(0), _ops._ptr(bias), _ops._ptr(gamma),
            _ops._ptr(residual), ldr, img_r, _ops._ptr(mul), ldu, img_u, out.data_ptr(), ldc, img_c, B, M, C, K, m_out,
            _ops.act_code(act), int(glu))
    if x.dtype == torch.bfloat16:
        _ops._call("tfimm_b200_token_gemm_bf16", dev, *args, _ops._code(out), block_n, flops=flops, nbytes=nbytes)
    elif x.dtype == torch.float32:
        assert out.dtype == torch.float32
        _ops._call("tfimm_b200_token_gemm_f32", dev, *args, flops=flops, nbytes=nbytes)
    else:
        raise _lib.KernelLibraryError(f"token_gemm: unsupported dtype {x.dtype}")
    return out


def gemm_glu(a, w, bias, n_out, act, block_n=0):
    """Channel GLU: (a @ w_value.T + b) * act(a @ w_gate.T + b) -> (M, n_out), with w / bias in ``glu_interleave`` order
    (bf16: axis_rows=False, fp32: axis_rows=True).  The full-width hidden tensor is never written."""
    dev = _ops._cuda(a, w, bias)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and a.stride(1) == 1 and w.stride(1) == 1 and a.dtype == w.dtype
    assert bias.dtype == torch.float32 and bias.shape == (N,)
    ldc = _ceil(n_out, 8)
    buf = torch.empty((M, ldc), device=a.device, dtype=a.dtype)
    out = buf[:, :n_out] if ldc != n_out else buf
    flops, nbytes = 2.0 * M * N * K, _ops._nbytes(a, w, out)
    args = (a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), bias.data_ptr(), out.data_ptr(), ldc, M, N)
    if a.dtype == torch.bfloat16:
        assert N == 2 * n_out
        _ops._call("tfimm_b200_gemm_glu_bf16", dev, *args, K, _ops.act_code(act), block_n, flops=flops, nbytes=nbytes)
    elif a.dtype == torch.float32:
        _ops._call("tfimm_b200_gemm_glu_f32", dev, *args, n_out, K, _ops.act_code(act), flops=flops, nbytes=nbytes)
    else:
        raise _lib.KernelLibraryError(f"gemm_glu: unsupported dtype {a.dtype}")
    return out


def affine(x, alpha, beta, out_dtype):
    """ResMLP's Affine norm alpha[c] x + beta[c] of a 2-D fp32 x (unit column stride) -> (rows, C) in out_dtype."""
    dev = _ops._cuda(x, alpha, beta)
    rows, C = x.shape
    assert x.dtype == torch.float32 and x.stride(1) == 1
    assert alpha.shape == beta.shape == (C,) and alpha.dtype == beta.dtype == torch.float32
    out = torch.empty((rows, C), device=x.device, dtype=out_dtype)
    _ops._call("tfimm_b200_affine", dev, x.data_ptr(), x.stride(0), alpha.data_ptr(), beta.data_ptr(), out.data_ptr(),
               _ops._code(out), out.stride(0), rows, C, nbytes=_ops._nbytes(x, out))
    return out
