"""The staged epilogue of the plain bf16 GEMM (64- and 128-wide tiles: residual in by TMA, result out by TMA through a
shared-memory tile) against the fragment epilogue, which the 256-wide tile keeps.

The tile width does not change an output element's fp32 sum, and both epilogues apply the same fp32 operations in the
same order, so every case must match the 256-wide result bit for bit (for bf16 output with N % 8 != 0, where the
staged epilogue does not apply, this checks that the fragment epilogue was chosen).  Each case also checks the float64 statement of
the op within the bounds of tests/test_kernels_gpu.py, and that nothing outside the output view changed: the output is
a column slice of a wider buffer with a padded row stride and rows past M, all filled with canaries.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

ACTS = [None, "gelu", "swish", "relu", "relu6", "tanh", "sigmoid"]
# M, N, K: M % 128 != 0 and N % 64, N % 128 != 0; M < 128 and N % 8 != 0.  A bf16 row of N = 100 does not end on a
# 16-byte boundary, where the TMA store would not clip it, so that shape checks that bf16 output keeps the fragment
# epilogue there (fp32 output, 400-byte rows, takes the staged one).
SHAPES = [(300, 200, 192), (77, 100, 256)]


def _ops():
    from tfimm.backend import ops

    return ops


def _act64(x, act):
    if act is None:
        return x
    return {"gelu": torch.nn.functional.gelu, "swish": lambda v: v * torch.sigmoid(v), "relu": torch.relu,
            "relu6": lambda v: torch.clamp(v, 0, 6), "tanh": torch.tanh, "sigmoid": torch.sigmoid}[act](x)


def _inputs(M, N, K, out_dtype, res_mode, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g)
    width = (N + 7) // 8 * 8 + 48   # padded row stride; the view starts 24 columns in (16-byte aligned)
    canvas = (torch.randn(M + 3, width, device="cuda", generator=g) * 100).to(out_dtype)
    res = None
    if res_mode == "separate":   # its own row stride, ldr != ldc
        res_full = torch.randn(M, width + 16, device="cuda", generator=g).to(out_dtype)
        res = res_full[:, 8:8 + N]
    elif res_mode == "inplace":
        canvas[:M, 24:24 + N] = torch.randn(M, N, device="cuda", generator=g).to(out_dtype)
    return a, w, bias, gamma, canvas, res


def _run(a, w, bias, gamma, canvas, res, res_mode, N, act, act_post, block_n):
    M = a.shape[0]
    buf = canvas.clone()
    out = buf[:M, 24:24 + N]
    residual = out if res_mode == "inplace" else res
    _ops().gemm(a, w, bias=bias, act=act, gamma=gamma, residual=residual, out=out, block_n=block_n,
                act_after_residual=act_post)
    return buf


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("res_mode", ["none", "separate", "inplace"])
@pytest.mark.parametrize("with_gamma", [False, True], ids=["nogamma", "gamma"])
@pytest.mark.parametrize("act_post", [False, True], ids=["act", "act_post"])
def test_staged_epilogue_matches_fragment_epilogue(M, N, K, block_n, out_dtype, res_mode, with_gamma, act_post):
    a, w, bias, gamma, canvas, res = _inputs(M, N, K, out_dtype, res_mode, seed=M * 7 + N * 3 + K + block_n)
    gamma = gamma if with_gamma else None
    for act in ACTS:
        got = _run(a, w, bias, gamma, canvas, res, res_mode, N, act, act_post, block_n)
        want = _run(a, w, bias, gamma, canvas, res, res_mode, N, act, act_post, 256)
        torch.cuda.synchronize()
        # bit for bit against the fragment epilogue, over the whole buffer (canaries included)
        assert torch.equal(got.view(torch.int16 if out_dtype == torch.bfloat16 else torch.int32),
                           want.view(torch.int16 if out_dtype == torch.bfloat16 else torch.int32)), act
        # nothing outside the output view changed
        outside = torch.ones_like(got, dtype=torch.bool)
        outside[:M, 24:24 + N] = False
        assert torch.equal(got[outside], canvas[outside]), act
        # the float64 statement
        y = a.double() @ w.double().t() + bias.double()
        r = (canvas[:M, 24:24 + N] if res_mode == "inplace" else res).double() if res_mode != "none" else 0.0
        s = gamma.double() if gamma is not None else 1.0
        ref = _act64(r + s * y, act) if act_post else r + s * _act64(y, act)
        err = (got[:M, 24:24 + N].double() - ref).abs().max().item()
        tol = 2e-3 if out_dtype == torch.float32 else 2e-2 + 4e-3 * ref.abs().max().item()
        assert err < tol, (act, err, tol)
