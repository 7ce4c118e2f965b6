"""GPU kernel numerics: every CUDA kernel against a plain PyTorch fp32 statement of the same op.

All calls go through the C ABI (ctypes -> libtfimm_b200.so).  Tolerances are written next to
each comparison: bf16 kernels are compared with fp32 references computed from the SAME
bf16-rounded inputs, so the only differences are accumulation order and output rounding.
"""
import math

import pytest
import torch

from oracle.shadow import faithful

pytestmark = pytest.mark.gpu


def _ops():
    from tfimm.backend import ops

    return ops


def _act_ref(x, act):
    if act in (None, "linear"):
        return x
    if act == "gelu":
        return torch.nn.functional.gelu(x)  # exact erf
    if act == "swish":
        return x * torch.sigmoid(x)
    if act == "relu":
        return torch.relu(x)
    if act == "relu6":
        return torch.clamp(x, 0, 6)
    if act == "tanh":
        return torch.tanh(x)
    if act == "sigmoid":
        return torch.sigmoid(x)
    raise ValueError(act)


GEMM_SHAPES = [
    # M, N, K
    (128, 256, 64),
    (128, 256, 768),
    (256, 768, 768),
    (394, 2304, 768),     # M tail, several N tiles
    (1000, 1000, 1024),   # N tail (classifier head), M tail
    (50432 // 8, 3072, 768),
    (640, 24, 48),        # EfficientNet-like tiny N / K tail
    (512, 56, 336),
    (300, 384, 128),
    (77, 1000, 192),
]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_gemm_bf16_plain(M, N, K, out_dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    out = ops.gemm(a, w, bias=bias, out_dtype=out_dtype)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias
    err = (out.float() - ref).abs().max().item()
    # fp32 out: accumulation-order noise only; bf16 out: one rounding (2^-9 relative)
    tol = 2e-3 if out_dtype == torch.float32 else 2e-2 + 4e-3 * ref.abs().max().item()
    assert err < tol, (err, tol)


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 768, 768), (394, 2304, 768), (1000, 1000, 1024),
                                   (50432 // 4, 768, 3072), (300, 384, 128), (77, 1000, 192), (4736, 3072, 768)])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_gemm_bf16_256_wide_tile(M, N, K, out_dtype):
    """block_n=2 (an alias of block_n=256) forces the 256-wide tile: M/N tails, many tiles per grid (smem-ring and
    mbarrier-phase wrap-around), residual in place."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g).to(out_dtype)
    ref = x.float() + torch.nn.functional.gelu(a.float() @ w.float().t() + bias)
    ops.gemm(a, w, bias=bias, act="gelu", residual=x, out=x, block_n=2)
    torch.cuda.synchronize()
    err = (x.float() - ref).abs().max().item()
    tol = 3e-3 if out_dtype == torch.float32 else 2e-2 + 4e-3 * ref.abs().max().item()
    assert err < tol, (err, tol)


@pytest.mark.parametrize("block_n", [64, 128, 256, 2])
@pytest.mark.parametrize("act", [None, "gelu", "swish", "relu", "relu6", "tanh", "sigmoid"])
def test_gemm_bf16_epilogues(block_n, act):
    ops = _ops()
    M, N, K = 777, 520, 264
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    out = ops.gemm(a, w, bias=bias, act=act, gamma=gamma, residual=res, out_dtype=torch.float32, block_n=block_n)
    torch.cuda.synchronize()
    ref = res + gamma * _act_ref(a.float() @ w.float().t() + bias, act)
    err = (out - ref).abs().max().item()
    assert err < 2e-3, err


def test_gemm_bf16_inplace_residual_bf16():
    ops = _ops()
    M, N, K = 1024, 768, 3072
    g = torch.Generator(device="cuda").manual_seed(2)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    ref = x.float() + a.float() @ w.float().t() + bias
    ops.gemm(a, w, bias=bias, residual=x, out=x)
    torch.cuda.synchronize()
    err = (x.float() - ref).abs().max().item()
    assert err < 2e-2 + 4e-3 * ref.abs().max().item(), err


def test_gemm_bf16_strided_a():
    """A given as a row-strided view (e.g. token 0 of every image)."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    full = torch.randn(64, 5, 256, device="cuda", generator=g).to(torch.bfloat16)
    a = full[:, 0, :]
    w = (torch.randn(100, 256, device="cuda", generator=g) / 16).to(torch.bfloat16)
    out = ops.gemm(a, w, out_dtype=torch.float32)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t()
    assert (out - ref).abs().max().item() < 1e-3


@pytest.mark.parametrize("act", [None, "gelu", "swish"])
def test_gemm_f32(act):
    ops = _ops()
    M, N, K = 300, 200, 136
    g = torch.Generator(device="cuda").manual_seed(4)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    out = ops.gemm(a, w, bias=bias, act=act, gamma=gamma, residual=res)
    torch.cuda.synchronize()
    ref = res + gamma * _act_ref((a.double() @ w.double().t()).float() + bias, act)
    assert (out - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize("C", [32, 192, 768, 1024, 4096])
@pytest.mark.parametrize("in_dtype,out_dtype", [(torch.float32, torch.bfloat16), (torch.bfloat16, torch.bfloat16),
                                                (torch.float32, torch.float32)])
def test_layernorm(C, in_dtype, out_dtype):
    ops = _ops()
    rows = 1003
    g = torch.Generator(device="cuda").manual_seed(C)
    x = (torch.randn(rows, C, device="cuda", generator=g) * 3 + 1.5).to(in_dtype)
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    out = ops.layernorm(x, gamma, beta, 1e-6, out_dtype)
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x.float(), (C,), gamma, beta, 1e-6)
    # bf16 output: one rounding, 2^-9 relative to the element's magnitude
    tol = 1e-4 if out_dtype == torch.float32 else 2.0 ** -8 * ref.abs().max().item() + 1e-3
    assert (out.float() - ref).abs().max().item() < tol


def test_layernorm_strided_rows():
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(16, 197, 768, device="cuda", generator=g)
    gamma = torch.randn(768, device="cuda", generator=g)
    beta = torch.randn(768, device="cuda", generator=g)
    out = ops.layernorm(x[:, 0, :], gamma, beta, 1e-6, torch.float32)
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x[:, 0, :], (768,), gamma, beta, 1e-6)
    assert (out - ref).abs().max().item() < 1e-4


def test_layernorm_patch2x2_and_patch_merge():
    ops = _ops()
    B, H, W, C = 3, 8, 12, 64
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(B, H, W, C, device="cuda", generator=g)
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    out = ops.layernorm_patch2x2(x, gamma, beta, 1e-6, torch.float32)
    ln = torch.nn.functional.layer_norm(x, (C,), gamma, beta, 1e-6)
    ref = ln.view(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * H // 2 * W // 2, 4 * C)
    torch.cuda.synchronize()
    assert (out - ref).abs().max().item() < 1e-4
    # Swin patch merging: (0,0),(1,0),(0,1),(1,1) then LN over 4C
    g4 = torch.randn(4 * C, device="cuda", generator=g)
    b4 = torch.randn(4 * C, device="cuda", generator=g)
    out = ops.patch_merge_ln(x, g4, b4, 1e-5, torch.float32)
    cat = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], dim=-1)
    ref = torch.nn.functional.layer_norm(cat, (4 * C,), g4, b4, 1e-5).reshape(-1, 4 * C)
    torch.cuda.synchronize()
    assert (out - ref).abs().max().item() < 1e-4


def _attn_ref(qkv, B, N, H, dh, scale, bias=None, mask=None):
    q, k, v = qkv.float().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    s = scale * q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias[None]
    if mask is not None:
        nm = mask.shape[0]
        s = (s.view(B // nm, nm, H, N, N) + mask[None, :, None]).view(B, H, N, N)
    p = torch.softmax(s, dim=-1)
    o = (p @ v).permute(0, 2, 1, 3).reshape(B * N, H * dh)
    return o, p


@pytest.mark.parametrize("B,N,H,nq", [(3, 197, 12, 1), (2, 198, 3, 2), (5, 50, 6, 1), (1, 512, 2, 2)])
def test_attention_cls_rows_equal_full_attention(B, N, H, nq):
    ops = _ops()
    dh = 64
    g = torch.Generator(device="cuda").manual_seed(N + nq)
    qkv = (torch.randn(B * N, 3 * H * dh, device="cuda", generator=g) * 1.5).to(torch.bfloat16)
    out = ops.attention_cls(qkv, B, N, H, dh, dh ** -0.5, nq)
    torch.cuda.synchronize()
    ref, _ = _attn_ref(qkv, B, N, H, dh, dh ** -0.5)
    ref = ref.view(B, N, H * dh)[:, :nq].reshape(B * nq, H * dh)
    assert out.shape == ref.shape
    assert (out.float() - ref).abs().max().item() < 1.5e-2   # fp32 math, one bf16 output rounding


@pytest.mark.parametrize("B,N,H", [(2, 197, 12), (3, 5, 2), (1, 65, 3), (2, 128, 4), (1, 224, 2), (1, 577, 2), (2, 17, 1),
                                   (3, 198, 3), (2, 50, 12), (1, 193, 2), (1, 208, 2), (2, 200, 5), (1, 64, 2), (1, 49, 1),
                                   (300, 197, 3), (1, 785, 2)])
def test_attention_bf16(B, N, H):
    ops = _ops()
    dh = 64
    g = torch.Generator(device="cuda").manual_seed(N)
    qkv = (torch.randn(B * N, 3 * H * dh, device="cuda", generator=g) * 1.5).to(torch.bfloat16)
    out = ops.attention(qkv, B, N, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    ref, _ = _attn_ref(qkv, B, N, H, dh, dh ** -0.5)
    err = (out.float() - ref).abs().max().item()
    assert err < 3e-2, err   # P is rounded to bf16 before the PV product; output rounded to bf16
    if N <= 256:
        # vs the emulation that rounds P with the global row max: at these lengths the kernel's per-64-key-block
        # rounding of P in its online softmax stays within the output rounding (2^-9 relative) of it.  Longer
        # sequences are only held to the bound above.
        from oracle import emulate_bf16
        emu = emulate_bf16.attention(qkv, B, N, H, dh, dh ** -0.5).float()
        assert (out.float() - emu).abs().max().item() < 2.0 ** -8 * emu.abs().max().item() + 1e-6


def test_attention_f32_with_bias_mask_probs():
    ops = _ops()
    B, N, H, dh = 8, 49, 4, 32
    g = torch.Generator(device="cuda").manual_seed(9)
    qkv = torch.randn(B * N, 3 * H * dh, device="cuda", generator=g)
    bias = torch.randn(H, N, N, device="cuda", generator=g)
    mask = torch.where(torch.rand(4, N, N, device="cuda", generator=g) > 0.7, -100.0, 0.0)
    probs = torch.empty(B, H, N, N, device="cuda")
    out = ops.attention(qkv, B, N, H, dh, dh ** -0.5, bias=bias, mask=mask, probs=probs)
    torch.cuda.synchronize()
    ref, p = _attn_ref(qkv, B, N, H, dh, dh ** -0.5, bias, mask)
    assert (out - ref).abs().max().item() < 2e-5
    assert (probs - p).abs().max().item() < 2e-6


@pytest.mark.parametrize("p,C,H,W", [(16, 3, 224, 224), (4, 3, 64, 96), (2, 3, 32, 32), (2, 64, 8, 8), (8, 1, 32, 32)])
@pytest.mark.parametrize("in_dtype", [torch.float32, torch.uint8])
def test_patchify(p, C, H, W, in_dtype):
    ops = _ops()
    B = 2
    g = torch.Generator(device="cuda").manual_seed(p * C)
    if in_dtype == torch.uint8:
        img = torch.randint(0, 256, (B, H, W, C), device="cuda", generator=g, dtype=torch.uint8)
        mean = torch.tensor([0.485, 0.456, 0.406] * 22, device="cuda")[:C].contiguous()
        std = torch.tensor([0.229, 0.224, 0.225] * 22, device="cuda")[:C].contiguous()
        out = ops.patchify(img, p, torch.float32, mean=mean, inv_std=1.0 / std, scale=1.0 / 255.0)
        imgf = (img.float() / 255.0 - mean) / std
    else:
        img = torch.randn(B, H, W, C, device="cuda", generator=g)
        out = ops.patchify(img, p, torch.float32)
        imgf = img
    torch.cuda.synchronize()
    K = p * p * C
    ref = imgf.view(B, H // p, p, W // p, p, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, K)
    assert out.shape[1] == (K + 7) // 8 * 8
    assert (out[:, :K] - ref).abs().max().item() < 1e-5
    assert out[:, K:].abs().max().item() == 0 if out.shape[1] > K else True


def test_assemble_tokens():
    ops = _ops()
    B, P, D = 3, 16, 64
    g = torch.Generator(device="cuda").manual_seed(11)
    patches = torch.randn(B * P, D, device="cuda", generator=g).to(torch.bfloat16)
    cls = torch.randn(D, device="cuda", generator=g)
    dist = torch.randn(D, device="cuda", generator=g)
    for d, ntok in ((None, 1), (dist, 2)):
        pos = torch.randn(P + ntok, D, device="cuda", generator=g)
        out = ops.assemble_tokens(patches, cls, d, pos, B, P, torch.float32)
        torch.cuda.synchronize()
        toks = [cls[None, None].expand(B, 1, D)] + ([d[None, None].expand(B, 1, D)] if d is not None else [])
        ref = torch.cat(toks + [patches.float().view(B, P, D)], dim=1) + pos[None]
        assert (out.view(B, P + ntok, D) - ref).abs().max().item() < 1e-6


@pytest.mark.parametrize("C,H,W", [(128, 56, 56), (256, 28, 28), (512, 14, 14), (1024, 7, 7), (96, 9, 13), (192, 5, 3),
                                   (192, 28, 28), (384, 14, 14), (768, 7, 7), (768, 14, 14), (1024, 14, 14),
                                   (512, 16, 9), (256, 15, 8), (128, 3, 20), (64, 14, 14), (1536, 7, 7)])
@pytest.mark.parametrize("in_dtype,out_dtype", [(torch.float32, torch.bfloat16), (torch.float32, torch.float32),
                                                (torch.bfloat16, torch.bfloat16)])
def test_dwconv7x7_ln(C, H, W, in_dtype, out_dtype):
    _check_dwconv7x7_ln(C, H, W, in_dtype, out_dtype, B=2)


@pytest.mark.parametrize("C,H,W,B", [(512, 14, 14, 48), (1024, 7, 7, 64), (128, 28, 28, 24), (96, 14, 14, 40)])
def test_dwconv7x7_ln_many_tiles(C, H, W, B):
    # more tiles than co-resident clusters: the persistent clusters loop, re-using halo / stash / mbarrier phases
    _check_dwconv7x7_ln(C, H, W, torch.float32, torch.bfloat16, B=B)


def _check_dwconv7x7_ln(C, H, W, in_dtype, out_dtype, B):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(C + H)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).to(in_dtype)
    wgt = torch.randn(49, C, device="cuda", generator=g) / 7
    bias = torch.randn(C, device="cuda", generator=g)
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    out = ops.dwconv_ln(x, wgt, bias, gamma, beta, 1e-6, out_dtype)
    torch.cuda.synchronize()
    wt = wgt.view(7, 7, C).permute(2, 0, 1)[:, None]  # (C,1,7,7)
    y = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt, bias, padding=3, groups=C).permute(0, 2, 3, 1)
    ref = torch.nn.functional.layer_norm(y, (C,), gamma, beta, 1e-6).reshape(-1, C)
    # bf16 out: one output rounding (the tensor-memory kernel keeps fp32 up to there; the cluster / generic fallbacks
    # stage through fp16 / bf16)
    tol = 2e-4 if out_dtype == torch.float32 else 2.0 ** -7 * ref.abs().max().item() + 1e-3
    if out_dtype == torch.bfloat16 and in_dtype == torch.float32 and C % 64 == 0 and C // 64 in (2, 3, 4, 6, 8, 12, 16):
        # exact fp32 arithmetic: the result must round to the same bf16 value as the fp64 reference almost everywhere
        y64 = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=3,
                                         groups=C).permute(0, 2, 3, 1)
        r64 = torch.nn.functional.layer_norm(y64, (C,), gamma.double(), beta.double(), 1e-6).reshape(-1, C)
        flips = (out != r64.to(torch.bfloat16)).float().mean().item()
        assert flips < 2e-3, flips
    assert (out.float() - ref).abs().max().item() < tol


@pytest.mark.parametrize("ks,stride,padding", [(3, 1, "same"), (3, 2, "same"), (5, 1, "same"), (5, 2, "same"),
                                               (3, 2, "symmetric"), (5, 2, "symmetric"), (3, 1, "valid")])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("H,W", [(19, 23), (12, 12), (40, 70), (24, 24)])   # every tile shape of the TMA kernel
def test_dwconv_bias_act_and_pool(ks, stride, padding, dtype, H, W):
    ops = _ops()
    B, C = 2, 136
    g = torch.Generator(device="cuda").manual_seed(ks * 10 + stride)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).to(dtype)
    wgt = torch.randn(ks * ks, C, device="cuda", generator=g) / ks
    bias = torch.randn(C, device="cuda", generator=g)
    pool = torch.zeros(B, C, device="cuda")
    out = ops.dwconv_bias_act(x, wgt, bias, ks, stride, padding, act="swish", pool_sum=pool)
    torch.cuda.synchronize()
    xin = x.float().permute(0, 3, 1, 2)
    if padding == "same":
        oh, pt = ops.same_pad(H, ks, stride)
        ow, pl = ops.same_pad(W, ks, stride)
        tot_h = max((oh - 1) * stride + ks - H, 0)
        tot_w = max((ow - 1) * stride + ks - W, 0)
        xin = torch.nn.functional.pad(xin, (pl, tot_w - pl, pt, tot_h - pt))
    elif padding == "symmetric":
        pd = ((stride - 1) + (ks - 1)) // 2
        xin = torch.nn.functional.pad(xin, (pd, pd, pd, pd))
    wt = wgt.view(ks, ks, C).permute(2, 0, 1)[:, None]
    y = torch.nn.functional.conv2d(xin, wt, bias, stride=stride, groups=C)
    ref = (y * torch.sigmoid(y)).permute(0, 2, 3, 1)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    tol = 1e-4 if dtype == torch.float32 else 2.0 ** -8 * ref.abs().max().item() + 1e-3
    assert (out.float() - ref).abs().max().item() < tol
    pref = out.float().sum(dim=(1, 2))
    assert (pool - pref).abs().max().item() < 1e-2 * max(1.0, pref.abs().max().item())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_global_avg_pool(dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(21)
    x = torch.randn(5, 7, 7, 1000, device="cuda", generator=g).to(dtype)
    out = ops.global_avg_pool(x)
    torch.cuda.synchronize()
    assert (out - x.float().mean(dim=(1, 2))).abs().max().item() < 1e-5


@pytest.mark.parametrize("h,w,ws,shift,H", [(14, 14, 7, 3, 4), (14, 14, 7, 0, 4), (28, 21, 7, 3, 2), (8, 8, 4, 2, 3), (7, 7, 7, 0, 8),
                                            (24, 24, 12, 6, 4), (24, 12, 12, 0, 2), (16, 16, 8, 4, 3), (20, 10, 10, 5, 2)])
def test_window_attention_bf16(h, w, ws, shift, H):
    """Index-folded shifted-window attention vs explicit roll / partition / mask in torch."""
    from tfimm.architectures.swin import window_tables

    ops = _ops()
    B, dh = 5, 32
    n, nw, C = ws * ws, (h // ws) * (w // ws), H * 32
    g = torch.Generator(device="cuda").manual_seed(h * w + shift)
    qkv = (torch.randn(B * h * w, 3 * C, device="cuda", generator=g) * 1.2).to(torch.bfloat16)
    bias = torch.randn(H, n, n, device="cuda", generator=g)
    row_map, labels = window_tables(h, w, ws, shift)
    rm = torch.from_numpy(row_map).cuda()
    lab = torch.from_numpy(labels).cuda() if labels is not None else None
    out = ops.window_attention(qkv, bias, rm, lab, B, nw, n, H, dh, dh ** -0.5)
    torch.cuda.synchronize()
    # reference: explicit data movement
    x = qkv.float().view(B, h, w, 3 * C)
    xs = torch.roll(x, (-shift, -shift), (1, 2))
    xw = xs.view(B, h // ws, ws, w // ws, ws, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(B * nw, n, 3 * C)
    mask = None
    if labels is not None:
        lb = torch.from_numpy(labels).cuda().view(nw, n)
        mask = torch.where(lb[:, None, :] != lb[:, :, None], -100.0, 0.0)
    ow, _ = _attn_ref(xw.reshape(B * nw * n, 3 * C), B * nw, n, H, dh, dh ** -0.5, bias, mask)
    ow = ow.view(B, h // ws, w // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, h, w, C)
    ref = torch.roll(ow, (shift, shift), (1, 2)).reshape(B * h * w, C)
    err = (out.float() - ref).abs().max().item()
    assert err < 3e-2, err
    # padded-table entry point: padded bias table + per-row 64-bit region masks
    if n <= 52:
        bias_pad = torch.zeros(H, 64, 64, device="cuda")
        bias_pad[:, :n, :n] = bias
        bits = None
        if labels is not None:
            lb = torch.from_numpy(labels).view(nw, n)
            diff = (lb[:, :, None] != lb[:, None, :]).to(torch.int64)
            packed = (diff << torch.arange(n, dtype=torch.int64)[None, None, :]).sum(dim=-1)
            bits = torch.zeros(nw, 64, dtype=torch.int64)
            bits[:, :n] = packed
            bits = bits.cuda()
        for Bt in (B, 1, 5):   # odd window counts: the last item holds a single window
            q2 = qkv[: Bt * h * w]
            out_tc = ops.window_attention_tc(q2, bias_pad, rm, bits, Bt, nw, n, H, dh, dh ** -0.5)
            torch.cuda.synchronize()
            err_tc = (out_tc.float() - ref[: Bt * h * w]).abs().max().item() if Bt <= B else 0.0
            assert err_tc < 3e-2, (Bt, err_tc)
            from oracle import emulate_bf16
            emu = emulate_bf16.window_attention_tc(q2, bias_pad, rm, bits, Bt, nw, n, H, dh, dh ** -0.5).float()
            assert (out_tc.float() - emu).abs().max().item() < 2.0 ** -7 * emu.abs().max().item() + 1e-6
    # fp32 kernel with the same row map
    out32 = ops.attention(qkv.float(), B * nw, n, H, dh, dh ** -0.5, bias=bias, mask=mask, row_map=rm, nw_img=nw)
    torch.cuda.synchronize()
    assert (out32 - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize("ks,stride,padding,C", [(3, 2, "same", 3), (3, 1, 1, 16), (7, 2, 3, 3), (1, 2, 0, 64), (3, 2, "symmetric", 24),
                                                 (7, 2, 3, 6), (7, 2, 3, 1), (3, 2, 1, 6), (7, 2, 3, 5)])
def test_im2col_gemm_equals_conv(ks, stride, padding, C):
    ops = _ops()
    B, H, W, Cout = 2, 21, 18, 40
    g = torch.Generator(device="cuda").manual_seed(ks * 7 + C)
    x = torch.randn(B, H, W, C, device="cuda", generator=g)
    w = torch.randn(ks, ks, C, Cout, device="cuda", generator=g) / (ks * C ** 0.5)
    cols, Ho, Wo = ops.im2col(x, ks, stride, padding, torch.float32)
    K = ks * ks * C
    w2 = torch.zeros(Cout, cols.shape[1], device="cuda")
    w2[:, :K] = w.reshape(K, Cout).t()
    out = ops.gemm(cols, w2.contiguous()).view(B, Ho, Wo, Cout)
    torch.cuda.synchronize()
    _, _, pt, pl = ops.conv_geometry(H, W, ks, stride, padding)
    tot_h, tot_w = max((Ho - 1) * stride + ks - H, 0), max((Wo - 1) * stride + ks - W, 0)
    xin = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (pl, max(tot_w - pl, 0), pt, max(tot_h - pt, 0)))
    ref = torch.nn.functional.conv2d(xin, w.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    assert (out - ref).abs().max().item() < 1e-4


@pytest.mark.parametrize("in_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B,H,W", [(2, 37, 45), (1, 224, 224), (3, 64, 33)])
def test_im2col_rgb_stem_bf16_is_exact(B, H, W, in_dtype):
    """7x7 / stride-2 / pad-3 im2col of an RGB image into bf16 (the tiled shared-memory stem kernel): a pure gather,
    so it must equal torch's unfold of the bf16-rounded input bit for bit, in TF's (ky, kx, c) column order."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(H + W)
    x = torch.randn(B, H, W, 3, device="cuda", generator=g).to(in_dtype)
    cols, Ho, Wo = ops.im2col(x, 7, 2, 3, torch.bfloat16)
    torch.cuda.synchronize()
    assert (Ho, Wo) == ((H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1) and cols.shape == (B * Ho * Wo, 152)
    xb = x.to(torch.bfloat16).float().permute(0, 3, 1, 2)                       # (B, 3, H, W)
    ref = torch.nn.functional.unfold(xb, 7, padding=3, stride=2)                  # (B, 3*49, L), rows ordered (c, ky, kx)
    ref = ref.view(B, 3, 49, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 147)  # -> (m, (ky, kx), c)
    assert torch.equal(cols[:, :147].float(), ref)
    assert (cols[:, 147:] == 0).all()


def test_se_gate_scale_and_eca():
    ops = _ops()
    B, H, W, C, rd = 3, 5, 7, 48, 6
    g = torch.Generator(device="cuda").manual_seed(33)
    x = torch.randn(B, H, W, C, device="cuda", generator=g)
    wr = torch.randn(rd, C, device="cuda", generator=g) / C ** 0.5
    br = torch.randn(rd, device="cuda", generator=g)
    we = torch.randn(C, rd, device="cuda", generator=g) / rd ** 0.5
    be = torch.randn(C, device="cuda", generator=g)
    pooled_sum = x.sum(dim=(1, 2)).contiguous()
    gate = ops.se_gate(pooled_sum, H * W, wr, br, we.t().contiguous(), be, act="swish")  # expand weights as [rd][C]
    torch.cuda.synchronize()
    m = x.mean(dim=(1, 2))
    hdn = m @ wr.t() + br
    ref = torch.sigmoid((hdn * torch.sigmoid(hdn)) @ we.t() + be)
    assert (gate - ref).abs().max().item() < 1e-5
    y = x.clone()
    ops.scale_channels_(y, gate)
    assert (y - x * ref[:, None, None, :]).abs().max().item() < 1e-5
    wk = torch.randn(5, device="cuda", generator=g)
    eg = ops.eca_gate(m.contiguous(), wk)
    eref = torch.sigmoid(torch.nn.functional.conv1d(torch.nn.functional.pad(m, (2, 2))[:, None], wk[None, None])[:, 0])
    assert (eg - eref).abs().max().item() < 1e-5
    sc = torch.randn(B, H, W, C, device="cuda", generator=g)
    z = x.clone()
    ops.scale_add_act_(z, ref.contiguous(), sc, "relu")
    torch.cuda.synchronize()
    assert (z - torch.relu(x * ref[:, None, None, :] + sc)).abs().max().item() < 1e-5


def test_pool2d_modes():
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(34)
    x = torch.randn(2, 9, 11, 16, device="cuda", generator=g) - 1.0  # mostly negative: zero padding matters
    out = ops.pool2d(x, 3, 2, 1, "max_zero_pad")
    ref = torch.nn.functional.max_pool2d(torch.nn.functional.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1)), 3, 2).permute(0, 2, 3, 1)
    assert (out - ref).abs().max().item() == 0
    out = ops.pool2d(x, 2, 2, "same", "avg")
    xp = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (0, 1, 0, 1))
    ones = torch.nn.functional.pad(torch.ones_like(x.permute(0, 3, 1, 2)), (0, 1, 0, 1))
    ref = (torch.nn.functional.avg_pool2d(xp, 2, 2) / torch.nn.functional.avg_pool2d(ones, 2, 2)).permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    assert (out - ref).abs().max().item() < 1e-6


@pytest.mark.parametrize("cg,stride", [(4, 1), (8, 2), (16, 1), (32, 2)])
def test_grouped_conv(cg, stride):
    ops = _ops()
    B, H, W, groups = 2, 10, 9, 4
    C = cg * groups
    g = torch.Generator(device="cuda").manual_seed(cg)
    x = torch.randn(B, H, W, C, device="cuda", generator=g)
    w = torch.randn(3, 3, cg, C, device="cuda", generator=g) / (3 * cg ** 0.5)
    bias = torch.randn(C, device="cuda", generator=g)
    out = ops.grouped_conv(x, w.reshape(9, cg, C).contiguous(), bias, cg, 3, stride, 1, act="relu")
    torch.cuda.synchronize()
    ref = torch.relu(torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), bias, stride=stride,
                                                padding=1, groups=groups)).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    assert (out - ref).abs().max().item() < 1e-4


def test_gemm_act_after_residual():
    ops = _ops()
    M, N, K = 300, 136, 72
    g = torch.Generator(device="cuda").manual_seed(35)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    out = ops.gemm(a, w, bias=bias, act="relu", residual=res, act_after_residual=True)
    torch.cuda.synchronize()
    ref = torch.relu(a.float() @ w.float().t() + bias + res.float())
    assert (out.float() - ref).abs().max().item() < 2e-2 + 4e-3 * ref.abs().max().item()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C,groups", [(64, 32), (256, 32), (2048, 32), (64, 1)])
def test_group_norm_with_residual_and_act(C, groups, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(C + groups)
    x = (torch.randn(3, 7, 9, C, device="cuda", generator=g) * 2 + 0.5).to(dtype)
    res = torch.randn(3, 7, 9, C, device="cuda", generator=g).to(dtype)
    gamma, beta = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)
    out = ops.group_norm(x, gamma, beta, groups, 1e-5, act="relu", residual=res)
    torch.cuda.synchronize()
    ref = torch.nn.functional.group_norm(x.float().permute(0, 3, 1, 2), groups, gamma, beta, 1e-5).permute(0, 2, 3, 1)
    ref = torch.relu(ref + res.float())
    tol = 2e-5 if dtype == torch.float32 else 2.0 ** -8 * ref.abs().max().item() + 1e-3
    assert (out.float() - ref).abs().max().item() < tol


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("H,W,stride", [(8, 8, 2), (7, 9, 2), (5, 4, 1)])
def test_blur_pool_reflect(H, W, stride, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(H * W)
    x = torch.randn(2, H, W, 24, device="cuda", generator=g).to(dtype)
    out = ops.blur_pool(x, stride)
    torch.cuda.synchronize()
    xc = torch.nn.functional.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1), mode="reflect")
    k1 = torch.tensor([1.0, 2.0, 1.0], device="cuda")
    k = (k1[:, None] * k1[None, :] / 16)[None, None].repeat(24, 1, 1, 1)
    ref = torch.nn.functional.conv2d(xc, k, stride=stride, groups=24).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    assert (out.float() - ref).abs().max().item() < (1e-5 if dtype == torch.float32 else 2e-2)


@pytest.mark.parametrize("cg,stride", [(64, 1), (48, 2), (24, 1)])
def test_grouped_im2col_and_per_group_gemm_equal_grouped_conv(cg, stride):
    ops = _ops()
    G, B, H, W = 4, 2, 9, 11
    C = G * cg
    g = torch.Generator(device="cuda").manual_seed(cg)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(3, 3, cg, C, device="cuda", generator=g) / (3 * cg ** 0.5)          # TF layout (kh, kw, cin/G, cout)
    cols, Ho, Wo = ops.im2col(x, 3, stride, 1, torch.bfloat16, groups=G)
    assert cols.shape[0] == G and cols.shape[1] == B * Ho * Wo
    wg = w.reshape(9 * cg, G, cg).permute(1, 2, 0)
    wg = torch.nn.functional.pad(wg, (0, cols.shape[2] - 9 * cg)).to(torch.bfloat16).contiguous()
    out = torch.empty(B * Ho * Wo, C, device="cuda", dtype=torch.bfloat16)
    for i in range(G):
        ops.gemm(cols[i], wg[i], out=out[:, i * cg:(i + 1) * cg])
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.to(torch.bfloat16).float().permute(3, 2, 0, 1),
                                     stride=stride, padding=1, groups=G).permute(0, 2, 3, 1).reshape(-1, C)
    assert (out.float() - ref).abs().max().item() < 2e-2 + 4e-3 * ref.abs().max().item()


@pytest.mark.parametrize("B,H,W,C,N,ks,stride", [
    (3, 14, 14, 64, 64, 3, 1),       # one 8x16 patch row is partial in both directions
    (2, 56, 56, 64, 64, 3, 1),       # ResNet stage 1
    (2, 56, 56, 128, 128, 3, 2),     # strided: TMA traversal stride 2
    (3, 7, 7, 512, 512, 3, 1),       # 8x8 patches of two images per tile, odd batch (second image out of bounds)
    (5, 14, 14, 256, 320, 3, 2),     # -> 7x7, N tail over 256-wide tiles
    (2, 20, 33, 64, 72, 5, 1),       # other kernel size / odd sizes
])
@pytest.mark.parametrize("mode", ["plain", "residual"])
def test_implicit_gemm_conv(B, H, W, C, N, ks, stride, mode):
    """k x k convolution whose A tiles are 4-D TMA boxes of the NHWC input (zero padding = out-of-bounds fill)."""
    ops = _ops()
    pad = (ks - 1) // 2
    g = torch.Generator(device="cuda").manual_seed(H * 7 + C + stride)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(ks, ks, C, N, device="cuda", generator=g) / (ks * math.sqrt(C))).to(torch.bfloat16)  # TF layout
    bias = torch.randn(N, device="cuda", generator=g)
    w2 = w.reshape(ks * ks * C, N).t().contiguous()
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(3, 2, 0, 1), bias,
                                     stride=stride, padding=pad).permute(0, 2, 3, 1)
    if mode == "plain":
        out = ops.conv_gemm(x, w2, bias=bias, ks=ks, stride=stride, pad=pad, act="relu")
        ref = torch.relu(ref)
    else:
        res = torch.randn(ref.shape, device="cuda", generator=g)
        out = ops.conv_gemm(x, w2, bias=bias, ks=ks, stride=stride, pad=pad, act="relu", residual=res,
                            act_after_residual=True)
        ref = torch.relu(ref + res)
    torch.cuda.synchronize()
    assert out.shape == ref.shape
    tol = 3e-3 if out.dtype == torch.float32 else 2e-2 + 4e-3 * ref.abs().max().item()
    assert (out.float() - ref).abs().max().item() < tol



@pytest.mark.parametrize("act", ["gelu", "swish"])
@pytest.mark.parametrize("block_n", [2, 128])
def test_gemm_activation_epilogue_is_faithfully_rounded(act, block_n):
    """bf16 outputs of the fused GEMM + activation epilogue are the CORRECTLY ROUNDED exact values, or their bf16
    neighbour, and differ from the correct rounding on < 1 % of the elements: the accurate 4-element GELU / swish
    (common.cuh) are good to ~4e-6 before rounding.  (The tanh.approx forms of round 1 flipped 12 % / 25 %.)"""
    ops = _ops()
    M, N, K = 1024, 512, 128
    g = torch.Generator(device="cuda").manual_seed(3)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5 * 2.0).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    out = ops.gemm(a, w, bias=bias, act=act, block_n=block_n)
    torch.cuda.synchronize()
    y = a.double() @ w.double().t() + bias.double()
    ref = 0.5 * y * (1.0 + torch.erf(y / 2.0 ** 0.5)) if act == "gelu" else y * torch.sigmoid(y)
    flips, worst = faithful(out, ref)
    print(f"{act} block_n={block_n}: {100 * flips:.3f}% of the bf16 outputs (|y| >= 0.05) differ from the correct rounding, "
          f"worst error {worst:.3f} x max(bf16 spacing, 5e-6)")
    assert flips < 2e-2 and worst <= 1.0


def test_dwconv_swish_is_faithfully_rounded():
    ops = _ops()
    B, H, W, C = 2, 24, 32, 128
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(B, H, W, C, device="cuda", generator=g).to(torch.bfloat16)
    wgt = torch.randn(9, C, device="cuda", generator=g) / 3
    bias = torch.randn(C, device="cuda", generator=g)
    out = ops.dwconv_bias_act(x, wgt, bias, 3, 1, "same", act="swish")
    torch.cuda.synchronize()
    wt = wgt.double().view(3, 3, C).permute(2, 0, 1)[:, None]
    y = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt, bias.double(), padding=1, groups=C).permute(0, 2, 3, 1)
    ref = y * torch.sigmoid(y)
    flips, worst = faithful(out, ref)
    print(f"dwconv swish: {100 * flips:.3f}% flips, worst {worst:.3f} x max(bf16 spacing, 5e-6)")
    assert flips < 2e-2 and worst <= 1.0


@pytest.mark.parametrize("M,K,N", [(9000, 24, 144), (5000, 32, 192), (4096, 64, 512), (4100, 48, 24), (70001, 56, 336),
                                   (4097, 8, 8), (6000, 40, 72)])
@pytest.mark.parametrize("act", [None, "swish", "gelu", "relu6"])
def test_gemm_short_contraction_streaming_kernel(M, K, N, act):
    """K <= 64, bf16 out, no residual: the mma.sync streaming kernel (gemm_skinny.cu) behind the same entry point."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M + K + N)
    a_full = torch.randn(M, K + 8, device="cuda", generator=g).to(torch.bfloat16)
    a = a_full[:, :K]                                   # row stride != K: lda is honoured
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    out = ops.gemm(a, w, bias=bias, act=act)
    torch.cuda.synchronize()
    from oracle import emulate_bf16
    ref = emulate_bf16.gemm(a, w, bias=bias, act=act).float()
    assert out.shape == (M, N) and out.dtype == torch.bfloat16
    assert (out.float() - ref).abs().max().item() <= 2.0 ** -7 * ref.abs().max().item() + 1e-5
    assert (out != ref.to(torch.bfloat16)).float().mean().item() < 2e-2
    # the wgmma path gives the same numbers (forced through block_n)
    out2 = ops.gemm(a, w, bias=bias, act=act, block_n=64)
    assert (out.float() - out2.float()).abs().max().item() <= 2.0 ** -7 * ref.abs().max().item() + 1e-5
    # bf16 residual, also in place
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    ref_r = emulate_bf16.gemm(a, w, bias=bias, act=act, residual=res).float()
    out_r = ops.gemm(a, w, bias=bias, act=act, residual=res)
    buf = res.clone()
    ops.gemm(a, w, bias=bias, act=act, residual=buf, out=buf)
    torch.cuda.synchronize()
    assert (out_r.float() - ref_r).abs().max().item() <= 2.0 ** -7 * ref_r.abs().max().item() + 1e-5
    assert torch.equal(out_r, buf)


@pytest.mark.parametrize("M,C,mult", [(256, 128, 4), (1000, 128, 4), (37 * 256 + 13, 128, 4), (150 * 256, 128, 4),
                                      (512, 256, 4), (777, 256, 4), (90 * 256 + 5, 256, 4), (3000, 128, 2),
                                      (2048, 256, 3), (256, 96, 4), (75 * 256 + 77, 96, 4), (1000, 192, 4),
                                      (80 * 256 + 3, 192, 4), (1024, 192, 2)])
@pytest.mark.parametrize("act,with_gamma", [("gelu", True), ("gelu", False), ("swish", False)])
def test_mlp_fused_equals_two_gemms(M, C, mult, act, with_gamma):
    """fc1 -> act -> fc2 -> * gamma -> + residual in one kernel (csrc/mlp_sm90.cu): same rounding points as the
    two-GEMM form (bf16 hidden, fp32 accumulation in ascending k), so the two agree to fp32 summation noise."""
    ops = _ops()
    Hd = mult * C
    g = torch.Generator(device="cuda").manual_seed(M + C + Hd)
    a_full = torch.randn(M, C + 8, device="cuda", generator=g).to(torch.bfloat16)
    a = a_full[:, :C]                                   # lda != C
    w1 = (torch.randn(Hd, C, device="cuda", generator=g) / C ** 0.5).to(torch.bfloat16)
    w2 = (torch.randn(C, Hd, device="cuda", generator=g) / Hd ** 0.5).to(torch.bfloat16)
    b1 = torch.randn(Hd, device="cuda", generator=g)
    b2 = torch.randn(C, device="cuda", generator=g)
    gamma = torch.randn(C, device="cuda", generator=g) if with_gamma else None
    res = torch.randn(M, C, device="cuda", generator=g)
    out = ops.mlp_fused(a, w1, b1, w2, b2, act, gamma=gamma, residual=res)
    buf = res.clone()
    ops.mlp_fused(a, w1, b1, w2, b2, act, gamma=gamma, residual=buf, out=buf)     # in place
    plain = ops.mlp_fused(a, w1, b1, w2, b2, act, gamma=gamma)                    # no residual
    hid = ops.gemm(a, w1, bias=b1, act=act)
    two = ops.gemm(hid, w2, bias=b2, gamma=gamma, residual=res, out_dtype=torch.float32)
    torch.cuda.synchronize()
    from oracle import emulate_bf16
    ref = emulate_bf16.mlp_fused(a, w1, b1, w2, b2, act, gamma=gamma, residual=res).double()
    scale = ref.abs().max().item()
    assert out.shape == (M, C) and out.dtype == torch.float32
    assert torch.equal(out, buf)
    assert (plain.double() - (ref - res.double())).abs().max().item() <= 3e-3 * scale
    # against the two kernels: identical hidden roundings up to the rare flip caused by fp32 summation order
    assert (out - two).abs().max().item() <= 2e-3 * scale
    assert ((out - two).abs() > 1e-5 * scale).float().mean().item() < 5e-2
    # against exact arithmetic with the same storage points
    assert (out.double() - ref).abs().max().item() <= 3e-3 * scale
    assert (out.double() - ref).pow(2).mean().sqrt().item() <= 2e-4 * scale


def test_mlp_fused_rejects_other_shapes():
    ops = _ops()
    assert not ops.mlp_fused_supported(64, 256) and not ops.mlp_fused_supported(512, 2048)
    assert ops.mlp_fused_supported(96, 384) and ops.mlp_fused_supported(192, 768)
    assert ops.mlp_fused_supported(128, 512) and ops.mlp_fused_supported(256, 1024)
    a = torch.zeros(256, 512, device="cuda", dtype=torch.bfloat16)
    w1 = torch.zeros(2048, 512, device="cuda", dtype=torch.bfloat16)
    w2 = torch.zeros(512, 2048, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(Exception, match="mlp_fused"):
        ops.mlp_fused(a, w1, None, w2, None, "gelu")


@pytest.mark.parametrize("B,HW,K,N", [(3, 9025, 144, 32), (4, 2304, 192, 32), (2, 576, 336, 56), (5, 144, 1632, 272),
                                      (7, 130, 48, 24), (2, 100, 960, 160), (3, 36, 2688, 448), (3, 9025, 48, 24),
                                      (2, 36100, 32, 16), (5, 1000, 56, 336)])
@pytest.mark.parametrize("with_res", [False, True])
def test_gemm_gated_equals_scale_then_gemm(B, HW, K, N, with_res):
    """Squeeze-excite gate applied to the A tile in shared memory (wgmma kernel) or to the A fragments in registers
    (K <= 64: streaming kernel): the products scale_channels_ would have written, then the same GEMM."""
    ops = _ops()
    M = B * HW
    g = torch.Generator(device="cuda").manual_seed(B + HW + K + N)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    gate = torch.sigmoid(torch.randn(B, K, device="cuda", generator=g))
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16) if with_res else None
    out = ops.gemm_gated(a, gate, HW, w, bias=bias, residual=res)
    scaled = ops.scale_channels_(a.clone().view(B, HW, K), gate).view(M, K)
    want = ops.gemm(scaled, w, bias=bias, residual=res, block_n=64)
    torch.cuda.synchronize()
    from oracle import emulate_bf16
    ref = emulate_bf16.gemm_gated(a, gate, HW, w, bias=bias, residual=res).float()
    assert out.shape == (M, N) and out.dtype == torch.bfloat16
    assert (out.float() - ref).abs().max().item() <= 2.0 ** -7 * ref.abs().max().item() + 1e-5
    # same products, same k order: only the tile width (accumulation grouping inside the tensor core) may differ
    assert (out != want).float().mean().item() < 1e-2
    assert (out.float() - want.float()).abs().max().item() <= 2.0 ** -7 * ref.abs().max().item() + 1e-5


@pytest.mark.parametrize("C,ks,stride,padding,H,W", [(3, 7, 2, 3, 64, 80), (3, 3, 2, "same", 45, 38), (3, 3, 2, 1, 40, 40),
                                                     (1, 3, 2, "same", 33, 33), (6, 7, 2, 3, 32, 32), (8, 3, 1, 1, 20, 24)])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_im2col_uint8_fuses_preprocessing(C, ks, stride, padding, H, W, out_dtype):
    """Raw uint8 pixels: the gather applies (x / 255 - mean) / std per channel and keeps the padding at zero -- the same
    matrix as im2col of the preprocessed fp32 image."""
    ops = _ops()
    B = 3
    g = torch.Generator(device="cuda").manual_seed(C * 100 + ks)
    raw = torch.randint(0, 256, (B, H, W, C), device="cuda", generator=g, dtype=torch.uint8)
    mean = torch.rand(C, device="cuda", generator=g)
    inv_std = 1.0 / (0.2 + torch.rand(C, device="cuda", generator=g))
    cols, Ho, Wo = ops.im2col(raw, ks, stride, padding, out_dtype, pre=(mean, inv_std, 1.0 / 255.0))
    pre = ((raw.float() * (1.0 / 255.0) - mean) * inv_std).contiguous()
    want, Ho2, Wo2 = ops.im2col(pre, ks, stride, padding, out_dtype)
    torch.cuda.synchronize()
    assert (Ho, Wo) == (Ho2, Wo2) and cols.shape == want.shape
    if out_dtype == torch.bfloat16:
        assert (cols != want).float().mean().item() < 2e-3          # an fma contraction may flip a rare rounding
        assert (cols.float() - want.float()).abs().max().item() <= 2.0 ** -7 * want.float().abs().max().item()
    else:
        assert torch.allclose(cols, want, rtol=2e-6, atol=2e-6)     # x * scale - mean: fma in the kernel, two ops in torch
    assert torch.equal(cols == 0, want == 0)                        # the padding stays exactly zero
