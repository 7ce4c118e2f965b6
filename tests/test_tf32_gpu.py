"""precision="tf32" on the H100: the TF32 kernels against the emulation (tests/tf32_oracle.py) within the op-by-op shadow
bounds, whole tf32 forwards launch by launch, the accuracy against the fp32 oracle, and the benchmark configurations
through ``model.cuda_graph``.  ``-s`` prints the measured numbers.
"""
from contextlib import contextmanager

import pytest
import torch

from test_op_shadow_gpu import _inputs
from test_parity_budget_gpu import BUDGET, FULL, SMALL, _model, _nerr, _rms
from tf32_oracle import round_tf32, tf32_oracle

pytestmark = pytest.mark.gpu


@contextmanager
def _tf32_mode():
    """The launchers' tf32 dispatch, as inside a tf32 model's forward pass."""
    from tfimm.backend import lib

    token = lib.tf32_mode.set(True)
    try:
        yield
    finally:
        lib.tf32_mode.reset(token)


@contextmanager
def _shadowed_tf32(kernels=None):
    """Shadowed launches in tf32 mode; ``kernels`` (a set) collects the C entry points that ran."""
    from oracle import shadow
    from tfimm.backend import ops

    call = ops._call

    def recording_call(name, *a, **k):
        if kernels is not None:
            kernels.add(name)
        return call(name, *a, **k)

    ops._call = recording_call
    try:
        with tf32_oracle(), _tf32_mode(), shadow.shadowed_ops() as census:
            yield census
    finally:
        ops._call = call


def _weights(N, K, gen):
    return round_tf32(torch.randn(N, K, generator=gen) * K ** -0.5).cuda()


# ------------------------------------------------------------------------------------------------------ rounding
@pytest.mark.parametrize("K", [64, 256])
def test_gemm_tf32_rounds_a_in_the_kernel(K):
    """W = identity: the output is A as the tensor core saw it, which must be cvt.rna(A) bit for bit -- values whose
    low 13 bits are set, an eighth of them exact ties (round-to-even or truncation would differ there)."""
    from tfimm.backend import ops

    gen = torch.Generator().manual_seed(K)
    M = 300
    a = torch.randn(M, K, generator=gen) * 4
    bits = a.view(torch.int32)
    low = torch.randint(1, 0x2000, (M, K), generator=gen, dtype=torch.int32)
    low = torch.where(torch.rand(M, K, generator=gen) < 0.125, torch.full_like(low, 0x1000), low)
    a = ((bits & ~0x1FFF) | low).view(torch.float32)
    assert bool((a.abs() > 2.0 ** -100).all())                        # normal range
    with _tf32_mode():
        out = ops.gemm(a.cuda(), torch.eye(K).cuda())
    want = round_tf32(a)
    assert not torch.equal(want, a)
    assert torch.equal(out.cpu(), want)


# ------------------------------------------------------------------------------------------------------------ GEMM
GEMM_SHAPES = [(1, 8, 8), (127, 72, 40), (129, 1000, 48), (129, 2304, 32), (127, 1000, 3072), (1, 72, 768),
               (129, 8, 3072), (50432, 2304, 768), (50432, 768, 3072)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES, ids=[f"{m}x{n}x{k}" for m, n, k in GEMM_SHAPES])
@pytest.mark.parametrize("block_n", [0, 64, 128])
def test_gemm_tf32_against_emulation(M, N, K, block_n):
    from tfimm.backend import ops

    if M == 50432 and block_n != 0:
        pytest.skip("ViT-B shapes: the chosen tile width only")
    gen = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=gen).cuda()
    w = _weights(N, K, gen)
    bias = torch.randn(N, generator=gen).cuda()
    kernels = set()
    with _shadowed_tf32(kernels) as census:
        ops.gemm(a, w, bias=bias, block_n=block_n)
    census.assert_ok()
    assert kernels == {"tfimm_b200_gemm_tf32"}


def test_gemm_tf32_strided_a():
    from tfimm.backend import ops

    gen = torch.Generator().manual_seed(5)
    big = torch.randn(257, 40 + 24, generator=gen).cuda()
    a = big[:, 8:48]                                                  # row stride 64, offset 32 bytes
    w = _weights(136, 40, gen)
    with _shadowed_tf32() as census:
        ops.gemm(a, w, act="gelu")
    census.assert_ok()


EPILOGUES = [
    ("bias_gelu", dict(bias=True, act="gelu")),
    ("swish", dict(act="swish")),
    ("tanh", dict(bias=True, act="tanh")),
    ("gamma_residual_in_place", dict(bias=True, gamma=True, residual=True, in_place=True)),
    ("relu_after_residual", dict(bias=True, act="relu", residual=True, act_after_residual=True)),
    ("gelu_after_residual_in_place", dict(act="gelu", residual=True, act_after_residual=True, in_place=True)),
]


@pytest.mark.parametrize("what,opts", EPILOGUES, ids=[e[0] for e in EPILOGUES])
@pytest.mark.parametrize("block_n", [64, 128])
def test_gemm_tf32_epilogues(what, opts, block_n):
    from tfimm.backend import ops

    gen = torch.Generator().manual_seed(11)
    M, N, K = 333, 200, 96
    a = torch.randn(M, K, generator=gen).cuda()
    w = _weights(N, K, gen)
    kw = dict(act=opts.get("act"), act_after_residual=opts.get("act_after_residual", False), block_n=block_n)
    if opts.get("bias"):
        kw["bias"] = torch.randn(N, generator=gen).cuda()
    if opts.get("gamma"):
        kw["gamma"] = (torch.rand(N, generator=gen) * 2).cuda()
    if opts.get("residual"):
        ldr = 208
        kw["residual"] = torch.randn(M, ldr, generator=gen).cuda()[:, :N]
        if opts.get("in_place"):
            kw["out"] = kw["residual"]
    with _shadowed_tf32() as census:
        out = ops.gemm(a, w, **kw)
    census.assert_ok()
    if opts.get("in_place"):
        assert out.data_ptr() == kw["residual"].data_ptr()


# ----------------------------------------------------------------------------------------------------- convolution
CONVS = [(1, 1, 32), (3, 1, 64), (3, 2, 64), (7, 2, 32), (3, 1, 256), (3, 2, 256), (1, 2, 64)]


@pytest.mark.parametrize("ks,stride,C", CONVS, ids=[f"k{k}s{s}c{c}" for k, s, c in CONVS])
@pytest.mark.parametrize("epi", ["relu", "residual", "act_after_residual"])
def test_conv_tf32_against_emulation(ks, stride, C, epi):
    from tfimm.backend import ops

    gen = torch.Generator().manual_seed(ks * 100 + stride * 10 + C)
    B, H, W, N = 3, 19, 23, 136 if C != 256 else 64
    pad = (ks - 1) // 2
    x = torch.randn(B, H, W, C, generator=gen).cuda()
    w = _weights(N, ks * ks * C, gen)
    bias = torch.randn(N, generator=gen).cuda()
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    res = torch.randn(B, Ho, Wo, N, generator=gen).cuda() if epi != "relu" else None
    kernels = set()
    with _shadowed_tf32(kernels) as census:
        ops.conv_gemm(x, w, bias=bias, ks=ks, stride=stride, pad=pad, act="relu", residual=res,
                      act_after_residual=epi == "act_after_residual")
    census.assert_ok()
    assert kernels == {"tfimm_b200_conv_tf32"}


SMALL_MAPS = [(7, 7, 1, 32), (14, 14, 2, 64), (8, 5, 1, 96)]


@pytest.mark.parametrize("H,W,stride,C", SMALL_MAPS, ids=[f"{h}x{w}s{s}c{c}" for h, w, s, c in SMALL_MAPS])
def test_conv_tf32_small_feature_maps(H, W, stride, C):
    """Output maps of at most 8 columns: the 128-row tile is 8 x 8 pixels of two images (the cv_pb = 2 geometry), with
    the 32-channel fp32 box; odd batch, so the last tile's second image is out of range."""
    from tfimm.backend import ops

    gen = torch.Generator().manual_seed(H * W + C)
    B, N, ks = 3, 72, 3
    x = torch.randn(B, H, W, C, generator=gen).cuda()
    w = _weights(N, ks * ks * C, gen)
    bias = torch.randn(N, generator=gen).cuda()
    Ho, Wo = (H + 2 - ks) // stride + 1, (W + 2 - ks) // stride + 1
    assert Wo <= 8
    res = torch.randn(B, Ho, Wo, N, generator=gen).cuda()
    kernels = set()
    with _shadowed_tf32(kernels) as census:
        ops.conv_gemm(x, w, bias=bias, ks=ks, stride=stride, pad=1, act="relu", residual=res, act_after_residual=True)
    census.assert_ok()
    assert kernels == {"tfimm_b200_conv_tf32"}


# ------------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("N", [50, 197, 577, 785])
@pytest.mark.parametrize("H", [3, 12])
def test_attention_tf32_against_emulation(N, H):
    from tfimm.backend import ops

    gen = torch.Generator().manual_seed(N * H)
    B, dh = 3, 64
    qkv = (torch.randn(B * N, 3 * H * dh, generator=gen) * 1.5).cuda()
    kernels = set()
    with _shadowed_tf32(kernels) as census:
        ops.attention(qkv, B, N, H, dh, dh ** -0.5)
    census.assert_ok()
    assert kernels == {"tfimm_b200_attention_tf32"}


# ------------------------------------------------------------------------------------------------ whole forwards
def _shadowed_forward(model, x, title):
    kernels = set()
    with _shadowed_tf32(kernels) as census:
        model(x.cuda())
    torch.cuda.synchronize()
    print(f"\n=== {title}: {census.launches} launches, kernels {sorted(k for k in kernels if 'tf32' in k)}")
    bad = census.failures()
    if bad:
        print("\n".join(census._fmt(r) for r in bad[:20]))
    census.assert_ok()
    return kernels


def _expected_tf32_kernels(family, name):
    """The TF32 entry points a tf32 forward of this configuration must reach: the GEMM always, the ViT attention for
    ViT / DeiT (head dim 64), the implicit convolution for the ResNets whose 3 x 3 convolutions see C % 64 == 0 and no
    GroupNorm (the deep stems of the *26d / *26t models start at 32 channels; resnet50_gn normalises the data)."""
    want = {"tfimm_b200_gemm_tf32"}
    if family == "vit":
        want.add("tfimm_b200_attention_tf32")
    if name in ("resnet50", "resnetblur50", "ecaresnet26t"):
        want.add("tfimm_b200_conv_tf32")
    return want


@pytest.mark.parametrize("family,name,overrides", SMALL, ids=[c[1] for c in SMALL])
def test_small_config_tf32_every_launch_within_its_bound(family, name, overrides):
    model, _, _ = _model(name, family, "tf32", overrides)
    for what, x in _inputs(model, 2):
        kernels = _shadowed_forward(model, x, f"{name} tf32 {what}")
        assert _expected_tf32_kernels(family, name) <= kernels, kernels
        assert "tfimm_b200_gemm_f32" not in kernels and "tfimm_b200_gemm_bf16" not in kernels


BENCH = [("vit", "vit_base_patch16_224"), ("convnext", "convnext_base"), ("swin", "swin_base_patch4_window7_224"),
         ("resnet", "resnet50")]


@pytest.mark.parametrize("family,name", BENCH, ids=[c[1] for c in BENCH])
def test_benchmark_config_tf32_at_batch_256_every_launch_within_its_bound(family, name):
    model, _, _ = _model(name, family, "tf32", seed=29)
    _, x = _inputs(model, 256)[0]
    kernels = _shadowed_forward(model, x, f"{name} tf32 batch 256")
    assert _expected_tf32_kernels(family, name) <= kernels, kernels
    del x
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ accuracy budget
# bound on the tf32 total max-norm error against the fp32 oracle: ~1.3 x the value measured on an H100 80GB HBM3
# (400 W power limit), same weights, images and metric as tests/test_parity_budget_gpu.py::test_bf16_error_budget.
# Measured: 2.7e-4 (EfficientNet-B0) .. 1.01e-3 (Swin-B), 7-8x below bf16; rms 0.12-0.14 x bf16's.
TF32_TOTAL = {
    "vit_tiny_patch16_224": 1.1e-3,          # measured 8.4e-4
    "vit_base_patch16_224": 9.5e-4,          # 7.3e-4
    "swin_tiny_patch4_window7_224": 1.2e-3,  # 9.2e-4
    "swin_base_patch4_window7_224": 1.3e-3,  # 1.01e-3
    "convnext_tiny": 7.0e-4,                 # 5.4e-4
    "convnext_base": 9.5e-4,                 # 7.2e-4
    "efficientnet_b0": 3.5e-4,               # 2.7e-4
    "efficientnet_b4": 4.5e-4,               # 3.4e-4
    "resnet50": 6.3e-4,                      # 4.8e-4
    "seresnet50": 5.2e-4,                    # 4.0e-4
}


@pytest.mark.parametrize("family,name,overrides,batch,tol_bf16", BUDGET, ids=[c[1] for c in BUDGET])
def test_tf32_error_budget(family, name, overrides, batch, tol_bf16):
    from oracle import params

    model, omod, w = _model(name, family, "tf32", overrides)
    m16, _, _ = _model(name, family, "bf16", overrides)
    x = params.test_images(batch, *model.cfg.input_size, model.cfg.in_channels)
    y = model(x.cuda()).float().cpu()
    y16 = m16(x.cuda()).float().cpu()
    with torch.no_grad():
        ref = omod.forward(model.cfg, w, x)
    total, _ = _nerr(y, ref)
    total16, _ = _nerr(y16, ref)
    r32, r16 = _rms(y, ref), _rms(y16, ref)
    print(f"TF32 BUDGET {name}: max-norm tf32-vs-fp32 {total:.2e} (bf16 {total16:.2e}) | rms tf32 {r32:.2e} "
          f"bf16 {r16:.2e} ratio {r32 / r16:.3f} | within 1e-3: {total <= 1e-3}")
    assert total < TF32_TOTAL[name], f"total error {total:.3e}"
    assert r32 <= 0.25 * r16, (r32, r16)


# ------------------------------------------------------------------------------------------------------ CUDA graph
# ~1.3 x measured (H100 80GB HBM3, 400 W): 6.4e-4, 6.0e-4, 7.9e-4; EfficientNet-B4 from its batch-4 budget (3.4e-4)
TF32_FULL = {"vit_base_patch16_224": 8.5e-4, "convnext_base": 8.0e-4, "swin_base_patch4_window7_224": 1.05e-3,
             "efficientnet_b4": 6.0e-4}
# EfficientNet's fused squeeze accumulates with fp32 atomics, whose last bits vary with the order (run to run and with
# the grid, i.e. the batch).  The next layer's TF32 rounding turns such a perturbation into a whole TF32 ulp (2^-11) for
# a few elements, which then spreads like bf16's divergence floor at 1/8 of its size: measured 1.5e-4 between two
# replays.  The other families are bit-deterministic and batch-invariant.
TF32_EFFICIENTNET_FLOOR = 5e-4


@pytest.mark.parametrize("family,name,batch,nref,tol_bf16", FULL, ids=[c[1] for c in FULL])
def test_tf32_baseline_config_at_its_own_batch_through_cuda_graph(family, name, batch, nref, tol_bf16):
    from oracle import params

    model, omod, w = _model(name, family, "tf32", seed=29)
    h, wd = model.cfg.input_size
    x = params.test_images(batch, h, wd, model.cfg.in_channels, seed=77)
    fwd = model.cuda_graph(batch)
    y = fwd(x.cuda()).float().cpu().clone()
    y_again = fwd(x.cuda()).float().cpu()
    if family == "efficientnet":
        assert _nerr(y_again, y)[0] < TF32_EFFICIENTNET_FLOOR
    else:
        assert torch.equal(y, y_again)
    idx = torch.linspace(0, batch - 1, nref).round().long()
    with torch.no_grad():
        ref = omod.forward(model.cfg, w, x[idx])
    total, _ = _nerr(y[idx], ref)
    small = model(x[idx].cuda()).float().cpu()
    inv, _ = _nerr(y[idx], small)
    print(f"TF32 FULL {name} batch {batch}: tf32-vs-fp32-oracle {total:.3e} | graph vs eager batch-{nref} {inv:.3e} "
          f"({fwd.launches} launches per replay)")
    assert total < TF32_FULL[name]
    assert inv < (TF32_EFFICIENTNET_FLOOR if family == "efficientnet" else 1e-6)
