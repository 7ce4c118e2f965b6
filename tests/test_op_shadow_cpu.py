"""CPU rehearsal of the op-by-op shadow harness (oracle/shadow.py), which tests/test_op_shadow_gpu.py runs on the GPU.

The "kernel" here is the emulation evaluated in float32 arithmetic (``emulate_bf16.emulated_ops(torch.float32)``): an
honest implementation of every launcher with the engine's storage points that only rounds differently.  Every shadowed
launch of every model of tests/test_orchestration_cpu.py must pass -- so the bounds are not tighter than a legitimate
change of summation order, and the snapshot / aliasing / in-place plumbing works -- and each seeded defect on top of that
stand-in must be rejected, naming the op it is in.
"""
import math
from pathlib import Path

import pytest
import torch

from test_orchestration_cpu import CASES, _build

# Launchers no model of CASES reaches, each with the GPU kernel test that covers it; tests/test_op_shadow_gpu.py
# reaches all of them.
ALLOWED_UNREACHED = {
    "window_attention": "test_window_attention_bf16",          # 8x8 / 12x12 windows (swin *_window12_384)
    "blur_pool": "test_blur_pool_reflect",                     # resnetblur50
    "group_norm": "test_group_norm_with_residual_and_act",     # resnet50_gn
    "eca_gate": "test_se_gate_scale_and_eca",                  # ecaresnet26t
}


def _plan_on_any_device(self):
    if self._plan is None:
        self._plan = self._compile()
    return self._plan


@pytest.fixture(scope="module")
def cpu_models():
    """The engine's host orchestration on CPU tensors (as ``cpu_engine`` in tests/test_orchestration_cpu.py)."""
    from tfimm.models.model import Model

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(Model, "_ensure_plan", _plan_on_any_device)
        yield


def _images(model, batch, uint8=False):
    from oracle import params

    x = params.test_images(batch, *model.cfg.input_size, model.cfg.in_channels)
    return (x * 255).round().to(torch.uint8) if uint8 else x


def _shadowed_forward(model, x, return_features=False, mutate=None):
    """One forward with the float32 stand-in as the kernel (``mutate(ops)`` may replace some of it first)."""
    from oracle import emulate_bf16, shadow
    from tfimm.backend import ops

    with emulate_bf16.emulated_ops(arithmetic=torch.float32):
        if mutate is not None:
            mutate(ops)
        with shadow.shadowed_ops() as census:
            model(x, return_features=return_features)
    return census


@pytest.fixture(scope="module")
def rehearsal(cpu_models):
    """{(model, precision): [census, ...]}: fp32 images, raw uint8 pixels (fused preprocessing) where the family
    takes them, and one ``return_features=True`` pass (ViT: the fp32 attention that writes ``probs``)."""
    out = {}
    for family, name, overrides, batch in CASES:
        for precision in ("bf16", "fp32"):
            model, _, _ = _build(family, name, overrides, precision)
            runs = [_shadowed_forward(model, _images(model, batch))]
            if model.accepts_uint8:
                runs.append(_shadowed_forward(model, _images(model, batch, uint8=True)))
            runs.append(_shadowed_forward(model, _images(model, batch), return_features=True))
            out[(name, precision)] = runs
    return out


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("name", [c[1] for c in CASES])
def test_float32_standin_passes_every_shadowed_launch(rehearsal, name, precision):
    for census in rehearsal[(name, precision)]:
        assert census.rows
        census.assert_ok()
        # the fused MLP's cited bound is the one exception: everything else is held to the derived per-element rule
        assert all(r["cite"] is None for r in census.rows if r["op"] != "mlp_fused")


def test_census_reaches_every_launcher(rehearsal):
    from oracle import emulate_bf16, shadow
    from tfimm.backend import ops

    launchers = {n for n in dir(ops) if not n.startswith("_") and callable(getattr(ops, n))
                 and getattr(getattr(ops, n), "__module__", "") == ops.__name__
                 and n not in ("act_code", "same_pad", "conv_geometry", "attention_bf16_supported")}
    assert launchers - set(shadow.PREDICATES) == set(shadow.SHADOWED) <= set(emulate_bf16._EMULATED)
    reached = set().union(*(c.ops() for runs in rehearsal.values() for c in runs))
    assert set(shadow.SHADOWED) - reached == set(ALLOWED_UNREACHED), set(shadow.SHADOWED) - reached
    kernel_tests = (Path(__file__).parent / "test_kernels_gpu.py").read_text()
    for op, test in ALLOWED_UNREACHED.items():
        assert f"def {test}(" in kernel_tests, (op, test)


# ------------------------------------------------------------------------------------------------------ mutations
def _wrap(ops, name, make):
    setattr(ops, name, make(getattr(ops, name)))


def _tile(kind):
    def mutate(ops):
        def make(f):
            def gemm(*a, **k):
                out = f(*a, **k)
                if out.shape[0] >= 384:          # rows 128..255: the second 128-row output tile
                    out[128:256] = out[129:257].clone() if kind == "shift" else 0
                return out
            return gemm
        _wrap(ops, "gemm", make)
    return mutate


def _bias_last_group(ops):
    def make(f):
        def gemm(a, w, bias=None, **k):
            if bias is not None:
                bias = bias.clone()
                bias[-8:] = 0                    # columns n >= N - 8 lose their bias
            return f(a, w, bias=bias, **k)
        return gemm
    _wrap(ops, "gemm", make)


def _gelu_tanh(ops):
    def make(f):
        def gemm(a, w, bias=None, act=None, **k):
            if act != "gelu":
                return f(a, w, bias=bias, act=act, **k)
            assert not k, k
            z = f(a, w, bias=bias, out_dtype=torch.float32)
            y = 0.5 * z * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (z + 0.044715 * z ** 3)))
            return y.to(a.dtype)
        return gemm
    _wrap(ops, "gemm", make)


def _ulp_up(ops):
    def make(f):
        def gemm(*a, **k):
            out = f(*a, **k)
            if out.dtype == torch.bfloat16:
                sel = (torch.arange(out.numel()) % 20 == 0).view(out.shape)     # 5 % of the outputs
                bits = out.view(torch.int16)
                up = torch.where(out >= 0, bits + 1, bits - 1)                   # next bf16 value towards +inf
                out.view(torch.int16).copy_(torch.where(sel, up, bits))
            return out
        return gemm
    _wrap(ops, "gemm", make)


def _shifted_window_tables(mutation):
    def mutate(ops):
        from tfimm.architectures.swin import window_tables

        def make(f):
            def wa(qkv, bias_pad, row_map, maskbits, B, nw_img, N, H, dh, scale):
                if maskbits is not None:         # shifted block
                    if mutation == "mask":
                        maskbits = None
                    else:
                        ws, side = math.isqrt(N), math.isqrt(nw_img * N)
                        rm, _ = window_tables(side, side, ws, ws // 2 - 1)      # roll by shift - 1
                        row_map = torch.from_numpy(rm).to(row_map.device)
                return f(qkv, bias_pad, row_map, maskbits, B, nw_img, N, H, dh, scale)
            return wa
        _wrap(ops, "window_attention_tc", make)
    return mutate


def _pool_tile_missing(ops):
    def make(f):
        def dw(*a, pool_sum=None, **k):
            out = f(*a, pool_sum=pool_sum, **k)
            if pool_sum is not None:
                pool_sum[0] -= out[0, :8, :8].float().sum(dim=(0, 1))   # one 8x8 tile never added
            return out
        return dw
    _wrap(ops, "dwconv_bias_act", make)


MUTATIONS = [
    ("tile_shifted_by_a_row", "efficientnet_b0", "gemm", _tile("shift")),
    ("tile_zeroed", "efficientnet_b0", "gemm", _tile("zero")),
    ("bias_missing_on_last_column_group", "efficientnet_b0", "gemm", _bias_last_group),
    ("gelu_tanh_form", "vit_tiny_patch16_224", "gemm", _gelu_tanh),
    ("one_ulp_up_on_5_percent", "efficientnet_b0", "gemm", _ulp_up),
    ("swin_roll_off_by_one", "swin_tiny_patch4_window7_224", "window_attention_tc", _shifted_window_tables("roll")),
    ("region_mask_ignored", "swin_tiny_patch4_window7_224", "window_attention_tc", _shifted_window_tables("mask")),
    ("pool_sum_missing_a_tile", "efficientnet_b0", "dwconv_bias_act", _pool_tile_missing),
]


@pytest.mark.parametrize("mutation,name,op,mutate", MUTATIONS, ids=[m[0] for m in MUTATIONS])
def test_seeded_defect_is_rejected(cpu_models, mutation, name, op, mutate):
    family, _, overrides, batch = next(c for c in CASES if c[1] == name)
    model, _, _ = _build(family, name, overrides, "bf16")
    census = _shadowed_forward(model, _images(model, batch), mutate=mutate)
    print(f"\n{mutation}:\n" + "\n".join(census._fmt(r) for r in census.failures()[:5]))
    with pytest.raises(AssertionError, match=op):
        census.assert_ok()
    # the forward continues on the defective results, yet every other op is checked on its own inputs and passes
    assert {r["op"] for r in census.failures()} == {op}


def test_layernorm_eps_outside_the_square_root_is_rejected():
    """Where the variance is comparable to eps, (x - mean) / (sqrt(var) + eps) is far from (x - mean) / sqrt(var + eps);
    rows of spread ~1e-3 with eps = 1e-6 make that case.  The honest stand-in passes on the same rows."""
    from oracle import emulate_bf16, shadow
    from tfimm.backend import ops

    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 192, generator=g) * 1e-3 + 0.01
    gamma, beta = 1 + 0.2 * torch.randn(192, generator=g), 0.2 * torch.randn(192, generator=g)

    def eps_outside(x, gamma, beta, eps, out_dtype, out=None):
        mu = x.mean(-1, keepdim=True)
        var = (x - mu).pow(2).mean(-1, keepdim=True)
        y = ((x - mu) / (var.sqrt() + eps) * gamma + beta).to(out_dtype)
        return out.copy_(y) if out is not None else y

    for layernorm, rejected in ((None, False), (eps_outside, True)):
        with emulate_bf16.emulated_ops(arithmetic=torch.float32):
            if layernorm is not None:
                ops.layernorm = layernorm
            with shadow.shadowed_ops() as census:
                for dt in (torch.bfloat16, torch.float32):
                    ops.layernorm(x, gamma, beta, 1e-6, dt)
        assert len(census.rows) == 2
        if rejected:
            with pytest.raises(AssertionError, match="layernorm"):
                census.assert_ok()
            assert len(census.failures()) == 2
        else:
            census.assert_ok()


def test_shadowed_launches_refuse_cuda_graph_capture(monkeypatch):
    from oracle import emulate_bf16, shadow
    from tfimm.backend import ops

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with emulate_bf16.emulated_ops(arithmetic=torch.float32), shadow.shadowed_ops():
        with pytest.raises(RuntimeError, match="CUDA-graph capture"):
            ops.cast(torch.zeros(4), torch.bfloat16)

