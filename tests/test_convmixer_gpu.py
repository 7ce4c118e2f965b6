"""ConvMixer on the H100: the depthwise kernel against its float64 statement in the reference's form (the family's
shapes, maps smaller than the kernel, |t_in| ~ 1e3, interiors full of exact zeros), bitwise determinism, guard regions
around the output, and the three registrations in every precision, launch by launch under the shadow harness.  Peak
allocated memory stays well under 16 GB."""
import importlib
import sys
from contextlib import nullcontext
from copy import deepcopy
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = Path(__file__).resolve().parent
if str(HERE) not in sys.path:
    sys.path.insert(0, str(HERE))

import convmixer_oracle as co  # noqa: E402
from tf32_oracle import tf32_oracle  # noqa: E402

NAMES = ["convmixer_768_32", "convmixer_1024_20_ks9_p14", "convmixer_1536_20"]


@pytest.fixture
def convmixer():
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.convmixer"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


# ------------------------------------------------------------------------------------------------ the kernel alone
BF, F32 = torch.bfloat16, torch.float32
# (H, W), C, k, B, act, output dtype: the family's three shapes, maps smaller than the kernel (1 x 1, 2 x 3, 5 x 6) and
# an odd one (13 x 17, two 8 x 16 / 16 x 16 tiles with ragged edges), batch 1 to 64, relu and gelu, bf16 and fp32
KERNEL_CASES = [
    ((32, 32), 768, 7, 1, "relu", BF), ((32, 32), 768, 7, 2, "gelu", F32),
    ((16, 16), 1024, 9, 64, "gelu", BF), ((16, 16), 1024, 9, 1, "relu", F32),
    ((32, 32), 1536, 9, 2, "gelu", BF), ((32, 32), 1536, 9, 1, "gelu", F32),
    ((1, 1), 768, 9, 64, "gelu", BF), ((1, 1), 1024, 7, 3, "relu", F32),
    ((2, 3), 768, 7, 64, "relu", BF), ((2, 3), 1536, 9, 3, "gelu", F32),
    ((5, 6), 768, 7, 64, "relu", BF), ((5, 6), 1024, 9, 3, "gelu", F32),
    ((13, 17), 1024, 9, 64, "gelu", BF), ((13, 17), 768, 7, 3, "relu", F32),
]


def _params(C, k, seed, t_scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    s_in = torch.rand(C, generator=g, device="cuda") + 0.5
    t_in = torch.randn(C, generator=g, device="cuda") * t_scale
    taps = torch.randn((k * k, C), generator=g, device="cuda") / k
    bias = torch.randn(C, generator=g, device="cuda") * 0.2
    s1 = torch.rand(C, generator=g, device="cuda") + 0.25
    t1 = torch.randn(C, generator=g, device="cuda") * 0.2
    return s_in, t_in, taps, bias, s1, t1


def _act_input(shape, act, seed):
    """The previous layer's activation output: relu leaves exact zeros in about half the interior."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(shape, generator=g, device="cuda")
    return torch.relu(z) if act == "relu" else torch.nn.functional.gelu(z)


@pytest.mark.parametrize("hw,C,k,B,act,out", KERNEL_CASES,
                         ids=[f"{h}x{w}-C{c}-k{k}-B{b}-{a}-{'bf16' if o is BF else 'f32'}"
                              for (h, w), c, k, b, a, o in KERNEL_CASES])
def test_kernel_against_float64(hw, C, k, B, act, out):
    from tfimm.backend import convmixer_ops

    a = _act_input((B, *hw, C), act, C + B)
    with co.shadowed_convmixer_ops() as census:
        y = convmixer_ops.dwconv(a, *_params(C, k, k + B), act, out)
    census.assert_ok()
    assert census.ops() == {"dwconv"} and y.dtype == out and y.shape == a.shape


@pytest.mark.parametrize("hw,C,k", [((32, 32), 768, 7), ((16, 16), 1024, 9), ((5, 6), 1536, 9)])
def test_large_shift_and_exact_zeros(hw, C, k):
    """|t_in| ~ 1e3 with an input that is exactly 0 in most of the interior (relu): the shift must reach every interior
    cell, zero or not, and no padded cell; the kernel holds its bound and differs from a value-masked padding."""
    from tfimm.backend import convmixer_ops

    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.relu(torch.randn((3, *hw, C), generator=g, device="cuda") - 1.0)   # ~84 % exact zeros
    assert (a == 0).float().mean().item() > 0.8
    p = _params(C, k, 9, t_scale=1e3)
    with co.shadowed_convmixer_ops() as census:
        y = convmixer_ops.dwconv(a, *p, "relu", F32)
    census.assert_ok()
    assert p[1].abs().max().item() > 1e3 and torch.isfinite(y).all()


def test_determinism():
    from tfimm.backend import convmixer_ops

    for (hw, C, k, B, act, out) in (((32, 32), 1536, 9, 4, "gelu", BF), ((32, 32), 768, 7, 4, "relu", F32),
                                    ((13, 17), 1024, 9, 4, "gelu", F32)):
        a = _act_input((B, *hw, C), act, 1)
        p = _params(C, k, 2)
        y1 = convmixer_ops.dwconv(a, *p, act, out)
        y2 = convmixer_ops.dwconv(a, *p, act, out)
        bits = torch.int16 if out is BF else torch.int32
        assert torch.equal(y1.view(bits), y2.view(bits))


@pytest.mark.parametrize("out", [BF, F32])
def test_guard_regions_untouched(out):
    """The output written into the middle of a larger buffer: the guard cells on both sides keep their pattern, and
    the values equal the launcher's own output."""
    from tfimm.backend import convmixer_ops, ops

    B, H, W, C, k = 3, 13, 17, 768, 9
    a = _act_input((B, H, W, C), "gelu", 4)
    p = _params(C, k, 5)
    G = 64
    n = B * H * W * C
    buf = torch.full((n + 2 * G,), 777.0, device="cuda").to(out)
    y = buf[G:G + n]
    ops._call("tfimm_b200_convmixer_dwconv", a.device, a.data_ptr(), *(t.data_ptr() for t in p), y.data_ptr(),
              ops._code(y), B, H, W, C, k, ops.act_code("gelu"))
    torch.cuda.synchronize()
    guard = torch.cat((buf[:G], buf[-G:]))
    assert torch.equal(guard, torch.full_like(guard, 777.0).to(torch.float32).to(out))
    assert torch.equal(y.view(B, H, W, C), convmixer_ops.dwconv(a, *p, "gelu", out))


def test_refused_before_launch():
    from tfimm.backend import convmixer_ops

    a = torch.zeros((1, 4, 4, 64), device="cuda")
    p = list(_params(64, 5, 1))
    with pytest.raises(ValueError, match="kernel sizes"):
        convmixer_ops.dwconv(a, *p, "relu", F32)
    a = torch.zeros((1, 4, 4, 48), device="cuda")
    with pytest.raises(ValueError, match="C % 32"):
        convmixer_ops.dwconv(a, *_params(48, 7, 1), "relu", F32)


# ------------------------------------------------------------------------------------------------ whole models
def _weights(m, seed=11):
    from oracle import convmixer as oc
    from oracle import params

    return params.random_params(oc.param_shapes(m.cfg), seed=seed)


def _nerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("precision", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("name", NAMES)
def test_registered_models_shadowed(convmixer, name, precision):
    """Every launch of a batch-2 forward with features checked against its own float64 statement; the depthwise
    kernel ran; fp32 logits and features match the float64 oracle."""
    import tfimm
    from oracle import convmixer as oc
    from oracle import params
    from tfimm.backend import ops

    torch.cuda.reset_peak_memory_stats()
    m = tfimm.create_model(name, precision=precision, device="cuda")
    w = _weights(m)
    m.load_weights_dict(w)
    x = params.test_images(2, *m.cfg.input_size).cuda()
    ops.trace = []
    try:
        with (tf32_oracle() if precision == "tf32" else nullcontext()), co.shadowed_convmixer_ops() as census:
            y, feats = m(x, return_features=True)
        fams = {t[0] for t in ops.trace}
    finally:
        ops.trace = None
    census.assert_ok()
    assert "convmixer_dwconv" in fams and ("gemm_tf32" in fams) == (precision == "tf32"), fams
    assert y.shape == (2, 1000) and torch.isfinite(y).all() and list(feats) == m.feature_names
    if precision == "fp32":
        with torch.no_grad():
            ref, rfeats = oc.forward(m.cfg, {k: v.cuda() for k, v in w.items()}, x, return_features=True)
        err = _nerr(y, ref)
        print(f"{name} fp32: normalised max error vs float64 oracle {err:.3e}")
        assert err < 1e-5, err
        for k in ("stem", "block_0", "features_all", "features"):
            assert _nerr(feats[k], rfeats[k]) < 1e-5, k
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    assert peak < 16, peak


@pytest.mark.parametrize("name", NAMES)
def test_uint8_and_non_divisible_input(convmixer, name):
    """uint8 pixels equal create_preprocessing's floats; a 230 x 218 input drops the remainder as the reference's
    VALID stem does, and its fp32 logits match the oracle."""
    import tfimm
    from oracle import convmixer as oc

    m = tfimm.create_model(name, precision="fp32", device="cuda")
    w = _weights(m)
    m.load_weights_dict(w)
    u8 = torch.randint(0, 256, (2, 230, 218, 3), dtype=torch.uint8, device="cuda")
    xf = tfimm.create_preprocessing(name)(u8)
    yu, fu = m(u8, return_features=True)
    yf = m(xf)
    p = m.cfg.patch_size[0]
    assert tuple(fu["stem"].shape[1:3]) == (230 // p, 218 // p)
    assert _nerr(yu, yf) < 1e-5
    with torch.no_grad():
        ref = oc.forward(m.cfg, {k: v.cuda() for k, v in w.items()}, xf)
    assert _nerr(yf, ref) < 1e-5


@pytest.mark.parametrize("name", NAMES)
def test_cuda_graph_equals_eager(convmixer, name):
    import tfimm
    from oracle import params

    torch.cuda.reset_peak_memory_stats()
    m = tfimm.create_model(name, precision="bf16", device="cuda")
    m.load_weights_dict(_weights(m))
    x = params.test_images(16, 224, 224).cuda()
    eager = m(x)
    run = m.cuda_graph(16)
    assert torch.equal(run(x), eager)
    assert torch.cuda.max_memory_allocated() / 2 ** 30 < 16


def _rms(a, b):
    return ((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("name", NAMES)
def test_bf16_error_budget(convmixer, name):
    """The engine in bf16 is no farther from the float64 oracle than the ideal bf16 graph (every kernel replaced by
    its float64 statement at the engine's storage points), and diverges from that graph by no more than 1.6 x the
    float64-vs-float32 emulation floor."""
    import tfimm
    from oracle import convmixer as oc
    from oracle import params

    m = tfimm.create_model(name, precision="bf16", device="cuda")
    w = _weights(m)
    m.load_weights_dict(w)
    x = params.test_images(4, 224, 224).cuda()
    y = m(x).double()
    with co.emulated_convmixer_ops():
        y_ideal = m(x).double()
    with co.emulated_convmixer_ops(arithmetic=torch.float32):
        y_ideal32 = m(x).double()
    with torch.no_grad():
        ref = oc.forward(m.cfg, {k: v.cuda() for k, v in w.items()}, x)
    r_eng, r_ideal, r_kern, r_floor = _rms(y, ref), _rms(y_ideal, ref), _rms(y, y_ideal), _rms(y_ideal32, y_ideal)
    print(f"BUDGET {name}: rms engine-vs-oracle {r_eng:.2e} | ideal-vs-oracle {r_ideal:.2e} | engine-vs-ideal "
          f"{r_kern:.2e} | floor {r_floor:.2e}")
    assert r_kern < 1.6 * r_floor + 1e-4, (r_kern, r_floor)
    assert r_eng < 1.25 * r_ideal + 1e-4, (r_eng, r_ideal)
