"""PoolFormer on the H100: the three kernels against their float64 statements (including an input with mean 1e3 and
std 1), bitwise determinism, guard regions around every output, and the five registrations in every precision, launch
by launch under the shadow harness.  Peak allocated memory stays well under 16 GB."""
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

import poolformer_oracle as po  # noqa: E402
from tf32_oracle import tf32_oracle  # noqa: E402

NAMES = ["poolformer_s12", "poolformer_s24", "poolformer_s36", "poolformer_m36", "poolformer_m48"]


@pytest.fixture
def poolformer():
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.poolformer"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


# ------------------------------------------------------------------------------------------------ kernels alone
# every H x W in {56², 28², 14², 7², 1 x 1, 3 x 5, 13 x 17} and every C of the family appears; batch 64 only where the
# tensor stays small
KERNEL_CASES = [
    ((56, 56), 64, 3), ((56, 56), 96, 1), ((28, 28), 128, 3), ((28, 28), 192, 1), ((14, 14), 320, 3),
    ((14, 14), 384, 64), ((7, 7), 512, 64), ((7, 7), 768, 3), ((1, 1), 512, 64), ((1, 1), 768, 3),
    ((3, 5), 64, 64), ((13, 17), 320, 3), ((13, 17), 96, 64),
]


def _vecs(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    gamma = torch.rand(C, generator=g, device="cuda") + 0.5
    beta = torch.randn(C, generator=g, device="cuda")
    ls1 = torch.rand(C, generator=g, device="cuda") * 0.5
    return gamma, beta, ls1


def _run_all(x, gamma, beta, ls1):
    from tfimm.backend import poolformer_ops

    p = poolformer_ops.gn1_partials(x)
    out, p2 = poolformer_ops.poolformer_mixer(x, p, gamma, beta, ls1, 1e-5)
    yb = poolformer_ops.gn1_apply(out, p2, gamma, beta, 1e-5, torch.bfloat16)
    yf = poolformer_ops.gn1_apply(x, p, gamma, beta, 1e-5, torch.float32)
    return p, out, p2, yb, yf


@pytest.mark.parametrize("hw,C,B", KERNEL_CASES, ids=[f"{h}x{w}-C{c}-B{b}" for (h, w), c, b in KERNEL_CASES])
def test_kernels_against_float64(hw, C, B):
    """Each launch inside its derived bound: partials, the mixer (fp32, and its output's partials), the apply in bf16
    (within one bf16 ulp plus the arithmetic term) and fp32."""
    g = torch.Generator(device="cuda").manual_seed(C + B)
    x = torch.randn((B, *hw, C), generator=g, device="cuda") * 2 + 0.3
    with po.shadowed_poolformer_ops() as census:
        _run_all(x, *_vecs(C, B))
    census.assert_ok()
    assert census.ops() == {"gn1_partials", "poolformer_mixer", "gn1_apply"}


@pytest.mark.parametrize("hw,C", [((56, 56), 64), ((14, 14), 384), ((13, 17), 96)])
def test_large_mean_small_std(hw, C):
    """mean 1e3, std 1: a one-pass sum / sum of squares would lose the variance, and summing x_j before subtracting
    x_i the mixer's term; the centred M2 and the centred differences hold their bounds."""
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((3, *hw, C), generator=g, device="cuda") + 1e3
    gamma, beta, ls1 = _vecs(C, 3)
    with po.shadowed_poolformer_ops() as census:
        from tfimm.backend import poolformer_ops

        p = poolformer_ops.gn1_partials(x)
        out, p2 = poolformer_ops.poolformer_mixer(x, p, gamma, beta, ls1, 1e-5)
        poolformer_ops.gn1_apply(x, p, gamma, beta, 1e-5, torch.float32)
    census.assert_ok()
    # the merged variance itself, against float64
    mean, var = po.merge_partials(p.double())
    xd = x.double().reshape(3, -1)
    assert ((var - xd.var(1, unbiased=False)).abs() / xd.var(1, unbiased=False)).max().item() < 1e-3
    assert (mean - xd.mean(1)).abs().max().item() < 1e-3


def test_determinism():
    x = torch.randn((5, 28, 28, 192), device="cuda") * 3
    vecs = _vecs(192, 1)
    a = _run_all(x, *vecs)
    b = _run_all(x, *vecs)
    bits = {torch.float32: torch.int32, torch.bfloat16: torch.int16}
    for u, v in zip(a, b):
        assert torch.equal(u.view(bits[u.dtype]), v.view(bits[v.dtype]))


def test_guard_regions_untouched():
    """Outputs and partials written into the middle of larger buffers: the in-bounds guard cells on both sides keep
    their pattern."""
    from tfimm.backend import ops, poolformer_ops

    B, H, W, C = 3, 13, 17, 96
    N, S = H * W * C, poolformer_ops.splits(H, W, C)
    G = 64   # guard cells, a multiple of 4 so that the 16-byte alignment holds
    x = torch.randn((B, H, W, C), device="cuda")
    gamma, beta, ls1 = _vecs(C, 2)
    dev = x.device

    def guarded(n, dtype):
        buf = torch.full((n + 2 * G,), 777.0, device="cuda").to(dtype)   # 776 in bf16
        return buf, buf[G:G + n]

    pbuf, p = guarded(B * S * 3, torch.float32)
    obuf, out = guarded(B * N, torch.float32)
    qbuf, p2 = guarded(B * S * 3, torch.float32)
    ybuf, y = guarded(B * N, torch.bfloat16)
    ops._call("tfimm_b200_gn1_partials", dev, x.data_ptr(), p.data_ptr(), B, H, W, C, S)
    ops._call("tfimm_b200_poolformer_mixer", dev, x.data_ptr(), p.data_ptr(), gamma.data_ptr(), ls1.data_ptr(),
              out.data_ptr(), p2.data_ptr(), B, H, W, C, S, 1e-5)
    ops._call("tfimm_b200_gn1_apply", dev, out.data_ptr(), p2.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
              y.data_ptr(), ops.BF16, B, H, W, C, S, 1e-5)
    torch.cuda.synchronize()
    for buf in (pbuf, obuf, qbuf, ybuf):
        guard = torch.cat((buf[:G], buf[-G:]))
        assert torch.equal(guard, torch.full_like(guard, 777.0).to(torch.float32).to(buf.dtype))
    assert torch.isfinite(out).all() and torch.isfinite(y.float()).all()
    ref_out, _ = poolformer_ops.poolformer_mixer(x, poolformer_ops.gn1_partials(x), gamma, beta, ls1, 1e-5)
    assert torch.equal(out.view(B, H, W, C), ref_out)


# ------------------------------------------------------------------------------------------------ whole models
def _weights(m, seed=11):
    """Random weights with layer scales of a trained model's size, so that the mixer and MLP terms are visible."""
    from oracle import params
    from oracle import poolformer as op

    w = params.random_params(op.param_shapes(m.cfg), seed=seed)
    for k in w:
        if "layer_scale" in k:
            w[k] = 0.05 + 0.1 * w[k].abs()
    return w


def _nerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("precision", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("name", NAMES)
def test_registered_models_shadowed(poolformer, name, precision):
    """Every launch of a batch-3 forward checked against its own float64 statement; the mixer kernel ran; fp32 logits
    match the float64 oracle."""
    import tfimm
    from oracle import params
    from oracle import poolformer as op
    from tfimm.backend import ops

    torch.cuda.reset_peak_memory_stats()
    m = tfimm.create_model(name, precision=precision, device="cuda")
    w = _weights(m)
    m.load_weights_dict(w)
    x = params.test_images(3, *m.cfg.input_size).cuda()
    ops.trace = []
    try:
        # tf32: the GEMMs' statements and bounds are the TF32 ones (tests/tf32_oracle.py), entered first
        with (tf32_oracle() if precision == "tf32" else nullcontext()), po.shadowed_poolformer_ops() as census:
            y = m(x)
        fams = {t[0] for t in ops.trace}
    finally:
        ops.trace = None
    census.assert_ok()
    assert {"gn1_partials", "poolformer_mixer", "gn1_apply"} <= fams, fams
    assert y.shape == (3, 1000) and torch.isfinite(y).all()
    if precision == "bf16" and name.startswith("poolformer_m"):
        assert "mlp_bf16" in fams
    assert ("gemm_tf32" in fams) == (precision == "tf32"), fams
    if precision == "fp32":
        with torch.no_grad():
            ref = op.forward(m.cfg, {k: v.cuda() for k, v in w.items()}, x)
        err = _nerr(y, ref)
        print(f"{name} fp32: normalised max error vs float64 oracle {err:.3e}")
        assert err < 3e-6, err   # measured 6.6e-7 .. 8.5e-7
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    assert peak < 16, peak


def test_uint8_stem_equals_create_preprocessing(poolformer):
    import tfimm

    m = tfimm.create_model("poolformer_s12", precision="fp32", device="cuda")
    m.load_weights_dict(_weights(m))
    u8 = torch.randint(0, 256, (3, 224, 224, 3), dtype=torch.uint8, device="cuda")
    xf = tfimm.create_preprocessing("poolformer_s12")(u8)
    _, fu = m(u8, return_features=True)
    _, ff = m(xf, return_features=True)
    err = _nerr(fu["patch_embedding"], ff["patch_embedding"])
    print(f"uint8 stem vs create_preprocessing: {err:.3e}")
    assert err < 1e-5, err
    assert list(fu) == m.feature_names


def test_m48_bf16_batch64_cuda_graph(poolformer):
    import tfimm
    from oracle import params

    torch.cuda.reset_peak_memory_stats()
    m = tfimm.create_model("poolformer_m48", precision="bf16", device="cuda")
    m.load_weights_dict(_weights(m))
    x = params.test_images(64, 224, 224).cuda()
    eager = m(x)
    run = m.cuda_graph(64)
    assert torch.equal(run(x), eager)
    assert torch.cuda.max_memory_allocated() / 2 ** 30 < 16


def _rms(a, b):
    return ((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("name", ["poolformer_s12", "poolformer_m36"])
def test_bf16_error_budget(poolformer, name):
    """As for MLP-Mixer (tests/test_parity_budget_gpu.py B1 / B2): the kernels diverge from the ideal bf16 graph
    (emulated, float64 arithmetic, the engine's storage points) by no more than 1.6 x the float64-vs-float32 emulation
    floor, and add nothing measurable to the ideal graph's own distance from the float64 oracle."""
    import tfimm
    from oracle import params
    from oracle import poolformer as op

    m = tfimm.create_model(name, precision="bf16", device="cuda")
    w = _weights(m)
    m.load_weights_dict(w)
    x = params.test_images(4, 224, 224).cuda()
    y = m(x).double()
    with po.emulated_poolformer_ops():
        y_ideal = m(x).double()
    with po.emulated_poolformer_ops(arithmetic=torch.float32):
        y_ideal32 = m(x).double()
    with torch.no_grad():
        ref = op.forward(m.cfg, {k: v.cuda() for k, v in w.items()}, x)
    r_eng, r_ideal, r_kern, r_floor = _rms(y, ref), _rms(y_ideal, ref), _rms(y, y_ideal), _rms(y_ideal32, y_ideal)
    print(f"BUDGET {name}: rms engine-vs-oracle {r_eng:.2e} | ideal-vs-oracle {r_ideal:.2e} | engine-vs-ideal "
          f"{r_kern:.2e} | floor {r_floor:.2e}")
    assert r_kern < 1.6 * r_floor + 1e-4, (r_kern, r_floor)
    assert r_eng < 1.25 * r_ideal + 1e-4, (r_eng, r_ideal)
