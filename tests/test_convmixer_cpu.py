"""ConvMixer family on CPU: opt-in registration (and the registry left as it was found), the C entry point's argument
checks, the host orchestration on the float64 statements, the float32 shadow rehearsal and seeded defects."""
import importlib
import subprocess
import sys
from copy import deepcopy
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))


@pytest.fixture
def convmixer():
    """Registers the ConvMixer models for one test and restores the registry afterwards, so that the exact
    ``list_models()`` / ``list_modules()`` of the other suites hold in any test order."""
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


def test_import_tfimm_registers_nothing_new():
    code = ("import sys; sys.path[:0] = ['{0}', '{0}/tensorflow-image-models_b200']; import tfimm; "
            "from tfimm.models.registry import list_modules; print(len(tfimm.list_models()), sorted(list_modules()), "
            "'tfimm.architectures.convmixer' in sys.modules)").format(ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == "False"
    assert "convmixer" not in " ".join(out)


def test_registration_on_import(convmixer):
    import tfimm

    assert sorted(tfimm.list_models(module="convmixer")) == [
        "convmixer_1024_20_ks9_p14", "convmixer_1536_20", "convmixer_768_32"]
    m = tfimm.create_model("convmixer_768_32", device="meta")
    assert isinstance(m, convmixer.ConvMixer) and m.cfg.kernel_size == 7 and m.cfg.act_layer == "relu"
    assert m.feature_names == ["stem"] + [f"block_{j}" for j in range(32)] + ["features_all", "features", "logits"]
    assert m.nb_features == 768


PREFIX = "tfimm_b200_"


def test_entry_point_refusals_past_the_shape():
    """Unsupported kernel sizes and widths return TFIMM_ERR_UNSUPPORTED, bad arguments TFIMM_ERR_INVALID_ARGUMENT, each
    with its message and before any CUDA call."""
    from tfimm.backend import lib

    h = lib.load()
    p = 256

    def call(y_dtype=lib.BF16, C=64, k=9, act=1, y=2 * p):
        st = h.tfimm_b200_convmixer_dwconv(p, p, p, p, p, p, p, y, y_dtype, 2, 4, 4, C, k, act, None)
        return st, h.tfimm_b200_last_error().decode()

    assert call(k=5) == (3, "convmixer_dwconv: kernel size 5 is not supported (7 or 9)")
    assert call(k=3) == (3, "convmixer_dwconv: kernel size 3 is not supported (7 or 9)")
    assert call(C=48) == (3, "convmixer_dwconv: C = 48 is not a multiple of 32")
    assert call(y_dtype=lib.U8) == (1, "convmixer_dwconv: y_dtype must be bf16 or f32")
    assert call(act=9) == (1, "convmixer_dwconv: unknown activation code 9")
    assert call(y=p) == (1, "convmixer_dwconv: y must not alias a")


def test_trace_family_and_counts():
    from tfimm.backend import convmixer_ops, ops

    sys.path.insert(0, str(ROOT / "tools"))
    import ncu_traffic

    name = "void tfimm::(anonymous namespace)::convmixer_dwconv_kernel<9, 8, 16, float>(const float *)"
    assert ncu_traffic.family_of(name) == "convmixer_dwconv" == ops.TRACE_FAMILY[PREFIX + "convmixer_dwconv"]
    assert convmixer_ops.dwconv_nbytes(2, 16, 16, 1024, 9, torch.bfloat16) == 2 * 256 * 1024 * 6.0 + 4.0 * 1024 * 86
    assert convmixer_ops.supported(768, 7) and convmixer_ops.supported(1536, 9)
    assert not convmixer_ops.supported(768, 5) and not convmixer_ops.supported(80, 9)


def test_refusals(convmixer):
    cfg = convmixer.ConvMixerConfig
    with pytest.raises(ValueError, match="normalization"):
        convmixer.ConvMixer(cfg(name="t", norm_layer="layer_norm"), device="meta")
    for k in (3, 5, 8, 11):
        with pytest.raises(ValueError, match="kernel_size"):
            convmixer.ConvMixer(cfg(name="t", kernel_size=k), device="meta")
    with pytest.raises(ValueError, match="multiple of 32"):
        convmixer.ConvMixer(cfg(name="t", embed_dim=48), device="meta")
    with pytest.raises(ValueError, match="square"):
        convmixer.ConvMixer(cfg(name="t", patch_size=(7, 14)), device="meta")
    with pytest.raises(ValueError, match="activation"):
        convmixer.ConvMixer(cfg(name="t", act_layer="mish"), device="meta")


# ---------------------------------------------------------------- host orchestration on emulated kernels
SMALL = {
    # 37 x 44 at p 7: a 5 x 6 grid smaller than the kernel, the remainder dropped
    "k7_relu": dict(input_size=(37, 44), patch_size=(7, 7), embed_dim=32, depth=2, kernel_size=7, act_layer="relu",
                    nb_classes=5),
    "k9_gelu": dict(input_size=(52, 40), patch_size=(4, 4), embed_dim=64, depth=2, kernel_size=9, act_layer="gelu",
                    nb_classes=3),
    "1x1": dict(input_size=(9, 8), patch_size=(7, 7), embed_dim=32, depth=2, kernel_size=9, act_layer="gelu",
                nb_classes=0),
    "2x3": dict(input_size=(14, 21), patch_size=(7, 7), embed_dim=32, depth=1, kernel_size=7, act_layer="relu",
                nb_classes=4),
}


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def _small(convmixer, kind, precision, batch=2):
    from oracle import convmixer as oc
    from oracle import params

    cfg = convmixer.ConvMixerConfig(name="t", **SMALL[kind])
    m = convmixer.ConvMixer(cfg, precision=precision, device="cpu")
    w = params.random_params(oc.param_shapes(cfg), seed=7)
    m.load_weights_dict(w)
    return m, cfg, w, params.test_images(batch, *cfg.input_size)


def test_param_specs_equal_the_oracle_tables(convmixer):
    import tfimm
    from oracle import convmixer as oc

    for name in ("convmixer_768_32", "convmixer_1024_20_ks9_p14", "convmixer_1536_20"):
        cfg = tfimm.models.registry.model_config(name)
        m = convmixer.ConvMixer(cfg, device="meta")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(oc.param_shapes(cfg).items())
        keys = list(m.params)
        n_trainable = sum(w.trainable for w in m.weights)
        assert all("/moving_" in k for k in keys[n_trainable:]) and keys[n_trainable] == "stem/2/moving_mean"


@pytest.mark.parametrize("kind", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(convmixer, cpu_engine, kind):
    """The host graph with every kernel replaced by its float64 statement (fp32 storage) is the oracle's forward: the
    BN carried into the next reader equals the BN applied where the reference applies it."""
    from convmixer_oracle import emulated_convmixer_ops
    from oracle import convmixer as oc

    m, cfg, w, x = _small(convmixer, kind, "fp32")
    with emulated_convmixer_ops():
        y, feats = m(x, return_features=True)
    ref, rfeats = oc.forward(cfg, w, x, return_features=True)
    assert list(feats) == list(rfeats) == m.feature_names
    for k in rfeats:
        assert feats[k].shape == rfeats[k].shape, k
        assert (feats[k].double() - rfeats[k]).abs().max().item() <= 1e-5 * rfeats[k].abs().max().item(), k


def test_uint8_input_is_preprocessed(convmixer, cpu_engine):
    from convmixer_oracle import emulated_convmixer_ops
    from oracle import convmixer as oc

    m, cfg, w, _ = _small(convmixer, "2x3", "fp32")
    px = torch.randint(0, 256, (2, *cfg.input_size, 3), dtype=torch.uint8)
    mean, std = torch.tensor(cfg.mean), torch.tensor(cfg.std)
    with emulated_convmixer_ops():
        y = m(px)
    ref = oc.forward(cfg, w, (px.double() / 255 - mean.double()) / std.double())
    assert (y.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


def test_input_smaller_than_a_patch_is_refused(convmixer, cpu_engine):
    m, cfg, w, _ = _small(convmixer, "2x3", "fp32")
    with pytest.raises(ValueError, match="at least 7 x 7"):
        m(torch.zeros((1, 6, 30, 3)))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", list(SMALL))
def test_shadow_rehearsal_float32_stand_in(convmixer, cpu_engine, kind, precision):
    """The op-by-op harness on CPU: the float32 model of the kernel's folded algorithm and the float32 evaluation of
    the other statements play the kernels; every launch is inside its bound and the ConvMixer launchers are reached."""
    from convmixer_oracle import emulated_convmixer_ops, kernel_forms, shadowed_convmixer_ops

    m, cfg, w, x = _small(convmixer, kind, precision)
    with emulated_convmixer_ops(torch.float32), kernel_forms(), shadowed_convmixer_ops() as census:
        m(x, return_features=True)
    census.assert_ok()
    assert {"dwconv", "affine", "im2col", "gemm", "global_avg_pool"} <= census.ops(), census.ops()


def _defect(name):
    """(launcher, float32 stand-in with one seeded defect)."""
    import convmixer_oracle as co

    def folded(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype, x_of=None, resid_a=False, bn1_first=False,
               transpose=False):
        """The folded form in float32; x_of(a, s, t) -> the padded x (B, H + k - 1, W + k - 1, C)."""
        from oracle import emulate_bf16 as emu

        k, C = co._k(taps), a.shape[-1]
        p = (k - 1) // 2
        if transpose:
            taps = taps.reshape(k, k, C).transpose(0, 1).reshape(k * k, C)
        xp = x_of(a, s_in, t_in) if x_of else F.pad(s_in * a + t_in, (0, 0, p, p, p, p))
        z = F.conv2d(xp.permute(0, 3, 1, 2), taps.t().reshape(C, 1, k, k), bias, groups=C).permute(0, 2, 3, 1)
        h = emu._act(s1 * z + t1, act) if bn1_first else s1 * emu._act(z, act) + t1
        return (h + (a if resid_a else xp[:, p:-p, p:-p])).to(out_dtype).contiguous()

    if name == "bn_shift_on_padding":
        def f(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
            k = co._k(taps)
            p = (k - 1) // 2
            return folded(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype,
                          x_of=lambda a, s, t: s * F.pad(a, (0, 0, p, p, p, p)) + t)
        return "dwconv", f
    if name == "padding_masked_by_value":
        def f(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
            k = co._k(taps)
            p = (k - 1) // 2

            def x_of(a, s, t):
                ap = F.pad(a, (0, 0, p, p, p, p))
                return torch.where(ap == 0, torch.zeros_like(ap), s * ap + t)
            return folded(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype, x_of=x_of)
        return "dwconv", f
    if name == "residual_from_a":
        def f(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
            return folded(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype, resid_a=True)
        return "dwconv", f
    if name == "bn1_before_act":
        def f(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
            return folded(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype, bn1_first=True)
        return "dwconv", f
    if name == "taps_transposed":
        def f(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
            return folded(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype, transpose=True)
        return "dwconv", f
    if name == "block0_previous_bn_dropped":
        calls = []

        def f(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype):
            calls.append(1)
            if len(calls) == 1:
                s_in, t_in = torch.ones_like(s_in), torch.zeros_like(t_in)
            return co.kernel_form(a, s_in, t_in, taps, bias, s1, t1, act, out_dtype)
        return "dwconv", f
    if name == "head_pooled_without_shift":
        def f(x, alpha, beta, out_dtype):
            return (alpha * x).to(out_dtype)
        return "affine", f
    raise KeyError(name)


@pytest.mark.parametrize("defect,kind", [("bn_shift_on_padding", "k9_gelu"), ("padding_masked_by_value", "k7_relu"),
                                         ("residual_from_a", "2x3"), ("bn1_before_act", "k9_gelu"),
                                         ("taps_transposed", "k7_relu"), ("block0_previous_bn_dropped", "1x1"),
                                         ("head_pooled_without_shift", "k9_gelu")])
def test_seeded_defects_are_rejected(convmixer, cpu_engine, defect, kind):
    """Each seeded defect makes the harness fail, and the failing rows name the launcher that carries it."""
    from convmixer_oracle import emulated_convmixer_ops, kernel_forms, shadowed_convmixer_ops
    from tfimm.backend import convmixer_ops, mixer_ops

    m, cfg, w, x = _small(convmixer, kind, "fp32", batch=3)
    op, bad = _defect(defect)
    with emulated_convmixer_ops(torch.float32), kernel_forms():
        setattr(convmixer_ops if op == "dwconv" else mixer_ops, op, bad)
        with shadowed_convmixer_ops() as census:
            m(x)
    fails = census.failures()
    assert fails and {r["op"] for r in fails} == {op}, census.table()


def test_padding_mask_matters_on_relu_zeros():
    """With ReLU, exact zeros are common inside the image: a value mask and a position mask differ there."""
    import convmixer_oracle as co

    torch.manual_seed(0)
    a = torch.relu(torch.randn(1, 5, 6, 32))
    assert (a == 0).float().mean() > 0.3
    s, t = torch.rand(32) + 0.5, torch.randn(32)
    taps, bias, s1, t1 = torch.randn(49, 32), torch.randn(32), torch.rand(32), torch.randn(32)
    good = co.dwconv(a, s, t, taps, bias, s1, t1, "relu", torch.float32)
    bad = _defect("padding_masked_by_value")[1](a, s, t, taps, bias, s1, t1, "relu", torch.float32)
    assert (good - bad).abs().max() > 1e-2
