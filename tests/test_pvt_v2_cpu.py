"""PVT v2 without a GPU: the registrations and configs against the extracted zoo, the engine's variable table against
the oracle's, the refusals, the input geometry, and -- where the reference sources are present -- the float64 oracle
(oracle/pvt_v2.py) against the unmodified reference module run on the TensorFlow shim (oracle/pvt_v2_ref.py), the
variable tables in the reference's order; the ConvFFN statement's bound against four defects evaluated in float64; and
the host graph on emulated kernels (CPU engine): the fp32 orchestration against the oracle, the op-by-op harness
rehearsed with float32 stand-ins in every precision, and ten seeded defects, each rejected and named by the launcher
that carries it."""
import dataclasses
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tensorflow-image-models_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import pvt_v2_oracle as pvo  # noqa: E402
from oracle import params  # noqa: E402
from oracle import pvt_v2 as op  # noqa: E402
from oracle import ref_runner as rr  # noqa: E402

NAMES = ["pvt_v2_b0", "pvt_v2_b1", "pvt_v2_b2", "pvt_v2_b3", "pvt_v2_b4", "pvt_v2_b5"]
_SMALL = dict(embed_dim=(32, 64, 32, 64), nb_heads=(1, 1, 1, 1), nb_blocks=(1, 1, 1, 1), mlp_ratio=(2.0, 2.0, 2.0, 1.0))
# (config fields, image size): grids 16 x 16 .. 2 x 2; a 200 x 264 image (50 x 66, 25 x 33, 13 x 17, 7 x 9: the padded
# convolutions round up and no sr ratio divides); no head
CASES = {
    "pin_pvt_v2_plain": (dict(input_size=(64, 64), sr_ratio=(4, 2, 2, 1), nb_classes=5, **_SMALL), (64, 64)),
    "pin_pvt_v2_odd": (dict(input_size=(64, 64), sr_ratio=(8, 4, 2, 1), nb_classes=4, **_SMALL), (200, 264)),
    "pin_pvt_v2_noclass": (dict(input_size=(32, 32), sr_ratio=(2, 1, 1, 1), nb_classes=0, **_SMALL), (32, 32)),
}

needs_reference = pytest.mark.skipif(not rr.available(), reason="the reference sources are not present")


@pytest.fixture
def pvt_v2():
    with pvo.pvt_v2_registered() as mod:
        yield mod


def test_registrations(pvt_v2):
    import tfimm

    assert tfimm.list_models(module="pvt_v2") == NAMES
    cfg = tfimm.models.registry.model_config("pvt_v2_b0")
    assert cfg.embed_dim == (32, 64, 160, 256) and cfg.nb_heads == (1, 2, 5, 8) and cfg.nb_blocks == (2, 2, 2, 2)
    assert tfimm.models.registry.model_config("pvt_v2_b5").mlp_ratio == (4.0, 4.0, 4.0, 4.0)


@pytest.mark.parametrize("name", NAMES)
def test_variable_table_matches_the_oracle(pvt_v2, name):
    import tfimm

    cfg = tfimm.models.registry.model_config(name)
    m = pvt_v2.PyramidVisionTransformerV2(cfg, precision="fp32", device="cpu")
    assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(op.param_shapes(cfg).items())


@pytest.mark.parametrize("bad", [dict(linear_sr=True), dict(nb_heads=(2, 2, 5, 8)), dict(nb_heads=(1, 4, 5, 8)),
                                 dict(norm_layer="batch_norm"), dict(act_layer="mish")])
def test_refusals(pvt_v2, bad):
    import tfimm

    cfg = dataclasses.replace(tfimm.models.registry.model_config("pvt_v2_b0"), **bad)
    with pytest.raises(ValueError):
        pvt_v2.PyramidVisionTransformerV2(cfg, precision="bf16", device="cpu")


def test_grids_and_small_inputs(pvt_v2):
    assert pvt_v2.grids((224, 224), 4) == ((56, 56), (28, 28), (14, 14), (7, 7))
    assert pvt_v2.grids((200, 264), 4) == ((50, 66), (25, 33), (13, 17), (7, 9))
    import tfimm

    m = pvt_v2.PyramidVisionTransformerV2(tfimm.models.registry.model_config("pvt_v2_b0"), precision="fp32",
                                          device="cpu")
    assert m._check_input(224, 224) == ((56, 56), (28, 28), (14, 14), (7, 7))
    assert m._check_input(100, 100) == ((25, 25), (13, 13), (7, 7), (4, 4))
    with pytest.raises(ValueError):
        m._check_input(20, 20)   # stage 0's 5 x 5 grid is smaller than its sr ratio 8


def test_conv_mlp_bound_rejects_seeded_defects():
    """The ConvFFN statement's bound separates the correct arithmetic from the defects a fused kernel could carry:
    padding cells taken as fc1(0) + b1 = b1, transposed taps, the activation before b_dw, and no bf16 rounding of the
    hidden tensor between fc1 and the depthwise convolution (all evaluated in float64)."""
    g = torch.Generator().manual_seed(5)
    B, gh, gw, C, hidden = 2, 5, 6, 32, 64
    M = B * gh * gw
    h = torch.randn((M, C), generator=g).to(torch.bfloat16)
    w1 = (torch.randn((hidden, C), generator=g) * C ** -0.5).to(torch.bfloat16)
    b1, bdw = torch.randn(hidden, generator=g), torch.randn(hidden, generator=g)
    wdw = torch.randn((9, hidden), generator=g) / 3.0
    w2 = (torch.randn((C, hidden), generator=g) * hidden ** -0.5).to(torch.bfloat16)
    b2, res = torch.randn(C, generator=g), torch.randn((M, C), generator=g)
    args = (h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu")
    ref = pvo.pvt_v2_conv_mlp_bf16(*args).double()
    bound = pvo.conv_mlp_bound(*args)
    assert (bound > 0).all()

    def chain(pad_value=False, transpose=False, act_first=False, round_hidden=True):
        hid = h.double() @ w1.double().t() + b1.double()
        if round_hidden:
            hid = hid.to(torch.bfloat16).double()
        x = hid.view(B, gh, gw, hidden).permute(0, 3, 1, 2)
        x = torch.nn.functional.pad(x, (1, 1, 1, 1))
        if pad_value:   # padding cells hold b1 instead of 0
            x = x + (1 - torch.nn.functional.pad(torch.ones(1, 1, gh, gw, dtype=torch.float64), (1, 1, 1, 1))) * \
                b1.double().view(1, -1, 1, 1)
        wt = wdw.double().view(3, 3, hidden)
        if transpose:
            wt = wt.transpose(0, 1)
        z = torch.nn.functional.conv2d(x, wt.permute(2, 0, 1)[:, None], groups=hidden).permute(0, 2, 3, 1)
        z = z.reshape(M, hidden)
        from oracle import emulate_bf16 as emu

        a = emu._act(z, "gelu") + bdw.double() if act_first else emu._act(z + bdw.double(), "gelu")
        a = a.to(torch.bfloat16).double()
        return (res.double() + (a @ w2.double().t() + b2.double())).float().double()

    assert ((chain() - ref).abs() <= bound).all()
    for defect in (dict(pad_value=True), dict(transpose=True), dict(act_first=True), dict(round_hidden=False)):
        assert ((chain(**defect) - ref).abs() > bound).any(), defect


# ------------------------------------------------------------------------------------------ against the reference
def _ref_model(name, fields):
    from oracle import pvt_v2_ref

    pvt_v2_ref.register_test_model(name, **fields)
    ref = pvt_v2_ref.create_model(name)
    with rr._reference_modules(), torch.no_grad():
        ref.model(ref.model.dummy_inputs, training=False)
    return ref


@needs_reference
def test_reference_registrations_and_configs(pvt_v2):
    import tfimm
    from oracle import pvt_v2_ref

    assert pvt_v2_ref.list_models("pvt_v2") == NAMES
    for name in NAMES:
        ref_cfg = pvt_v2_ref.model_config(name)
        ours = dataclasses.asdict(tfimm.models.registry.model_config(name))
        for k, v in ref_cfg.items():
            assert ours[k] == (tuple(v) if isinstance(v, list) else v), (name, k)


@needs_reference
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_the_reference(case):
    fields, size = CASES[case]
    from tfimm.architectures.pvt_v2 import PyramidVisionTransformerV2Config

    cfg = PyramidVisionTransformerV2Config(name=case, **fields)
    rr.set_floatx("float64")
    try:
        ref = _ref_model(case, fields)
        shapes = ref.weight_shapes()
        assert [(k, tuple(v)) for k, v in shapes.items()] == list(op.param_shapes(cfg).items())
        w = params.random_params(shapes, seed=71, dtype=torch.float64)
        ref.assign(w)
        x = params.test_images(2, *size).double()
        y, feats = ref(x, return_features=True)
        yo, fo = op.forward(cfg, w, x, return_features=True)
    finally:
        rr.set_floatx("float32")
    assert list(fo) == list(feats)
    for k in feats:
        a, b = torch.as_tensor(fo[k]).double(), torch.as_tensor(feats[k]).double()
        assert a.shape == b.shape, k
        assert (a - b).abs().max().item() <= 1e-12 * max(1.0, b.abs().max().item()), k
    assert (torch.as_tensor(yo) - torch.as_tensor(y)).abs().max().item() <= 1e-12 * max(1.0, y.abs().max().item())


# ---------------------------------------------------------------- host orchestration on emulated kernels
SMALL = {k: v for k, v in zip(("plain", "odd", "noclass"), CASES.values())}


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def _small(pvt_v2, kind, precision, batch=2):
    fields, size = SMALL[kind]
    cfg = pvt_v2.PyramidVisionTransformerV2Config(name="t", **fields)
    m = pvt_v2.PyramidVisionTransformerV2(cfg, precision=precision, device="cpu")
    w = params.random_params(op.param_shapes(cfg), seed=5)
    m.load_weights_dict(w)
    return m, cfg, w, params.test_images(batch, *size)


@pytest.mark.parametrize("kind", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(pvt_v2, cpu_engine, kind):
    """The host graph with every kernel replaced by its float64 statement (fp32 storage) is the oracle's forward, every
    feature with the reference's name and shape.  The fp32 storage points alone keep it within 1e-6 of each feature's
    largest value (measured: 1.2-1.3e-7)."""
    m, cfg, w, x = _small(pvt_v2, kind, "fp32")
    with pvo.emulated_pvt_v2_ops():
        y, feats = m(x, return_features=True)
        y_plain = m(x)
    ref, rfeats = op.forward(cfg, w, x, return_features=True)
    assert list(feats) == list(rfeats) == m.feature_names
    for k in rfeats:
        assert feats[k].shape == rfeats[k].shape, k
        assert (feats[k].double() - rfeats[k]).abs().max().item() <= 1e-6 * rfeats[k].abs().max().item(), k
    assert torch.equal(y, y_plain)


@pytest.mark.parametrize("kind", list(SMALL))
def test_orchestration_catches_a_host_side_eps(pvt_v2, cpu_engine, monkeypatch, kind):
    """The harness builds each statement from the arguments the host passes, so it cannot see the host passing a wrong
    eps; the comparison above does: with eps 1e-6 for the patch embeddings' and the spatial reduction's LayerNorm
    (instead of the reference's "layer_norm", 1e-5) some feature is more than 1e-6 off (measured: 2-3e-5)."""
    monkeypatch.setattr(pvt_v2, "_EMBED_EPS", 1e-6)
    m, cfg, w, x = _small(pvt_v2, kind, "fp32")
    with pvo.emulated_pvt_v2_ops():
        _, feats = m(x, return_features=True)
    _, rfeats = op.forward(cfg, w, x, return_features=True)
    assert any((feats[k].double() - rfeats[k]).abs().max().item() > 1e-6 * rfeats[k].abs().max().item()
               for k in rfeats)


@pytest.mark.parametrize("precision", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("kind", list(SMALL))
def test_shadow_rehearsal_float32_stand_in(pvt_v2, cpu_engine, kind, precision):
    """The op-by-op harness on CPU: the float32 evaluation of every statement plays the kernels; every launch is inside
    its bound and the PVT v2 launchers of the precision are reached."""
    m, cfg, w, x = _small(pvt_v2, kind, precision)
    with pvo.emulated_pvt_v2_ops(torch.float32), pvo.shadowed_pvt_v2_ops() as census:
        m(x)
    census.assert_ok()
    want = {"im2col", "gemm", "layernorm", "global_avg_pool",
            "pvt_v2_sr_attention_bf16" if precision == "bf16" else "pvt_v2_sr_attention_f32",
            "pvt_sr_attention_bf16" if precision == "bf16" else "pvt_sr_attention_f32",
            "pvt_v2_conv_mlp_bf16" if precision == "bf16" else "dwconv_bias_act"}
    assert want <= census.ops(), census.ops()


def _conv_mlp_defect(pad_b1=False, transpose=False, act_first=False, round_hidden=True):
    """A float32 stand-in of pvt_v2_conv_mlp_bf16 with one seeded defect."""
    from oracle import emulate_bf16 as emu

    F = torch.nn.functional

    def f(h, w1, b1, wdw, bdw, w2, b2, residual, B, gh, gw, act, out=None):
        f32, hidden = torch.float32, w1.shape[0]
        hid = h.to(f32) @ w1.to(f32).t() + b1
        if round_hidden:
            hid = hid.to(torch.bfloat16).to(f32)
        x = F.pad(hid.view(B, gh, gw, hidden).permute(0, 3, 1, 2), (1, 1, 1, 1))
        if pad_b1:   # padding cells hold fc1(0) + b1 = b1
            x = x + (1 - F.pad(torch.ones(1, 1, gh, gw), (1, 1, 1, 1))) * b1.view(1, -1, 1, 1)
        wt = wdw.view(3, 3, hidden)
        if transpose:
            wt = wt.transpose(0, 1)
        z = F.conv2d(x, wt.permute(2, 0, 1)[:, None].contiguous(), groups=hidden).permute(0, 2, 3, 1)
        z = z.reshape(-1, hidden)
        a = emu._act(z, act) + bdw if act_first else emu._act(z + bdw, act)
        y = residual + (a.to(torch.bfloat16).to(f32) @ w2.to(f32).t() + b2)
        if out is not None:
            out.copy_(y)
            return out
        return y
    return f


def _defect(name, m):
    """A float32 stand-in of a launcher with one seeded defect: (launcher module, launcher name, function).  ``m``'s
    plan tells the stand-ins of the shared layernorm launcher which LayerNorm they are running."""
    from oracle import emulate_bf16 as emu
    from tfimm.backend import ops, pvt_v2_ops

    def norms(key):
        out = set()
        for st in m._plan["stages"]:
            if key in st:
                out.add(st[key][0].data_ptr())
            for blk in st["blocks"]:
                if key in blk:
                    out.add(blk[key][0].data_ptr())
        return out

    conv = {"dwconv_padding_b1": dict(pad_b1=True), "dwconv_taps_transposed": dict(transpose=True),
            "act_before_dw_bias": dict(act_first=True), "hidden_not_rounded": dict(round_hidden=False)}
    if name in conv:
        return pvt_v2_ops, "pvt_v2_conv_mlp_bf16", _conv_mlp_defect(**conv[name])
    if name == "patch_embed_padding_0":
        def f(x, ks, stride, padding, out_dtype, groups=1, pre=None):
            if isinstance(padding, int) and padding > 0:   # the windows start at the image's corner, not k // 2 before
                p = 2 * padding
                xs = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (0, p, 0, p)).permute(0, 2, 3, 1).contiguous()
                cols, Ho, Wo = emu.im2col(xs, ks, stride, "valid", out_dtype, groups, pre)
                H, W = emu.conv_geometry(x.shape[1], x.shape[2], ks, stride, padding)[:2]
                cols = cols.view(x.shape[0], Ho, Wo, -1)[:, :H, :W].reshape(x.shape[0] * H * W, -1)
                return cols.contiguous(), H, W
            return emu.im2col(x, ks, stride, padding, out_dtype, groups, pre)
        return ops, "im2col", f
    if name in ("patch_embed_ln_eps_1e-6", "sr_norm_eps_1e-6", "stage_norm_skipped"):
        key = {"patch_embed_ln_eps_1e-6": "pe_n", "sr_norm_eps_1e-6": "srn", "stage_norm_skipped": "norm"}[name]

        def f(x, gamma, beta, eps, out_dtype, out=None):
            if gamma.data_ptr() not in norms(key):
                return emu.layernorm(x, gamma, beta, eps, out_dtype, out)
            if key == "norm":
                return x.to(out_dtype).clone()
            return emu.layernorm(x, gamma, beta, 1e-6, out_dtype, out)
        return ops, "layernorm", f
    if name == "features_from_token_0":
        def f(x):
            B, C = x.shape[0], x.shape[-1]
            return x.to(torch.float32).reshape(B, -1, C)[:, 0].clone()
        return ops, "global_avg_pool", f
    if name == "dh32_k_v_swapped":
        def f(q, kv, B, N, Nk, H, dh, scale):
            swapped = kv.view(B * Nk, 2, H * dh).flip(1).reshape(B * Nk, -1)
            return pvo.pvt_v2_sr_attention_bf16(q, swapped, B, N, Nk, H, dh, scale)
        return pvt_v2_ops, "pvt_v2_sr_attention_bf16", f
    raise KeyError(name)


@pytest.mark.parametrize("defect,kind,precision", [
    ("dwconv_padding_b1", "plain", "bf16"), ("dwconv_taps_transposed", "plain", "bf16"),
    ("act_before_dw_bias", "plain", "bf16"), ("hidden_not_rounded", "plain", "bf16"),
    ("patch_embed_padding_0", "odd", "fp32"), ("patch_embed_ln_eps_1e-6", "plain", "fp32"),
    ("sr_norm_eps_1e-6", "odd", "fp32"), ("stage_norm_skipped", "plain", "fp32"),
    ("features_from_token_0", "plain", "fp32"), ("dh32_k_v_swapped", "plain", "bf16")])
def test_seeded_defects_are_rejected(pvt_v2, cpu_engine, defect, kind, precision):
    """Each seeded defect makes the harness fail, and the failing rows name the launcher that carries it."""
    m, cfg, w, x = _small(pvt_v2, kind, precision, batch=3)
    m._ensure_plan()
    module, name, bad = _defect(defect, m)
    with pvo.emulated_pvt_v2_ops(torch.float32):
        setattr(module, name, bad)
        with pvo.shadowed_pvt_v2_ops() as census:
            m(x)
    fails = census.failures()
    assert fails and {r["op"] for r in fails} == {name}, census.table()
