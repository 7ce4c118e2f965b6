"""MLP-Mixer family on CPU: opt-in registration (and the registry left as it was found), the variable tables against
the float64 oracle's, the C entry points, the plan-time GLU layouts and the refusals."""
import importlib
import json
import subprocess
import sys
from copy import deepcopy
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture
def mixer():
    """Registers the MLP-Mixer models for one test and restores the registry afterwards, so that the exact
    ``list_models()`` / ``list_modules()`` of tests/test_api_cpu.py hold in any test order."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.mlp_mixer"
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
            "'tfimm.architectures.mlp_mixer' in sys.modules)").format(ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == "False"
    assert "mlp_mixer" not in " ".join(out)


def test_registrations_and_variable_tables(mixer):
    import tfimm
    from oracle import mlp_mixer as om

    table = json.loads((ROOT / "tensorflow-image-models_b200/tfimm/architectures/zoo/mlp_mixer.json").read_text())
    names = tfimm.list_models(module="mlp_mixer")
    assert sorted(names) == sorted(table) and len(names) == 26
    for name in names:
        cfg = tfimm.models.registry.model_config(name)
        assert tfimm.models.registry.model_class(name) is mixer.MLPMixer
        for k, v in table[name].items():
            if not k.startswith("__"):
                got = getattr(cfg, k)
                assert (list(got) if isinstance(got, tuple) else got) == v, (name, k)
        m = mixer.MLPMixer(cfg, device="meta")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(om.param_shapes(cfg).items()), name


def test_initial_values(mixer):
    cfg = mixer.MLPMixerConfig(name="t", input_size=(32, 32), patch_size=8, embed_dim=16, nb_blocks=1,
                               mlp_ratio=(4.0, 4.0), block_layer="res_block", norm_layer="affine", init_values=1e-5)
    m = mixer.MLPMixer(cfg, device="cpu")
    assert torch.all(m.params["blocks/0/ls1"] == 1e-5) and torch.all(m.params["blocks/0/ls2"] == 1e-5)
    assert torch.all(m.params["blocks/0/norm1/alpha"] == 1) and torch.all(m.params["blocks/0/norm1/beta"] == 0)
    cfg = mixer.MLPMixerConfig(name="t", input_size=(32, 32), patch_size=8, embed_dim=16, nb_blocks=1,
                               mlp_ratio=(6.0, 6.0), block_layer="spatial_gating_block", mlp_layer="gated_mlp")
    m = mixer.MLPMixer(cfg, device="cpu")
    assert torch.all(m.params["blocks/0/mlp_channels/gate/proj/bias"] == 1)


def test_glu_interleave_layouts():
    from tfimm.backend import mixer_ops

    F, K = 2 * 12, 5
    w = torch.arange(F, dtype=torch.float64)[:, None].repeat(1, K)
    b = torch.arange(F, dtype=torch.float64)
    # pairwise (bf16 channel GLU): rows 2j / 2j + 1 = value j / gate j
    wi, bi = mixer_ops.glu_interleave(w, b, False)
    assert bi.tolist() == [v for j in range(12) for v in (j, 12 + j)]
    assert torch.equal(wi[:, 0], bi)
    # rows (token GLU, fp32 channel GLU): per 16 rows 8 values then their 8 gates, halves zero-padded to 16
    wi, bi = mixer_ops.glu_interleave(w, b, True)
    exp = []
    for q in range(2):
        exp += [float(j) if j < 12 else 0.0 for j in range(8 * q, 8 * q + 8)]
        exp += [float(12 + j) if j < 12 else 0.0 for j in range(8 * q, 8 * q + 8)]
    assert bi.tolist() == exp and wi.shape == (32, K) and torch.equal(wi[:, 0], bi)


def test_entry_points_declared():
    from tfimm.backend import lib

    header = (ROOT / "include" / "tfimm_b200.h").read_text()
    for name in ("tfimm_b200_token_gemm_bf16", "tfimm_b200_token_gemm_f32", "tfimm_b200_gemm_glu_bf16",
                 "tfimm_b200_gemm_glu_f32", "tfimm_b200_affine"):
        assert name in lib.SIGNATURES and f"int {name}(" in header
        assert getattr(lib.load(), name) is not None


def test_refusals(mixer):
    import tfimm

    with pytest.raises(ValueError, match="tf32"):
        tfimm.create_model("mixer_s32_224", precision="tf32", device="cpu")
    cfg = mixer.MLPMixerConfig(name="t", input_size=(32, 32), patch_size=8, embed_dim=16, nb_blocks=1)
    m = mixer.MLPMixer(cfg, device="cpu")
    with pytest.raises(ValueError, match="Input size"):
        m(torch.zeros((1, 40, 32, 3)))
    with pytest.raises(NotImplementedError):
        m(torch.zeros((1, 32, 32, 3)), training=True)
    with pytest.raises(ValueError, match="normalization"):
        mixer.MLPMixer(mixer.MLPMixerConfig(name="t", norm_layer="batch_norm"), device="meta")
    assert m.feature_names == ["stem", "block_0", "features_all", "features", "logits"]


# ---------------------------------------------------------------- host orchestration on emulated kernels
SMALL = {
    "mixer": dict(input_size=(28, 28), patch_size=4, embed_dim=16, nb_blocks=2, mlp_ratio=(0.5, 4.0), nb_classes=5),
    "gmixer": dict(input_size=(20, 24), patch_size=4, embed_dim=16, nb_blocks=2, mlp_ratio=(1.0, 4.0),
                   mlp_layer="glu_mlp", act_layer="swish", nb_classes=5),
    "resmlp": dict(input_size=(28, 28), patch_size=4, embed_dim=16, nb_blocks=2, mlp_ratio=(4.0, 4.0),
                   block_layer="res_block", norm_layer="affine", init_values=0.1, nb_classes=5),
    "gmlp": dict(input_size=(20, 24), patch_size=4, embed_dim=16, nb_blocks=2, mlp_ratio=(6.0, 6.0),
                 block_layer="spatial_gating_block", mlp_layer="gated_mlp", nb_classes=5),
}


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def _small(mixer, kind, precision):
    from oracle import mlp_mixer as om
    from oracle import params

    cfg = mixer.MLPMixerConfig(name="t", **SMALL[kind])
    m = mixer.MLPMixer(cfg, precision=precision, device="cpu")
    w = params.random_params(om.param_shapes(cfg), seed=5)
    m.load_weights_dict(w)
    return m, cfg, w, params.test_images(2, *cfg.input_size)


@pytest.mark.parametrize("kind", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(mixer, cpu_engine, kind):
    """The host graph with every kernel replaced by its float64 statement (fp32 storage) is the oracle's forward."""
    sys.path.insert(0, str(ROOT / "tests"))
    from mixer_oracle import emulated_mixer_ops
    from oracle import mlp_mixer as om

    m, cfg, w, x = _small(mixer, kind, "fp32")
    with emulated_mixer_ops():
        y, feats = m(x, return_features=True)
    ref, rfeats = om.forward(cfg, w, x, return_features=True)
    assert list(feats) == list(rfeats)
    assert (y.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", list(SMALL))
def test_shadow_rehearsal_float32_stand_in(mixer, cpu_engine, kind, precision):
    """The op-by-op harness on CPU: the float32 evaluation of each statement plays the kernel; every launch is inside
    its bound and every mixer launcher is reached."""
    sys.path.insert(0, str(ROOT / "tests"))
    from mixer_oracle import emulated_mixer_ops, shadowed_mixer_ops

    m, cfg, w, x = _small(mixer, kind, precision)
    with emulated_mixer_ops(torch.float32), shadowed_mixer_ops() as census:
        m(x)
    census.assert_ok()
    want = {"token_gemm"} | ({"gemm_glu"} if kind == "gmixer" else set()) | ({"affine"} if kind == "resmlp" else set())
    assert want <= census.ops(), census.ops()


def _defect(name):
    """A float32 stand-in of a mixer launcher with one seeded defect."""
    sys.path.insert(0, str(ROOT / "tests"))
    import mixer_oracle as mo

    if name == "bias_per_column":
        def f(wt, x, bias=None, **kw):
            y = mo.token_gemm(wt, x, bias=None, **{**kw, "out": None, "residual": None, "mul": None,
                                                   "out_dtype": torch.float32})
            C = x.shape[2]
            y = y + bias[torch.arange(C) % bias.shape[0]] if bias is not None else y
            return _finish(y, kw)
        return "token_gemm", f
    if name == "glu_pairing_shifted":
        def f(a, w, bias, n_out, act, block_n=0):
            return mo.gemm_glu(a, w.roll(1, 0), bias.roll(1, 0), n_out, act)
        return "gemm_glu", f
    if name == "tile_reads_next_image":
        def f(wt, x, **kw):
            x2 = x.clone()
            x2[:, x.shape[1] // 2:] = x.roll(-1, 0)[:, x.shape[1] // 2:]
            return mo.token_gemm(wt, x2, **kw)
        return "token_gemm", f
    if name == "u_v_swapped":
        def f(wt, x, mul=None, **kw):
            if mul is not None:   # the multiplier read from the v half instead of the u half
                mul = torch.as_strided(mul, mul.shape, mul.stride(), mul.storage_offset() + mul.shape[2])
            return mo.token_gemm(wt, x, mul=mul, **kw)
        return "token_gemm", f
    raise KeyError(name)


def _finish(y, kw):
    """Epilogue tail of a stand-in that computed the plain product: gamma, mul, residual and the store."""
    import mixer_oracle as mo  # noqa: F401

    m_out = y.shape[1] if kw.get("m_out") is None else kw["m_out"]
    y = y[:, :m_out].double()
    if kw.get("act") not in (None, ""):
        from oracle import emulate_bf16 as emu
        y = emu._act(y, kw["act"])
    if kw.get("gamma") is not None:
        y = y * kw["gamma"].double()
    if kw.get("mul") is not None:
        y = y * kw["mul"].double()
    if kw.get("residual") is not None:
        y = y + kw["residual"].double()
    out = kw.get("out")
    if out is not None:
        out.copy_(y.to(out.dtype))
        return out
    return y.to(kw.get("out_dtype") or (kw["residual"].dtype if kw.get("residual") is not None else torch.bfloat16))


@pytest.mark.parametrize("defect,kind", [("bias_per_column", "mixer"), ("glu_pairing_shifted", "gmixer"),
                                         ("tile_reads_next_image", "resmlp"), ("u_v_swapped", "gmlp")])
def test_seeded_defects_are_rejected(mixer, cpu_engine, defect, kind):
    """Each seeded defect makes the harness fail, and the failing row names the launcher that carries it."""
    sys.path.insert(0, str(ROOT / "tests"))
    from mixer_oracle import emulated_mixer_ops, shadowed_mixer_ops
    from tfimm.backend import mixer_ops

    m, cfg, w, x = _small(mixer, kind, "fp32")
    op, bad = _defect(defect)
    with emulated_mixer_ops(torch.float32):
        setattr(mixer_ops, op, bad)
        with shadowed_mixer_ops() as census:
            m(x)
    fails = census.failures()
    assert fails and {r["op"] for r in fails} == {op}, census.table()
