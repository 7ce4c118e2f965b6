"""PoolFormer family on CPU: opt-in registration (and the registry left as it was found), the C entry points and their
ctypes table, the host orchestration on the float64 statements, the float32 shadow rehearsal and seeded defects."""
import ctypes
import importlib
import re
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
def poolformer():
    """Registers the PoolFormer models for one test and restores the registry afterwards, so that the exact
    ``list_models()`` / ``list_modules()`` of the other suites hold in any test order."""
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


def test_import_tfimm_registers_nothing_new():
    code = ("import sys; sys.path[:0] = ['{0}', '{0}/tensorflow-image-models_b200']; import tfimm; "
            "from tfimm.models.registry import list_modules; print(len(tfimm.list_models()), sorted(list_modules()), "
            "'tfimm.architectures.poolformer' in sys.modules)").format(ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == "False"
    assert "poolformer" not in " ".join(out)


def test_registration_on_import(poolformer):
    import tfimm

    assert sorted(tfimm.list_models(module="poolformer")) == [
        "poolformer_m36", "poolformer_m48", "poolformer_s12", "poolformer_s24", "poolformer_s36"]
    m = tfimm.create_model("poolformer_s12", device="meta")
    assert isinstance(m, poolformer.PoolFormer) and m.cfg.init_scale == 1e-5 and m.cfg.crop_pct == 0.9
    assert len(m.feature_names) == 1 + 12 + 3 + 3


PREFIX = "tfimm_b200_"
ZERO_CALL = {
    "gn1_partials": (1, "gn1_partials: need B, H, W > 0 and C % 4 == 0 (B=0 H=0 W=0 C=0)"),
    "poolformer_mixer": (1, "poolformer_mixer: need B, H, W > 0 and C % 4 == 0 (B=0 H=0 W=0 C=0)"),
    "gn1_apply": (1, "gn1_apply: need B, H, W > 0 and C % 4 == 0 (B=0 H=0 W=0 C=0)"),
}


def test_entry_points_reject_all_zero_arguments_with_their_own_message():
    from tfimm.backend import poolformer_ops

    handle = poolformer_ops.load()
    assert {PREFIX + n for n in ZERO_CALL} == set(poolformer_ops.SIGNATURES)
    got = {}
    for name, argtypes in poolformer_ops.SIGNATURES.items():
        args = [None if t is ctypes.c_void_p else 0.0 if t is ctypes.c_float else 0 for t in argtypes]
        got[name[len(PREFIX):]] = (getattr(handle, name)(*args), handle.tfimm_b200_last_error().decode())
    assert got == ZERO_CALL


def test_entry_point_argument_checks_past_the_shape():
    """A wrong chunking and an in-place mixer are refused before any CUDA call."""
    from tfimm.backend import poolformer_ops

    h = poolformer_ops.load()
    assert h.tfimm_b200_gn1_partials(16, 16, 1, 56, 56, 64, 3, None) == 1
    assert "splits 3, the chunking of H*W*C=200704 gives 49" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_poolformer_mixer(16, 16, 16, 16, 16, 32, 1, 7, 7, 64, 1, 1e-5, None) == 1
    assert "must not alias" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_gn1_apply(16, 16, 16, 16, 16, 5, 1, 7, 7, 64, 1, 1e-5, None) == 1
    assert "out_dtype" in h.tfimm_b200_last_error().decode()
    assert poolformer_ops.splits(56, 56, 64) == 49 and poolformer_ops.splits(1, 1, 512) == 1


def test_header_declares_the_ctypes_table():
    """include/tfimm_b200_poolformer.h declares exactly the three entry points, each parameter of the kind the ctypes
    table passes, and the library exports them; the core header does not name them."""
    from tfimm.backend import lib, poolformer_ops

    header = (ROOT / "include" / "tfimm_b200_poolformer.h").read_text()
    assert set(re.findall(r"^int (tfimm_b200_[a-z0-9_]+)\(", header, re.M)) == set(poolformer_ops.SIGNATURES)
    core = (ROOT / "include" / "tfimm_b200.h").read_text()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(lib.LIB_PATH)], capture_output=True, text=True).stdout
    for name, argtypes in poolformer_ops.SIGNATURES.items():
        assert name not in core and name not in lib.SIGNATURES and re.search(r"\sT\s+" + name + r"\b", nm)
        params = [p.strip() for p in re.search(name + r"\s*\(([^;]*?)\)\s*;", header, re.S).group(1).split(",")]
        assert len(params) == len(argtypes), name
        for p, ct in zip(params, argtypes):
            want = ctypes.c_void_p if "*" in p else ctypes.c_float if p.startswith("float") else \
                ctypes.c_long if p.startswith("long") else ctypes.c_int
            assert ct is want, (name, p, ct)


def test_trace_family_names():
    from tfimm.backend import ops, poolformer_ops

    assert poolformer_ops.TRACE_FAMILY == {n: n[len(PREFIX):] for n in poolformer_ops.SIGNATURES}
    assert not set(poolformer_ops.SIGNATURES) & set(ops.TRACE_FAMILY)
    sys.path.insert(0, str(ROOT / "tools"))
    import ncu_traffic

    for kernel in ("gn1_partials_kernel", "poolformer_mixer_kernel", "gn1_apply_kernel<float>"):
        assert ncu_traffic.family_of(f"tfimm::(anonymous namespace)::{kernel}(const float *)") == \
            kernel.split("_kernel")[0]


def test_byte_counts():
    from tfimm.backend import poolformer_ops as po

    N = 7 * 7 * 512   # 25088 values, 7 chunks
    assert po.mixer_nbytes(2, 7, 7, 512) == 4.0 * 2 * (2 * N + 2 * 3 * 7)
    assert po.apply_nbytes(1, 3, 5, 64, torch.bfloat16) == 4.0 * 960 + 2.0 * 960 + 12


def test_refusals(poolformer):
    with pytest.raises(ValueError, match="normalization"):
        poolformer.PoolFormer(poolformer.PoolFormerConfig(name="t", norm_layer="layer_norm"), device="meta")
    with pytest.raises(ValueError, match="multiple of 8"):
        poolformer.PoolFormer(poolformer.PoolFormerConfig(name="t", embed_dim=(12, 16, 24, 32)), device="meta")
    m = poolformer.PoolFormer(poolformer.PoolFormerConfig(name="t", embed_dim=(8, 16, 24, 32), nb_blocks=(1, 1, 1, 1)),
                              device="cpu")
    with pytest.raises(NotImplementedError):
        m(torch.zeros((1, 32, 32, 3)), training=True)


# ---------------------------------------------------------------- host orchestration on emulated kernels
SMALL = {
    "sq64": dict(input_size=(64, 64), embed_dim=(8, 16, 24, 32), nb_blocks=(1, 1, 2, 1), init_scale=0.3,
                 nb_classes=5),
    # stage 0 is 15 x 11 x 32 = 5280 values: two chunks per image
    "odd": dict(input_size=(61, 45), embed_dim=(32, 8, 24, 16), nb_blocks=(1, 2, 1, 1), init_scale=0.5, nb_classes=3),
    "last1x1": dict(input_size=(32, 32), embed_dim=(8, 16, 16, 24), nb_blocks=(1, 1, 1, 2), init_scale=0.4,
                    nb_classes=0),
}


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def _small(poolformer, kind, precision, batch=2):
    from oracle import params
    from oracle import poolformer as op

    cfg = poolformer.PoolFormerConfig(name="t", **SMALL[kind])
    m = poolformer.PoolFormer(cfg, precision=precision, device="cpu")
    w = params.random_params(op.param_shapes(cfg), seed=5)
    for k in w:   # layer scales of a trained model's size, so that the mixer's term is visible
        if "layer_scale" in k:
            w[k] = w[k].abs() + cfg.init_scale
    m.load_weights_dict(w)
    return m, cfg, w, params.test_images(batch, *cfg.input_size)


def test_param_specs_equal_the_oracle_tables(poolformer):
    from oracle import poolformer as op

    for name in ("poolformer_s12", "poolformer_m48"):
        import tfimm

        cfg = tfimm.models.registry.model_config(name)
        m = poolformer.PoolFormer(cfg, device="meta")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(op.param_shapes(cfg).items())
    for kind in SMALL:
        cfg = poolformer.PoolFormerConfig(name="t", **SMALL[kind])
        m = poolformer.PoolFormer(cfg, device="cpu")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(op.param_shapes(cfg).items())
        assert all(torch.all(v == cfg.init_scale) for k, v in m.params.items() if "layer_scale" in k)


@pytest.mark.parametrize("kind", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(poolformer, cpu_engine, kind):
    """The host graph with every kernel replaced by its float64 statement (fp32 storage) is the oracle's forward."""
    from oracle import poolformer as op
    from poolformer_oracle import emulated_poolformer_ops

    m, cfg, w, x = _small(poolformer, kind, "fp32")
    with emulated_poolformer_ops():
        y, feats = m(x, return_features=True)
    ref, rfeats = op.forward(cfg, w, x, return_features=True)
    assert list(feats) == list(rfeats) == m.feature_names
    for k in rfeats:
        assert feats[k].shape == rfeats[k].shape, k
        assert (feats[k].double() - rfeats[k]).abs().max().item() <= 1e-5 * rfeats[k].abs().max().item(), k
    if kind == "last1x1":
        # a 1 x 1 image: the pool is x itself, so the mixer adds exactly nothing
        assert feats["stage_3/block_0"].shape[1:3] == (1, 1)


def test_mixer_is_identity_on_a_1x1_image():
    from poolformer_oracle import poolformer_mixer

    x = torch.randn(3, 1, 1, 16) * 5 + 2
    out, _ = poolformer_mixer(x, None, torch.rand(16), torch.rand(16), torch.rand(16), 1e-5)
    assert torch.equal(out, x)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", list(SMALL))
def test_shadow_rehearsal_float32_stand_in(poolformer, cpu_engine, kind, precision):
    """The op-by-op harness on CPU: float32 models of the PoolFormer kernels' algorithms and the float32 evaluation of
    the other statements play the kernels; every launch is inside its bound and every PoolFormer launcher is reached."""
    from poolformer_oracle import emulated_poolformer_ops, kernel_forms, shadowed_poolformer_ops

    m, cfg, w, x = _small(poolformer, kind, precision)
    with emulated_poolformer_ops(torch.float32), kernel_forms(), shadowed_poolformer_ops() as census:
        m(x)
    census.assert_ok()
    assert {"gn1_partials", "poolformer_mixer", "gn1_apply", "im2col", "gemm"} <= census.ops(), census.ops()


def _defect(name):
    """A float32 stand-in of a PoolFormer launcher with one seeded defect."""
    import poolformer_oracle as po

    def gn(x, gamma, beta, eps, per_channel=False):
        dims = (1, 2) if per_channel else (1, 2, 3)
        mean = x.mean(dim=dims, keepdim=True)
        var = ((x - mean) ** 2).mean(dim=dims, keepdim=True)
        return (x - mean) / torch.sqrt(var + eps) * gamma + beta

    def nchw(f, t):
        return f(t.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)

    if name == "pool_counts_padded_cells":
        def f(x, partials, gamma, beta, ls1, eps):
            n = gn(x, gamma, beta, eps)
            pool = nchw(lambda t: F.avg_pool2d(t, 3, 1, 1, count_include_pad=True), n)
            out = (x + ls1 * (pool - n)).contiguous()
            return out, po.gn1_partials(out)
        return "poolformer_mixer", f
    if name == "beta_on_zero_fill":
        def f(x, partials, gamma, beta, ls1, eps):
            n = gn(x, gamma, beta, eps)
            mean = x.mean(dim=(1, 2, 3), keepdim=True)
            rstd = 1 / torch.sqrt(((x - mean) ** 2).mean(dim=(1, 2, 3), keepdim=True) + eps)
            fill = (0 - mean) * rstd * gamma + beta          # GN of a zero-padded x: the fill is GN(0), not absent
            padded = F.pad(n - fill, (0, 0, 1, 1, 1, 1)) + fill
            pool = nchw(lambda t: F.avg_pool2d(t, 3, 1, 0), padded)
            out = (x + ls1 * (pool - n)).contiguous()
            return out, po.gn1_partials(out)
        return "poolformer_mixer", f
    if name == "stats_per_channel":
        def f(x, partials, gamma, beta, eps, out_dtype):
            B, H, W, C = x.shape
            return gn(x, gamma, beta, eps, per_channel=True).reshape(B * H * W, C).to(out_dtype)
        return "gn1_apply", f
    if name == "merge_drops_last_split":
        def f(x, partials, gamma, beta, eps, out_dtype):
            B, H, W, C = x.shape
            p = partials[:, :-1] if partials.shape[1] > 1 else partials     # an off-by-one in the merge loop
            n = p[..., 0].sum(1)
            mean = (p[..., 0] * p[..., 1]).sum(1) / n
            m2 = (p[..., 2] + p[..., 0] * (p[..., 1] - mean[:, None]) ** 2).sum(1)
            rstd = 1 / torch.sqrt(m2 / n + eps)
            y = (x - mean.view(B, 1, 1, 1)) * rstd.view(B, 1, 1, 1) * gamma + beta
            return y.reshape(B * H * W, C).to(out_dtype)
        return "gn1_apply", f
    if name == "merge_reads_next_image":
        def f(x, partials, gamma, beta, eps, out_dtype):
            return _apply_with_stats_of(x, x.roll(-1, 0), gamma, beta, eps, out_dtype)
        return "gn1_apply", f
    if name == "ls1_on_pool_term_only":
        def f(x, partials, gamma, beta, ls1, eps):
            n = gn(x, gamma, beta, eps)
            out = (x + ls1 * po._pool_same(n) - n).contiguous()
            return out, po.gn1_partials(out)
        return "poolformer_mixer", f
    raise KeyError(name)


def _apply_with_stats_of(x, src, gamma, beta, eps, out_dtype):
    """GN of x with the image statistics of src (the next image's)."""
    B, H, W, C = x.shape
    mean = src.mean(dim=(1, 2, 3), keepdim=True)
    var = ((src - mean) ** 2).mean(dim=(1, 2, 3), keepdim=True)
    return ((x - mean) / torch.sqrt(var + eps) * gamma + beta).reshape(B * H * W, C).to(out_dtype)


@pytest.mark.parametrize("defect,kind", [("pool_counts_padded_cells", "odd"), ("beta_on_zero_fill", "sq64"),
                                         ("stats_per_channel", "sq64"), ("merge_drops_last_split", "odd"),
                                         ("merge_reads_next_image", "last1x1"), ("ls1_on_pool_term_only", "odd")])
def test_seeded_defects_are_rejected(poolformer, cpu_engine, defect, kind):
    """Each seeded defect makes the harness fail, and the failing rows name the launcher that carries it."""
    from poolformer_oracle import emulated_poolformer_ops, kernel_forms, shadowed_poolformer_ops
    from tfimm.backend import poolformer_ops

    m, cfg, w, x = _small(poolformer, kind, "fp32", batch=3)
    op, bad = _defect(defect)
    with emulated_poolformer_ops(torch.float32), kernel_forms():
        setattr(poolformer_ops, op, bad)
        with shadowed_poolformer_ops() as census:
            m(x)
    fails = census.failures()
    assert fails and {r["op"] for r in fails} == {op}, census.table()
