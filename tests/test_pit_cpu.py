"""PiT family on CPU: opt-in registration (and the registry left as it was found), the C entry points' argument checks,
the attention dispatch, the host orchestration on the float64 statements, the float32 shadow rehearsal and seeded
defects."""
import dataclasses
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
def pit():
    """Registers the PiT models for one test and restores the registry afterwards, so that the exact ``list_models()``
    / ``list_modules()`` of the other suites hold in any test order."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.pit"
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
            "'tfimm.architectures.pit' in sys.modules)").format(ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == "False"
    assert "'pit'" not in " ".join(out)


def test_registration_on_import(pit):
    import tfimm

    assert sorted(tfimm.list_models(module="pit")) == sorted(
        f"pit_{s}{d}_224" for s in ("ti", "xs", "s", "b") for d in ("", "_distilled"))
    m = tfimm.create_model("pit_b_distilled_224", device="meta")
    assert isinstance(m, pit.PoolingVisionTransformer) and m.cfg.grid_size == (31, 31) and m.cfg.nb_tokens == 2
    assert len(m.feature_names) == 1 + 13 + 2 + 3


PREFIX = "tfimm_b200_"


def test_entry_point_argument_checks_past_the_shape():
    """Head dims other than 32 / 48 / 64, misaligned pointers and a token copy without token rows are refused before
    any CUDA call."""
    from tfimm.backend import lib, pit_ops

    h = lib.load()
    assert h.tfimm_b200_pit_attention_bf16(16, 16, 2, 197, 4, 40, 0.1, None) == 1
    assert "head_dim must be 32, 48 or 64 (got 40)" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pit_attention_bf16(16, 24, 2, 197, 4, 32, 0.1, None) == 1
    assert "16-byte aligned" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pit_pool(16, 16, 16, 16, 16, 2, 0, 7, 7, 64, None) == 1
    assert "tokens_bf16 given without token rows" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pit_pool(16, 16, 16, 16, None, 2, 1, 7, 7, 66, None) == 1
    assert pit_ops.pool_geometry(27, 27) == (14, 14) and pit_ops.pool_geometry(14, 14) == (7, 7)
    assert pit_ops.pool_geometry(31, 31) == (16, 16) and pit_ops.pool_geometry(16, 16) == (8, 8)
    assert pit_ops.pool_geometry(1, 1) == (1, 1) and pit_ops.pool_geometry(6, 5) == (3, 3)


def test_trace_family_names():
    from tfimm.backend import ops

    sys.path.insert(0, str(ROOT / "tools"))
    import ncu_traffic

    assert ncu_traffic.family_of("void tfimm::(anonymous namespace)::pit_attention_bf16_kernel<48>(const __nv_bfloat16 *)") \
        == "pit_attention_bf16" == ops.TRACE_FAMILY[PREFIX + "pit_attention_bf16"]
    assert ncu_traffic.family_of("tfimm::(anonymous namespace)::pit_pool_kernel(const float *)") == "pit_pool" == \
        ops.TRACE_FAMILY[PREFIX + "pit_pool"]


def test_byte_counts():
    from tfimm.backend import pit_ops

    # 27 x 27 x 64 in, 14 x 14 x 128 out, 10 rows of 128 weights and biases, one token row read in fp32, written in bf16
    assert pit_ops.pool_nbytes(2, 1, 27, 27, 64, True) == 4.0 * (2 * 729 * 64 + 2 * 196 * 128 + 1280) + 2 * 64 * 6.0
    assert pit_ops.pool_nbytes(2, 1, 27, 27, 64, False) == 4.0 * (2 * 729 * 64 + 2 * 196 * 128 + 1280)


def test_attention_dispatch(monkeypatch):
    """bf16 -> pit_attention_bf16 at every head dim (the ViT kernel only where ``vit_kernel_preferred``); fp32 ->
    ops.attention (the SIMT kernel, or TF32 at head dim 64 in a tf32 forward); head dims without a kernel refused."""
    from tfimm.backend import lib, ops, pit_ops

    calls = []
    monkeypatch.setattr(pit_ops, "pit_attention_bf16", lambda qkv, B, T, H, dh, s: calls.append(("pit", T, dh)))
    monkeypatch.setattr(ops, "attention", lambda qkv, B, T, H, dh, s: calls.append(("ops", T, dh)))
    for T, dh in ((731, 32), (198, 48), (963, 64), (258, 64), (66, 64)):
        pit_ops.attention(torch.zeros((T, 3 * dh), dtype=torch.bfloat16), 1, T, 1, dh, 0.1)
        pit_ops.attention(torch.zeros((T, 3 * dh)), 1, T, 1, dh, 0.1)
    want = []
    for T, dh in ((731, 32), (198, 48), (963, 64), (258, 64), (66, 64)):
        vit = ops.attention_bf16_supported(T, dh) and pit_ops.vit_kernel_preferred(T, dh)
        want += [("ops" if vit else "pit", T, dh), ("ops", T, dh)]
    assert calls == want
    assert not pit_ops.vit_kernel_preferred(963, 64) and not pit_ops.vit_kernel_preferred(198, 48)
    with pytest.raises(lib.KernelLibraryError, match="head_dim 80"):
        pit_ops.attention(torch.zeros((5, 240), dtype=torch.bfloat16), 1, 5, 1, 80, 0.1)


def test_refusals(pit):
    C = pit.PoolingVisionTransformerConfig
    with pytest.raises(ValueError, match="normalization"):
        pit.PoolingVisionTransformer(C(name="t", norm_layer="batch_norm"), device="meta")
    with pytest.raises(ValueError, match="head_dim"):
        pit.PoolingVisionTransformer(C(name="t", embed_dim=(80, 160, 320), nb_heads=(1, 2, 4)), device="meta")
    with pytest.raises(ValueError, match="doubles"):
        pit.PoolingVisionTransformer(C(name="t", embed_dim=(64, 96, 192), nb_heads=(2, 3, 6)), device="meta")
    m = pit.PoolingVisionTransformer(C(name="t", input_size=(32, 32), embed_dim=(32, 64, 128), nb_heads=(1, 2, 4),
                                       nb_blocks=(1, 1, 1)), device="cpu")
    with pytest.raises(NotImplementedError):
        m(torch.zeros((1, 32, 32, 3)), training=True)


def test_transform_pos_embed(pit):
    """transform_weights["pos_embed"] resizes the NCHW grid bicubically (tf.image.resize, float32) to the target's."""
    import tfimm
    from oracle import tf_ops

    cfg = tfimm.models.registry.model_config("pit_ti_224")
    m = pit.PoolingVisionTransformer(cfg, device="cpu")
    tgt = dataclasses.replace(cfg, input_size=(288, 160))
    got = cfg.transform_weights["pos_embed"](m, m.params["pos_embed"], tgt)
    assert got.shape == (1, 64, 35, 19)
    ref = tf_ops.resize_bicubic(m.params["pos_embed"].double().permute(0, 2, 3, 1), (35, 19)).permute(0, 3, 1, 2)
    assert (got.double() - ref).abs().max().item() < 1e-6


# ---------------------------------------------------------------- host orchestration on emulated kernels
SMALL = {
    # grid 5 x 5 -> 3 x 3 -> 2 x 2, head dim 32
    "plain": dict(input_size=(48, 48), embed_dim=(32, 64, 128), nb_heads=(1, 2, 4), nb_blocks=(1, 2, 1), nb_classes=5),
    # grid 9 x 13 -> 5 x 7 -> 3 x 4, head dim 48, two token rows
    "dist": dict(input_size=(40, 56), patch_size=8, stride=4, embed_dim=(48, 96, 192), nb_heads=(1, 2, 4),
                 nb_blocks=(1, 1, 2), distilled=True, classifier=("head", "head_dist"), nb_classes=3),
    # grid 6 x 5 -> 3 x 3 -> 2 x 2: an even grid, where TF "same" padding would be asymmetric; head dim 64
    "even": dict(input_size=(56, 48), embed_dim=(64, 128, 256), nb_heads=(1, 2, 4), nb_blocks=(1, 1, 1),
                 distilled=True, classifier=("head", "head_dist"), nb_classes=0),
}


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def _grids(cfg):
    from tfimm.backend import pit_ops

    g = [cfg.grid_size]
    for _ in cfg.nb_blocks[1:]:
        g.append(pit_ops.pool_geometry(*g[-1]))
    return g


def _small(pit, kind, precision, batch=2):
    from oracle import params
    from oracle import pit as op

    cfg = pit.PoolingVisionTransformerConfig(name="t", **SMALL[kind])
    m = pit.PoolingVisionTransformer(cfg, precision=precision, device="cpu")
    w = params.random_params(op.param_shapes(cfg), seed=5)
    m.load_weights_dict(w)
    return m, cfg, w, params.test_images(batch, *cfg.input_size)


def test_param_specs_equal_the_oracle_tables(pit):
    import tfimm
    from oracle import pit as op

    for name in ("pit_ti_224", "pit_b_distilled_224"):
        cfg = tfimm.models.registry.model_config(name)
        m = pit.PoolingVisionTransformer(cfg, device="meta")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(op.param_shapes(cfg).items())
    for kind in SMALL:
        cfg = pit.PoolingVisionTransformerConfig(name="t", **SMALL[kind])
        m = pit.PoolingVisionTransformer(cfg, device="cpu")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(op.param_shapes(cfg).items())


@pytest.mark.parametrize("kind", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(pit, cpu_engine, kind):
    """The host graph with every kernel replaced by its float64 statement (fp32 storage) is the oracle's forward."""
    from oracle import pit as op
    from pit_oracle import emulated_pit_ops

    m, cfg, w, x = _small(pit, kind, "fp32")
    with emulated_pit_ops():
        y, feats = m(x, return_features=True)
    ref, rfeats = op.forward(cfg, w, x, return_features=True)
    assert list(feats) == list(rfeats) == m.feature_names
    for k in rfeats:
        assert feats[k].shape == rfeats[k].shape, k
        assert (feats[k].double() - rfeats[k]).abs().max().item() <= 1e-5 * rfeats[k].abs().max().item(), k


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", list(SMALL))
def test_shadow_rehearsal_float32_stand_in(pit, cpu_engine, kind, precision):
    """The op-by-op harness on CPU: the float32 evaluation of every statement plays the kernels; every launch is inside
    its bound and the PiT launchers of the precision are reached."""
    from pit_oracle import emulated_pit_ops, shadowed_pit_ops
    from tfimm.backend import pit_ops

    m, cfg, w, x = _small(pit, kind, precision)
    with emulated_pit_ops(torch.float32), shadowed_pit_ops() as census:
        m(x)
    census.assert_ok()
    want = {"pit_pool", "assemble_tokens", "im2col", "gemm", "layernorm"}
    if precision == "bf16":
        T = [cfg.nb_tokens + g[0] * g[1] for g in _grids(cfg)]
        dhs = [D // H for D, H in zip(cfg.embed_dim, cfg.nb_heads)]
        vit = [pit_ops.vit_kernel_preferred(t, dh) for t, dh in zip(T, dhs)]
        want |= ({"attention"} if any(vit) else set()) | ({"pit_attention_bf16"} if not all(vit) else set())
    else:
        want.add("attention")
    assert want <= census.ops(), census.ops()


def _defect(name):
    """A float32 stand-in of a launcher with one seeded defect: (launcher module, launcher name, function)."""
    from oracle import emulate_bf16 as emu
    from oracle import tf_ops
    from tfimm.backend import ops, pit_ops

    def grid_nchw(x, B, skip, H, W):
        C = x.shape[1]
        return x.view(B, -1, C)[:, skip:skip + H * W].reshape(B, H, W, C).permute(0, 3, 1, 2)

    def pool_out(x, y, B, nb, tokens_bf16):
        C = x.shape[1]
        out = torch.full((B, nb + y.shape[2] * y.shape[3], 2 * C), float("nan"))
        out[:, nb:] = y.permute(0, 2, 3, 1).reshape(B, -1, 2 * C)
        tok = x.view(B, -1, C)[:, :nb].reshape(B * nb, C).to(torch.bfloat16) if tokens_bf16 else None
        return out.view(-1, 2 * C), tok

    def kernel(w, C):
        return w.view(3, 3, 1, 2 * C).permute(3, 2, 0, 1)

    if name == "conv_reads_o_mod_C":
        def f(x, w, bias, B, nb_tokens, H, W, tokens_bf16=False):
            C = x.shape[1]
            g = grid_nchw(x, B, nb_tokens, H, W)[:, [o % C for o in range(2 * C)]]
            y = F.conv2d(g, kernel(w, C), bias, stride=2, padding=1, groups=2 * C)
            return pool_out(x, y, B, nb_tokens, tokens_bf16)
        return pit_ops, "pit_pool", f
    if name == "same_style_padding":
        def f(x, w, bias, B, nb_tokens, H, W, tokens_bf16=False):
            C = x.shape[1]
            g = grid_nchw(x, B, nb_tokens, H, W)
            (pt, pb), (pl, pr) = tf_ops.same_padding(H, 3, 2), tf_ops.same_padding(W, 3, 2)   # (0, 1) on even sides
            y = F.conv2d(F.pad(g, (pl, pr, pt, pb)), kernel(w, C), bias, stride=2, groups=C)
            return pool_out(x, y, B, nb_tokens, tokens_bf16)
        return pit_ops, "pit_pool", f
    if name == "token_rows_through_conv":
        def f(x, w, bias, B, nb_tokens, H, W, tokens_bf16=False):
            C = x.shape[1]
            y = F.conv2d(grid_nchw(x, B, 0, H, W), kernel(w, C), bias, stride=2, padding=1, groups=C)
            return pool_out(x, y, B, nb_tokens, tokens_bf16)
        return pit_ops, "pit_pool", f
    if name == "pos_on_class_token":
        def f(patches, cls, dist, pos, B, P, out_dtype):
            ntok = 2 if dist is not None else 1
            y = emu.assemble_tokens(patches, cls, dist, pos, B, P, torch.float32).view(B, P + ntok, -1)
            y[:, 0] += pos[ntok]          # the class token picks up the first grid position's embedding
            return y.view(B * (P + ntok), -1).to(out_dtype)
        return ops, "assemble_tokens", f
    if name == "keys_past_T_in_softmax":
        def f(qkv, B, T, H, dh, scale):
            Tp = (T + 63) // 64 * 64      # zero keys up to the 64-key block boundary, not masked
            x = F.pad(qkv.float().view(B, T, 3 * H * dh), (0, 0, 0, Tp - T))
            q, k, v = x.view(B, Tp, 3, H, dh).permute(2, 0, 3, 1, 4)
            o = torch.softmax(scale * q @ k.transpose(-1, -2), -1) @ v
            return o[:, :, :T].permute(0, 2, 1, 3).reshape(B * T, H * dh).to(torch.bfloat16)
        return pit_ops, "pit_attention_bf16", f
    if name == "cls_dist_swapped":
        def f(patches, cls, dist, pos, B, P, out_dtype):
            return emu.assemble_tokens(patches, dist, cls, pos, B, P, out_dtype)
        return ops, "assemble_tokens", f
    raise KeyError(name)


@pytest.mark.parametrize("defect,kind,precision", [
    ("conv_reads_o_mod_C", "plain", "fp32"), ("same_style_padding", "even", "fp32"),
    ("token_rows_through_conv", "dist", "fp32"), ("pos_on_class_token", "dist", "fp32"),
    ("keys_past_T_in_softmax", "dist", "bf16"), ("cls_dist_swapped", "even", "fp32")])
def test_seeded_defects_are_rejected(pit, cpu_engine, defect, kind, precision):
    """Each seeded defect makes the harness fail, and the failing rows name the launcher that carries it."""
    from pit_oracle import emulated_pit_ops, shadowed_pit_ops

    m, cfg, w, x = _small(pit, kind, precision, batch=3)
    module, op, bad = _defect(defect)
    with emulated_pit_ops(torch.float32):
        setattr(module, op, bad)
        with shadowed_pit_ops() as census:
            m(x)
    fails = census.failures()
    assert fails and {r["op"] for r in fails} == {op}, census.table()
