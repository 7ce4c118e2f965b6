"""Segment Anything on CPU: registration (and the registry left as it was found), the variable tables, the host
orchestration of the image encoder with every kernel replaced by its float64 statement (as tests/test_orchestration_cpu
does for the classifiers), weight save / load / resize, and the refusals."""
import importlib
import subprocess
import sys
from copy import deepcopy
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture
def sam():
    """Registers the SAM models for one test and restores the registry afterwards, so that the exact
    ``list_models()`` / ``list_modules()`` of tests/test_api_cpu.py hold in any test order."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.segment_anything.sam"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def _nerr(out, ref):
    out, ref = out.double().cpu(), ref.double().cpu()
    return (out - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)


# small configurations: a padded window grid (10 -> 12 with window 4), head_dim 80, and the unpadded case
SMALL = {
    "pad": dict(input_size=(40, 40), encoder_patch_size=4, encoder_embed_dim=64, encoder_nb_heads=2, encoder_nb_blocks=3,
                encoder_global_attn_indices=(1,), encoder_window_size=4, embed_dim=64, fixed_input_size=False),
    "dh80": dict(input_size=(32, 32), encoder_patch_size=4, encoder_embed_dim=160, encoder_nb_heads=2,
                 encoder_nb_blocks=2, encoder_global_attn_indices=(1,), encoder_window_size=3, embed_dim=64),
    "nopad": dict(input_size=(32, 32), encoder_patch_size=4, encoder_embed_dim=64, encoder_nb_heads=1,
                  encoder_nb_blocks=2, encoder_global_attn_indices=(0,), encoder_window_size=4, embed_dim=64),
}


def _build(overrides, precision="fp32", seed=7):
    import tfimm
    from oracle import params
    from oracle import sam as osam

    model = tfimm.create_model("sam_vit_b", precision=precision, device="cpu", **overrides)
    w = params.random_params(osam.param_shapes(model.cfg), seed=seed)
    model.load_weights_dict(w)
    return model, w


def test_import_of_tfimm_alone_registers_no_sam_model():
    code = ("import sys; sys.path[:0] = ['tensorflow-image-models_b200']; import tfimm; "
            "from tfimm.models import list_modules; assert 'sam' not in list_modules(); "
            "assert not tfimm.list_models('sam_*')")
    res = subprocess.run([sys.executable, "-c", code], cwd=str(ROOT), capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr[-2000:]


def test_registration(sam):
    from tfimm.models import list_models, model_config

    assert list_models(module="sam") == ["sam_vit_b", "sam_vit_h", "sam_vit_l"]
    assert list_models("sam_*", pretrained=True) == ["sam_vit_b", "sam_vit_h", "sam_vit_l"]
    cfg = model_config("sam_vit_h")
    assert (cfg.encoder_embed_dim, cfg.encoder_nb_blocks, cfg.encoder_nb_heads) == (1280, 32, 16)
    assert cfg.encoder_global_attn_indices == (7, 15, 23, 31)
    assert (cfg.input_size, cfg.encoder_window_size, cfg.embed_dim, cfg.fixed_input_size) == ((1024, 1024), 14, 256,
                                                                                              True)


@pytest.mark.parametrize("name,count", [("sam_vit_b", 93_735_472), ("sam_vit_l", 312_342_832),
                                        ("sam_vit_h", 641_090_608)])
def test_variable_table(sam, name, count):
    """Names and shapes equal the oracle's table; the parameter count is the published checkpoint's plus the prompt
    encoder's (2, 128) Gaussian matrix, which PyTorch keeps as a buffer."""
    import tfimm
    from oracle import sam as osam

    model = tfimm.create_model(name, device="meta")
    table = osam.param_shapes(model.cfg)
    assert {k: tuple(v.shape) for k, v in model.params.items()} == {k: tuple(v) for k, v in table.items()}
    assert model.count_params() == count + 256
    assert not model.param_specs()["prompt_encoder/pe_layer/positional_encoding_gaussian_matrix"].trainable
    assert len(model.image_encoder.params) == sum(k.startswith("image_encoder/") for k in table)


def test_model_surface(sam):
    import tfimm

    model = tfimm.create_model("sam_vit_b", device="meta")
    assert model.grid_size() == (64, 64) and model.grid_size((512, 768)) == (32, 48)
    assert model.mask_size() == (256, 256) and model.mask_threshold == 0.0
    assert set(model.dummy_inputs) == {"images", "points", "labels", "boxes", "masks"}
    assert tuple(model.dummy_inputs["masks"].shape) == (1, 1, 256, 256)
    with pytest.raises(NotImplementedError, match="image_encoder"):
        model(model.dummy_inputs)
    with pytest.raises(ValueError, match="tf32"):
        tfimm.create_model("sam_vit_b", precision="tf32", device="meta")


def test_image_encoder_has_the_model_attributes(sam):
    """ImageEncoder sets Model.__init__'s bookkeeping attributes itself (it must not create variables): every attribute
    a Model instance has, the encoder has too."""
    import tfimm

    model = tfimm.create_model("sam_vit_b", device="meta")
    missing = [k for k in vars(model) if k != "image_encoder" and not hasattr(model.image_encoder, k)]
    assert not missing, missing


def test_window_partition_round_trip():
    from oracle import sam as osam

    x = torch.randn(2, 10, 7, 3, dtype=torch.float64)
    win, pad_hw = osam.window_partition(x, 4)
    assert win.shape == (2 * 3 * 2, 4, 4, 3) and pad_hw == (12, 8)
    assert torch.equal(osam.window_unpartition(win, 4, pad_hw, (10, 7)), x)
    assert torch.equal(win[1, :, :3], x[0, :4, 4:7])           # window (0, 1) of image 0
    assert not win[1, :, 3].any() and not win[4, 2:].any()      # zero padding on the right / bottom


def test_rel_pos_terms_by_definition():
    """add_decomposed_rel_pos against rel_h[i, j] = q_i . R_h[qy - ky + S - 1] written out per element."""
    from oracle import sam as osam

    g = torch.Generator().manual_seed(0)
    S_h, S_w, c = 3, 4, 5
    q = torch.randn(1, S_h * S_w, c, generator=g, dtype=torch.float64)
    Rh = torch.randn(2 * S_h - 1, c, generator=g, dtype=torch.float64)
    Rw = torch.randn(2 * S_w - 1, c, generator=g, dtype=torch.float64)
    out = osam.add_decomposed_rel_pos(torch.zeros(1, S_h * S_w, S_h * S_w, dtype=torch.float64), q, Rh, Rw,
                                      (S_h, S_w), (S_h, S_w), False)
    for i in range(S_h * S_w):
        for j in range(S_h * S_w):
            (qy, qx), (ky, kx) = divmod(i, S_w), divmod(j, S_w)
            want = q[0, i] @ Rh[qy - ky + S_h - 1] + q[0, i] @ Rw[qx - kx + S_w - 1]
            assert abs(out[0, i, j] - want) < 1e-12


def test_bilinear_resize_matches_the_oracle():
    from oracle import sam as osam
    from tfimm.layers.resize import tf_bilinear_resize

    x = torch.randn(1, 7, 5, 3, dtype=torch.float64)
    for size in ((13, 9), (3, 4), (7, 5)):
        assert torch.allclose(tf_bilinear_resize(x, size), osam.resize_bilinear(x, size), atol=1e-12)
    assert torch.equal(osam.resize_bilinear(x, (7, 5)), x)


@pytest.mark.parametrize("case", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(sam, cpu_engine, case):
    from oracle import params
    from oracle import sam as osam
    from sam_oracle import emulated_sam_ops

    model, w = _build(SMALL[case])
    sizes = [model.cfg.input_size] + ([(32, 48)] if not model.cfg.fixed_input_size else [])
    for size in sizes:
        x = params.test_images(2, *size)
        with emulated_sam_ops():
            y, feats = model.image_encoder(x, return_features=True)
        ref, rfeats = osam.image_encoder(model.cfg, {k: v.double() for k, v in w.items()}, x.double(), True)
        assert y.shape == ref.shape == (2, size[0] // 4, size[1] // 4, 64)
        assert list(feats) == list(rfeats)
        assert _nerr(y, ref) < 1e-5, case
        for k in feats:
            assert _nerr(feats[k], rfeats[k]) < 1e-5, (case, k)


@pytest.mark.parametrize("case", ["pad", "dh80"])
def test_bf16_orchestration_stays_inside_the_bf16_budget(sam, cpu_engine, case):
    from oracle import params
    from oracle import sam as osam
    from sam_oracle import emulated_sam_ops

    model, w = _build(SMALL[case], precision="bf16")
    x = params.test_images(2, *model.cfg.input_size)
    with emulated_sam_ops():
        y = model.image_encoder(x)
    ref = osam.image_encoder(model.cfg, {k: v.double() for k, v in w.items()}, x.double())
    assert _nerr(y, ref) < 2e-2


def test_uint8_pixels_equal_preprocessed_floats(sam, cpu_engine):
    import tfimm
    from sam_oracle import emulated_sam_ops

    model, _ = _build(SMALL["nopad"])
    px = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (1, 32, 32, 3), dtype=np.uint8))
    pre = tfimm.create_preprocessing("sam_vit_b")
    with emulated_sam_ops():
        a = model.image_encoder(px)
        b = model.image_encoder(pre(px))
    assert _nerr(a, b) < 1e-6


def _register_small(sam):
    """A registration with the "pad" geometry, as the reference's tests register sam_vit_test_model: create_model
    loads a checkpoint into the REGISTERED configuration first."""
    from tfimm.models import register_model

    def sam_small_pad():
        return sam.SegmentAnythingModel, sam.SegmentAnythingModelConfig(name="sam_small_pad", **SMALL["pad"])

    register_model(sam_small_pad)


def test_weights_save_load_and_sharing(sam, tmp_path):
    import tfimm
    from tfimm.models import save_weights

    _register_small(sam)
    model, w = _build(SMALL["pad"])
    enc = model.image_encoder
    assert enc.params["pos_embed"] is model.params["image_encoder/pos_embed"]
    path = str(tmp_path / "sam.npz")
    save_weights(model, path)
    loaded = tfimm.create_model("sam_small_pad", model_path=path, device="cpu")
    for k, v in w.items():
        assert torch.equal(loaded.params[k].cpu(), v), k
    # a load through the encoder writes the parent's tensors (one copy) and invalidates the plans
    new = torch.full_like(w["image_encoder/neck/1/gamma"], 2.0)
    enc.load_weights_dict({"neck/1/gamma": new}, strict=False)
    assert torch.equal(model.params["image_encoder/neck/1/gamma"], new)
    with pytest.raises(AttributeError):
        loaded.load_weights_dict({k: v for k, v in w.items() if not k.startswith("mask_decoder/")}, strict=True)


def test_transform_weights_resizes_like_the_reference(sam, cpu_engine, tmp_path):
    """create_model(..., input_size=) resizes pos_embed and the global blocks' tables bilinearly (reference
    sam.py:158-203), and then the resized model computes what the original computes at that size
    (the reference's test_transfer_weights)."""
    import tfimm
    from oracle import params
    from oracle import sam as osam
    from sam_oracle import emulated_sam_ops
    from tfimm.models import save_weights

    _register_small(sam)
    model, w = _build(SMALL["pad"])
    path = str(tmp_path / "sam.npz")
    save_weights(model, path)
    big = tfimm.create_model("sam_small_pad", model_path=path, device="cpu", precision="fp32", input_size=(48, 48))
    pos = osam.resize_bilinear(w["image_encoder/pos_embed"].double(), (12, 12))
    assert torch.allclose(big.params["image_encoder/pos_embed"].double(), pos, atol=1e-6)
    rh = osam.resize_bilinear(w["image_encoder/blocks/1/attn/rel_pos_h"].double()[None, None], (1, 23))[0, 0]
    assert torch.allclose(big.params["image_encoder/blocks/1/attn/rel_pos_h"].double(), rh, atol=1e-6)
    assert torch.equal(big.params["image_encoder/blocks/0/attn/rel_pos_h"], w["image_encoder/blocks/0/attn/rel_pos_h"])
    x = params.test_images(1, 48, 48)
    with emulated_sam_ops():
        a = model.image_encoder(x)
        b = big.image_encoder(x)
    assert _nerr(a, b) < 1e-5
