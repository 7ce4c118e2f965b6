"""Model-level parity on the GPU: engine logits vs the CPU oracle on identical seeded inputs.

Error metric is the reference's own (tests/test_timm.py:71): max|a-b| / (max|b| + 1e-6); plain
max|a-b| is printed next to it.  Tolerances:
  * precision="fp32": 1e-5, north_star's own bound (measured: 0.3-2e-6)
  * precision="bf16": north_star asks 1e-3, which no implementation that STORES activations in bf16 can meet (the
    ideal one -- exact arithmetic, same storage points -- is 3-7e-3 from the fp32 reference, see
    tests/test_parity_budget_gpu.py).  Asserted here: ~1.3x the measured value for each family, so that a
    regression shows: ViT / Swin 1e-2 (measured 5-7e-3), ConvNeXt 7e-3 (4.5e-3), BN families 8e-3 (3-4e-3).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-5
BF16_TOL = 1e-2     # ViT / Swin
BF16_TOL_CONVNEXT = 7e-3
BF16_TOL_BN = 8e-3  # EfficientNet / ResNet families (bf16 activation stream, BatchNorm folded)


def _nerr(out, ref):
    out, ref = out.float().cpu(), ref.float().cpu()
    d = (out - ref).abs().max().item()
    return d / (ref.abs().max().item() + 1e-6), d


def _run(name, family, precision, batch, overrides=None, seed=3):
    import importlib

    import tfimm
    from oracle import params

    omod = importlib.import_module(f"oracle.{family}")
    model = tfimm.create_model(name, precision=precision, device="cuda", **(overrides or {}))
    w = params.random_params(omod.param_shapes(model.cfg), seed=seed)
    model.load_weights_dict(w)
    h, wd = model.cfg.input_size
    x = params.test_images(batch, h, wd, model.cfg.in_channels)
    out = model(x.cuda())
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = omod.forward(model.cfg, w, x)
    return model, w, x, out, ref


@pytest.mark.parametrize("name", ["vit_tiny_patch16_224", "deit_tiny_distilled_patch16_224", "vit_small_patch32_224"])
def test_vit_fp32_parity(name):
    _, _, _, out, ref = _run(name, "vit", "fp32", 2)
    rel, ab = _nerr(out, ref)
    print(f"{name} fp32: normalised {rel:.3e} abs {ab:.3e}")
    assert out.shape == ref.shape
    assert rel < FP32_TOL


@pytest.mark.parametrize("name,batch", [("vit_tiny_patch16_224", 3), ("deit_tiny_distilled_patch16_224", 2),
                                        ("vit_base_patch16_224", 2), ("vit_base_patch32_224_in21k", 2)])
def test_vit_bf16_parity(name, batch):
    _, _, _, out, ref = _run(name, "vit", "bf16", batch)
    rel, ab = _nerr(out, ref)
    print(f"{name} bf16: normalised {rel:.3e} abs {ab:.3e}")
    assert out.shape == ref.shape
    assert rel < BF16_TOL


def test_vit_return_features_matches_plain_call():
    """reference tests/models/test_factory.py:205-222: same logits, exactly `feature_names` keys."""
    import tfimm
    from oracle import params
    from oracle import vit as ovit

    model = tfimm.create_model("vit_tiny_patch16_224", precision="fp32", device="cuda")
    w = params.random_params(ovit.param_shapes(model.cfg), seed=5)
    model.load_weights_dict(w)
    x = params.test_images(2, 224, 224)
    y = model(x.cuda())
    y2, feats = model(x.cuda(), return_features=True)
    assert (y - y2).abs().max().item() < 1e-5
    assert list(feats.keys()) == model.feature_names
    _, ofeats = ovit.forward(model.cfg, w, x, return_features=True)
    assert list(feats.keys()) == list(ofeats.keys())
    for k in ("patch_embedding", "block_5/attn", "block_11", "features_all", "features", "logits"):
        rel, _ = _nerr(feats[k], ofeats[k])
        assert rel < 5e-5, (k, rel)


def test_vit_nb_classes_zero_and_other_sizes():
    import tfimm
    from oracle import params
    from oracle import vit as ovit

    model = tfimm.create_model("vit_tiny_patch16_224", precision="fp32", device="cuda", nb_classes=0,
                               input_size=(96, 64))
    w = params.random_params(ovit.param_shapes(model.cfg), seed=6)
    model.load_weights_dict(w)
    x = params.test_images(2, 96, 64)
    out = model(x.cuda())
    ref = ovit.forward(model.cfg, w, x)
    assert out.shape == (2, 192)
    assert _nerr(out, ref)[0] < FP32_TOL


def test_vit_interpolate_input():
    """interpolate_input=True: pos_embed is resampled (TF bicubic) to the grid of the actual input
    (tfimm/architectures/vit.py:434-443; reference tests/models/test_factory.py:156-179)."""
    import tfimm
    from oracle import params
    from oracle import vit as ovit

    model = tfimm.create_model("vit_tiny_patch16_224", precision="fp32", device="cuda", interpolate_input=True,
                               input_size=(64, 64))
    w = params.random_params(ovit.param_shapes(model.cfg), seed=8)
    model.load_weights_dict(w)
    x = params.test_images(1, 96, 128)
    out = model(x.cuda())
    ref = ovit.forward(model.cfg, w, x)
    assert _nerr(out, ref)[0] < FP32_TOL
    # native size stays a no-op
    x = params.test_images(1, 64, 64)
    assert _nerr(model(x.cuda()), ovit.forward(model.cfg, w, x))[0] < FP32_TOL


@pytest.mark.parametrize("name,overrides", [("convnext_tiny", {}), ("convnext_tiny", {"input_size": (96, 160)}),
                                            ("convnext_tiny_in22k", {"conv_mlp_block": True})])
def test_convnext_fp32_parity(name, overrides):
    _, _, _, out, ref = _run(name, "convnext", "fp32", 2, overrides)
    rel, ab = _nerr(out, ref)
    print(f"{name} fp32: normalised {rel:.3e} abs {ab:.3e}")
    assert out.shape == ref.shape
    assert rel < FP32_TOL


@pytest.mark.parametrize("name", ["convnext_tiny", "convnext_base"])
def test_convnext_bf16_parity(name):
    _, _, _, out, ref = _run(name, "convnext", "bf16", 2)
    rel, ab = _nerr(out, ref)
    print(f"{name} bf16: normalised {rel:.3e} abs {ab:.3e}")
    assert rel < BF16_TOL_CONVNEXT


def test_convnext_return_features():
    import tfimm
    from oracle import convnext as oc
    from oracle import params

    model = tfimm.create_model("convnext_tiny", precision="fp32", device="cuda", input_size=(64, 64))
    w = params.random_params(oc.param_shapes(model.cfg), seed=5)
    model.load_weights_dict(w)
    x = params.test_images(2, 64, 64)
    y = model(x.cuda())
    y2, feats = model(x.cuda(), return_features=True)
    assert (y - y2).abs().max().item() < 1e-5
    _, ofeats = oc.forward(model.cfg, w, x, return_features=True)
    assert list(feats.keys()) == list(ofeats.keys()) == model.feature_names
    for k in ("stem", "stage_1/downsample", "stage_2/block_3", "conv_features", "features", "logits"):
        assert _nerr(feats[k], ofeats[k])[0] < 5e-5, k


@pytest.mark.parametrize("name,overrides", [("swin_tiny_patch4_window7_224", {}),
                                            ("swin_tiny_patch4_window7_224", {"input_size": (112, 112), "window_size": 7,
                                                                              "nb_blocks": (2, 2), "nb_heads": (3, 6)})])
def test_swin_fp32_parity(name, overrides):
    _, _, _, out, ref = _run(name, "swin", "fp32", 2, overrides)
    rel, ab = _nerr(out, ref)
    print(f"{name} fp32: normalised {rel:.3e} abs {ab:.3e}")
    assert out.shape == ref.shape
    assert rel < FP32_TOL


@pytest.mark.parametrize("name", ["swin_tiny_patch4_window7_224", "swin_base_patch4_window7_224"])
def test_swin_bf16_parity(name):
    _, _, _, out, ref = _run(name, "swin", "bf16", 2)
    rel, ab = _nerr(out, ref)
    print(f"{name} bf16: normalised {rel:.3e} abs {ab:.3e}")
    assert rel < BF16_TOL


def test_swin_window12_bf16_runs_on_the_tensor_core_window_kernel():
    """*_window12_384 registrations (144 tokens per window): the bf16 mma.sync window kernel, not the fp32 fallback."""
    import tfimm
    from tfimm.backend import ops

    name = "swin_base_patch4_window12_384"
    overrides = {"nb_blocks": (2, 2, 2, 2)}
    _, _, _, out, ref = _run(name, "swin", "bf16", 1, overrides)
    rel, ab = _nerr(out, ref)
    print(f"{name} (2 blocks per stage) bf16: normalised {rel:.3e} abs {ab:.3e}")
    assert rel < BF16_TOL
    model = tfimm.create_model(name, precision="bf16", device="cuda", **overrides)
    ops.trace = []
    model(torch.zeros(1, 384, 384, 3, device="cuda"))
    torch.cuda.synchronize()
    fams = {t[0] for t in ops.trace}
    ops.trace = None
    assert "window_attention_bf16" in fams and "attention_f32" not in fams, fams


def test_swin_return_features():
    import tfimm
    from oracle import params
    from oracle import swin as osw

    model = tfimm.create_model("swin_tiny_patch4_window7_224", precision="fp32", device="cuda")
    w = params.random_params(osw.param_shapes(model.cfg), seed=5)
    model.load_weights_dict(w)
    x = params.test_images(1, 224, 224)
    y = model(x.cuda())
    y2, feats = model(x.cuda(), return_features=True)
    assert (y - y2).abs().max().item() < 1e-5
    _, ofeats = osw.forward(model.cfg, w, x, return_features=True)
    assert list(feats.keys()) == list(ofeats.keys()) == model.feature_names
    for k in ("patch_embedding", "block_1", "stage_0", "block_7", "features_all", "features", "logits"):
        assert _nerr(feats[k], ofeats[k])[0] < 5e-5, k


@pytest.mark.parametrize("name,overrides", [
    ("efficientnet_b0", {}),                                   # TF "same" padding, BN eps 1e-3, SE, swish
    ("pt_efficientnet_b0", {"input_size": (192, 160)}),        # symmetric padding
    ("mobilenet_v2_100", {}),                                  # relu6, no SE
    ("efficientnet_es", {}),                                   # EdgeResidual blocks
    ("efficientnet_lite0", {}),
    ("efficientnet_v2_b0", {"input_size": (128, 128)}),        # cn + er + ir mix
])
def test_efficientnet_fp32_parity(name, overrides):
    _, _, _, out, ref = _run(name, "efficientnet", "fp32", 2, overrides)
    rel, ab = _nerr(out, ref)
    print(f"{name} fp32: normalised {rel:.3e} abs {ab:.3e}")
    assert out.shape == ref.shape
    assert rel < FP32_TOL


@pytest.mark.parametrize("name,size", [("efficientnet_b0", 224), ("efficientnet_b4", 380)])
def test_efficientnet_bf16_parity(name, size):
    _, _, _, out, ref = _run(name, "efficientnet", "bf16", 2, {"input_size": (size, size)})
    rel, ab = _nerr(out, ref)
    print(f"{name} bf16: normalised {rel:.3e} abs {ab:.3e}")
    assert rel < BF16_TOL_BN


@pytest.mark.parametrize("name", ["resnet18", "resnet50", "resnet50d", "resnext50_32x4d", "seresnet50", "ecaresnet26t",
                                  "resnetrs50"])
def test_resnet_fp32_parity(name):
    _, _, _, out, ref = _run(name, "resnet", "fp32", 2, {"input_size": (128, 128)})
    rel, ab = _nerr(out, ref)
    print(f"{name} fp32: normalised {rel:.3e} abs {ab:.3e}")
    assert out.shape == ref.shape
    assert rel < FP32_TOL


@pytest.mark.parametrize("name,overrides", [
    ("resnet50_gn", {}),                                       # GroupNormalization instead of every BatchNorm
    ("resnetblur50", {}),                                      # BlurPool2D anti-aliasing (stem pool + strided blocks)
    ("resnext101_32x8d", {"nb_blocks": (1, 1, 1, 1)}),         # 64 channels per group in the last stage
    ("ig_resnext101_32x48d", {"nb_blocks": (1, 1, 1, 1), "input_size": (64, 64)}),  # 48..384 channels per group
])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_resnet_norm_blur_and_wide_group_variants(name, overrides, precision):
    _, _, _, out, ref = _run(name, "resnet", precision, 2, overrides)
    rel, ab = _nerr(out, ref)
    print(f"{name} {precision}: normalised {rel:.3e} abs {ab:.3e}")
    # GroupNorm (resnet50_gn) re-normalises every activation from batch-free statistics: measured ~1e-2 in bf16
    assert rel < (FP32_TOL if precision == "fp32" else (1.5e-2 if name == "resnet50_gn" else BF16_TOL_BN))


@pytest.mark.parametrize("name", ["resnet50", "resnext50_32x4d"])
def test_resnet_bf16_parity(name):
    _, _, _, out, ref = _run(name, "resnet", "bf16", 2)
    rel, ab = _nerr(out, ref)
    print(f"{name} bf16: normalised {rel:.3e} abs {ab:.3e}")
    assert rel < BF16_TOL_BN


def _golden_cases():
    from pathlib import Path

    return sorted(p.name for p in (Path(__file__).resolve().parent / "golden").glob("*.npz"))


@pytest.mark.parametrize("fixture", _golden_cases())
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_engine_matches_committed_golden_logits(fixture, precision):
    """Engine vs the stored oracle logits (tests/golden, tools/make_golden.py): nothing here reads the
    oracle's code path, only the committed numbers."""
    import importlib
    from pathlib import Path

    import numpy as np

    import tfimm
    from oracle import params

    data = np.load(Path(__file__).resolve().parent / "golden" / fixture, allow_pickle=True)
    meta = data["meta"].item()
    mod = importlib.import_module(f"oracle.{meta['family']}")
    model = tfimm.create_model(meta["model"], precision=precision, device="cuda", **meta["overrides"])
    model.load_weights_dict(params.random_params(mod.param_shapes(model.cfg), seed=meta["seed"]))
    if "images" in data.files:
        images = torch.from_numpy(data["images"])
    else:  # full-size BASELINE configs store logits only; images are regenerated from their seed
        images = params.test_images(meta["batch"], *model.cfg.input_size, model.cfg.in_channels,
                                    seed=meta.get("images_seed", 2021))
    out = model(images.cuda())
    rel, ab = _nerr(out, torch.from_numpy(data["logits"]))
    print(f"{fixture} {precision}: normalised {rel:.3e} abs {ab:.3e}")
    assert rel < (FP32_TOL if precision == "fp32" else BF16_TOL)


def test_cuda_graph_replay_matches_eager():
    import tfimm
    from oracle import params
    from oracle import vit as ovit

    model = tfimm.create_model("vit_tiny_patch16_224", precision="bf16", device="cuda", nb_blocks=3)
    model.load_weights_dict(params.random_params(ovit.param_shapes(model.cfg), seed=9))
    fwd = model.cuda_graph(4)
    for seed in (1, 2):
        x = params.test_images(4, 224, 224, seed=seed).cuda()
        eager = model(x).clone()
        replay = fwd(x).clone()
        assert torch.equal(eager, replay)
    assert fwd.launches > 0


@pytest.mark.parametrize("name,family", [("vit_tiny_patch16_224", "vit"), ("convnext_tiny", "convnext"),
                                         ("swin_tiny_patch4_window7_224", "swin"), ("efficientnet_b0", "efficientnet"),
                                         ("resnet18", "resnet"), ("resnet26d", "resnet")])
def test_fused_uint8_preprocessing_equals_create_preprocessing(name, family):
    """model(uint8 pixels) == model(create_preprocessing(name)(pixels))  (reference factory.py:153-169)."""
    import importlib

    import numpy as np

    import tfimm
    from oracle import params

    omod = importlib.import_module(f"oracle.{family}")
    model = tfimm.create_model(name, precision="fp32", device="cuda")
    model.load_weights_dict(params.random_params(omod.param_shapes(model.cfg), seed=21))
    raw = np.random.default_rng(5).integers(0, 256, (2, 224, 224, 3), dtype=np.uint8)
    pre = tfimm.create_preprocessing(name)
    a = model(torch.from_numpy(raw).cuda())
    b = model(torch.from_numpy(pre(raw)).cuda())
    assert _nerr(a, b)[0] < 1e-5
    # bf16 engine: the stem sees bf16((x / 255 - mean) / std) either way
    m16 = tfimm.create_model(name, precision="bf16", device="cuda")
    m16.load_weights_dict(params.random_params(omod.param_shapes(m16.cfg), seed=21))
    a16 = m16(torch.from_numpy(raw).cuda())
    b16 = m16(torch.from_numpy(pre(raw)).cuda())
    assert _nerr(a16, b16)[0] < 2e-3


def test_inference_pipeline_matches_direct_calls():
    import tfimm
    from oracle import params
    from oracle import vit as ovit
    from tfimm.serving import InferencePipeline

    model = tfimm.create_model("vit_tiny_patch16_224", precision="bf16", device="cuda", nb_blocks=2)
    model.load_weights_dict(params.random_params(ovit.param_shapes(model.cfg), seed=22))
    pipe = InferencePipeline(model, 4, depth=2)
    batches = [params.test_images(4, 224, 224, seed=s).pin_memory() for s in (1, 2, 3, 4, 5)]
    outs = []
    for xb in batches:
        o = pipe.submit(xb)
        pipe.synchronize()
        outs.append(o.clone())
    for xb, o in zip(batches, outs):
        assert torch.equal(model(xb.cuda()).cpu(), o)


@pytest.mark.parametrize("name,overrides", [
    ("vit_huge_patch14_224_in21k", {"nb_blocks": 2}),          # head_dim 80: no bf16 tensor-core attention kernel
    ("vit_base_patch8_224", {"nb_blocks": 2}),                 # 785 tokens: resident-K/V kernel with 128-row tiles
    ("vit_base_patch16_384", {"nb_blocks": 2}),                # 577 tokens
    ("vit_base_patch8_224", {"nb_blocks": 1, "input_size": (256, 256)}),   # 1025 tokens: fp32 attention fallback
])
def test_vit_shapes_outside_the_tcgen05_attention_kernel_run_in_bf16(name, overrides):
    """Every registered ViT shape must run at the default precision (ADVICE r01): shapes the bf16 attention kernels
    do not take fall back to the fp32 SIMT attention on the same bf16 qkv values."""
    _, _, _, out, ref = _run(name, "vit", "bf16", 1, overrides)
    rel, ab = _nerr(out, ref)
    print(f"{name} {overrides} bf16: normalised {rel:.3e}")
    assert rel < BF16_TOL


def test_cuda_graph_rejects_wrong_dtype_and_stale_weights():
    import tfimm
    from oracle import params
    from oracle import vit as ovit

    model = tfimm.create_model("vit_tiny_patch16_224", precision="bf16", device="cuda", nb_blocks=1)
    w = params.random_params(ovit.param_shapes(model.cfg), seed=9)
    model.load_weights_dict(w)
    fwd = model.cuda_graph(2)
    x = params.test_images(2, 224, 224).cuda()
    fwd(x)
    with pytest.raises(TypeError):
        fwd((x * 255).to(torch.uint8))          # a float capture must not silently cast raw pixels
    with pytest.raises(TypeError):
        fwd(x[:1])
    fwd8 = model.cuda_graph(2, dtype=torch.uint8)   # raw pixels: capture with the fused preprocessing
    raw = (x * 255).to(torch.uint8)
    assert torch.equal(fwd8(raw), model(raw))
    model.load_weights_dict(w)
    with pytest.raises(RuntimeError):
        fwd(x)                                   # weights changed after capture


def test_model_on_second_device_if_present():
    """Launches follow the tensors' device, not torch's current device (ADVICE r01)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import tfimm
    from oracle import params
    from oracle import vit as ovit

    m0 = tfimm.create_model("vit_tiny_patch16_224", precision="bf16", device="cuda:0", nb_blocks=2)
    m1 = tfimm.create_model("vit_tiny_patch16_224", precision="bf16", device="cuda:1", nb_blocks=2)
    w = params.random_params(ovit.param_shapes(m0.cfg), seed=9)
    m0.load_weights_dict(w)
    m1.load_weights_dict(w)
    x = params.test_images(2, 224, 224)
    a = m0(x.to("cuda:0")).cpu()
    b = m1(x.to("cuda:1")).cpu()          # current device is still cuda:0
    assert torch.equal(a, b)
