"""Pins the oracle (and the engine's host-side API) to the REFERENCE ITSELF.

TensorFlow cannot be installed here, so ``oracle/ref_runner.py`` executes the unmodified reference sources
(``tfimm/architectures/{vit,swin,convnext,efficientnet,resnet}.py`` + ``tfimm/layers`` +
``tfimm/models/{factory,registry}.py`` + ``tfimm/utils/timm.py``) on a torch-CPU restatement of the TF/Keras calls
they make (``oracle/tf_shim``).  ``tools/make_reference_pins.py`` ran the cases below through that reference code and
recorded what it computed (its own variable names, on identical seeded inputs, tests/test_timm.py:56-71 of the
reference) in ``tests/golden/reference/pins.npz``; everything below compares against that recording.
"""
import hashlib
import importlib
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tensorflow-image-models_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import params  # noqa: E402

PINS = ROOT / "tests" / "golden" / "reference" / "pins.npz"
# elements recorded per array: logits, intermediate features, variables written by transfer_weights
LOGIT_SAMPLE, FEATURE_SAMPLE, TRANSFER_SAMPLE = 8, 4, 4


def sample_index(n, k, seed=0):
    """The fixed element sample recorded for a flattened array of n elements (all of them when n <= k)."""
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.default_rng(seed + n).choice(n, k, replace=False))


def table_digest(table, ordered=False):
    """Digest of a {name: shape} table, sorted by name unless the order itself is pinned."""
    items = [(k, list(v)) for k, v in table.items()]
    return hashlib.sha256(json.dumps(items if ordered else sorted(items)).encode()).hexdigest()[:16]


def params_digest(weights):
    """Digest of a {name: array} parameter set: names and exact float32 values."""
    h = hashlib.sha256()
    for k in sorted(weights):
        h.update(k.encode())
        h.update(np.ascontiguousarray(np.asarray(weights[k], dtype=np.float32)).tobytes())
    return h.hexdigest()[:16]


@pytest.fixture(scope="module")
def pins():
    with np.load(PINS) as z:
        arrays = {k: z[k] for k in z.files}
    return arrays, json.loads(arrays.pop("meta").tobytes())


IGNORE = ("attn_mask", "relative_position_index", "blur_kernel")

# (family, registered name, create_model overrides) -- the small configurations of the reference's own test-suite
# (tests/models/architectures.py: *_test_model) expressed as overrides of registered models, plus real registrations.
CASES = [
    ("vit", "vit_tiny_patch16_224", {"input_size": (32, 32), "patch_size": 8, "embed_dim": 4, "nb_blocks": 2, "nb_heads": 2, "nb_classes": 12}),
    ("vit", "deit_tiny_distilled_patch16_224", {"input_size": (32, 32), "patch_size": 8, "embed_dim": 4, "nb_blocks": 2, "nb_heads": 2, "nb_classes": 12}),
    ("vit", "vit_base_patch32_224_in21k", {"input_size": (64, 64), "embed_dim": 24, "nb_blocks": 2, "nb_heads": 3, "representation_size": 16, "nb_classes": 7}),
    ("vit", "vit_tiny_patch16_224", {"input_size": (96, 64), "nb_blocks": 3}),
    ("swin", "swin_tiny_patch4_window7_224", {"input_size": (32, 32), "patch_size": 2, "embed_dim": 4, "nb_blocks": (2, 2), "nb_heads": (1, 2), "window_size": 4, "nb_classes": 12}),
    ("swin", "swin_tiny_patch4_window7_224", {"input_size": (112, 112), "nb_blocks": (2, 2, 2), "nb_heads": (3, 6, 12)}),
    ("convnext", "convnext_tiny", {"input_size": (32, 32), "embed_dim": (3, 4, 5, 6), "nb_blocks": (1, 1, 1, 1), "nb_classes": 12}),
    ("convnext", "convnext_tiny", {"input_size": (64, 96), "nb_blocks": (1, 1, 2, 1)}),
    ("convnext", "convnext_tiny_in22k", {"input_size": (64, 64), "nb_blocks": (1, 1, 1, 1), "conv_mlp_block": True}),
    ("efficientnet", "efficientnet_b0", {"input_size": (64, 64)}),
    ("efficientnet", "efficientnet_b4", {"input_size": (76, 76)}),
    ("efficientnet", "pt_efficientnet_b0", {"input_size": (64, 80)}),
    ("efficientnet", "mobilenet_v2_100", {"input_size": (64, 64)}),
    ("efficientnet", "efficientnet_es", {"input_size": (64, 64)}),
    ("efficientnet", "efficientnet_lite0", {"input_size": (64, 64)}),
    ("efficientnet", "efficientnet_v2_b0", {"input_size": (64, 64)}),
    ("resnet", "resnet18", {"input_size": (64, 64)}),
    ("resnet", "resnet50", {"input_size": (64, 64)}),
    ("resnet", "resnet50d", {"input_size": (64, 64)}),
    ("resnet", "resnext50_32x4d", {"input_size": (64, 64)}),
    ("resnet", "seresnext26d_32x4d", {"input_size": (64, 64)}),
    ("resnet", "ecaresnet26t", {"input_size": (64, 64)}),
    ("resnet", "resnetblur50", {"input_size": (64, 64)}),
    ("resnet", "resnet50_gn", {"input_size": (64, 64)}),
    ("resnet", "resnetrs50", {"input_size": (64, 64)}),
]


def _nerr(a, b):
    a, b = a.double(), b.double()
    return (a - b).abs().max().item() / (b.abs().max().item() + 1e-6)


def _engine_cfg(name, overrides):
    import tfimm

    base = tfimm.models.model_config(name)
    return type(base)(**{**base.__dict__, **overrides})


@pytest.mark.parametrize("case", range(len(CASES)), ids=[f"{c[1]}-{i}" for i, c in enumerate(CASES)])
def test_oracle_equals_reference_code_run_on_the_shim(case, pins):
    """Same variables (names + shapes) and, in float64, the same logits to 1e-12: the oracle restates the
    reference's graph exactly.  (float32 run of the same comparison: ~3e-7, see tools/make_golden.py.)"""
    arrays, meta = pins
    family, name, overrides = CASES[case]
    rec = meta["shim"][case]
    omod = importlib.import_module(f"oracle.{family}")
    cfg = _engine_cfg(name, overrides)
    shapes = omod.param_shapes(cfg)
    assert table_digest(shapes) == rec["weights"]   # the reference's loadable variables: same names and shapes
    w = params.random_params(shapes, seed=31, dtype=torch.float64)
    x = params.test_images(2, *cfg.input_size, cfg.in_channels).double()
    with torch.no_grad():
        y_or, f_or = omod.forward(cfg, w, x, return_features=True)
    # arrays are recorded as a fixed element sample plus the max-abs value of the whole array
    assert arrays["shim_logits"].dtype == np.float64 and list(y_or.shape) == rec["logits_shape"]
    idx = sample_index(y_or.numel(), LOGIT_SAMPLE)
    want = arrays["shim_logits"][rec["logits_offset"]:rec["logits_offset"] + len(idx)]
    got = y_or.reshape(-1)[torch.from_numpy(idx)].double()
    assert (got - torch.from_numpy(want)).abs().max().item() / (rec["logits_absmax"] + 1e-6) < 1e-12
    # intermediate features: same keys in the same order with the same shapes, same values
    # (tests/models/test_factory.py:205-222)
    assert table_digest({k: v.shape for k, v in f_or.items()}, ordered=True) == rec["features"]
    off = rec["feature_offset"]
    for i, (k, v) in enumerate(f_or.items()):
        idx = sample_index(v.numel(), FEATURE_SAMPLE)
        got = v.reshape(-1)[torch.from_numpy(idx)].double()
        want = torch.from_numpy(arrays["shim_features"][off:off + len(idx)])
        off += len(idx)
        absmax = arrays["shim_feature_absmax"][rec["feature_index"] + i]
        assert (got - want).abs().max().item() / (absmax + 1e-6) < 1e-11, k


def test_oracle_equals_reference_in_float32_at_full_size(pins):
    """The reference's default dtype and a real registration at its native 224 px."""
    from oracle import vit as ovit

    cfg = _engine_cfg("vit_tiny_patch16_224", {})
    w = params.random_params(ovit.param_shapes(cfg), seed=3)
    x = params.test_images(1, 224, 224)
    assert _nerr(ovit.forward(cfg, w, x), torch.from_numpy(pins[0]["full_size_logits"])) < 2e-6


def test_vit_interpolate_input_equals_reference(pins):
    """interpolate_input=True resamples pos_embed with tf.image.resize(bicubic) (layers/transformers.py:13-47)."""
    from oracle import vit as ovit

    ov = {"input_size": (64, 64), "nb_blocks": 1, "interpolate_input": True}
    cfg = _engine_cfg("vit_tiny_patch16_224", ov)
    w = params.random_params(ovit.param_shapes(cfg), seed=4, dtype=torch.float64)
    x = params.test_images(1, 96, 128).double()
    # tf.image.resize returns float32, so agreement is at float32 rounding of the position table
    assert _nerr(ovit.forward(cfg, w, x), torch.from_numpy(pins[0]["interpolate_logits"])) < 1e-6


INITIAL_VALUE_CASES = (("convnext_tiny", {"input_size": (32, 32), "nb_blocks": (1, 1, 1, 1)}),
                       ("vit_tiny_patch16_224", {"input_size": (32, 32), "nb_blocks": 1}),
                       ("resnet18", {"input_size": (32, 32)}), ("resnet50_gn", {"input_size": (32, 32)}))


def test_reference_initial_values_match_engine_initialisers(pins):
    """Variables created by build(): the engine's ParamSpec initialisers name the same constants
    (zeros cls/pos tokens vit.py:378-400, ConvNeXt layer scale 1e-6 convnext.py:211-217, zero-init last BN gamma
    with moving_variance = zeros only where the reference passes it, resnet.py:147-155)."""
    import tfimm

    for name, ov in INITIAL_VALUE_CASES:
        ref = pins[1]["initial_values"][name]   # reference variable -> its initial value, where that is one constant
        eng = tfimm.create_model(name, device="cpu", **ov)
        for key, spec in eng.param_specs().items():
            kind, _, arg = spec.init.partition(":")
            if kind in ("zeros", "ones", "const"):
                want = {"zeros": 0.0, "ones": 1.0}.get(kind, float(arg) if arg else 0.0)
                assert key in ref and np.isclose(ref[key], want), (name, key, spec.init, ref.get(key))


REGISTRY_CONFIGS = ("vit_base_patch16_224", "swin_base_patch4_window7_224", "convnext_base", "efficientnet_b4",
                    "resnet50")


def test_list_models_and_configs_equal_the_reference_registry(pins):
    import dataclasses

    import tfimm

    meta = pins[1]
    for fam, ref_names in meta["registry"].items():
        assert tfimm.list_models(module=fam) == ref_names
    assert set(meta["configs"]) == set(REGISTRY_CONFIGS)
    for n, rc in meta["configs"].items():
        ec = json.loads(json.dumps(dataclasses.asdict(tfimm.models.model_config(n))))   # tuples -> lists, as stored
        for k, v in rc.items():
            assert ec[k] == v or list(ec[k]) == list(v), (n, k, ec[k], v)


PREPROCESSING_MODELS = ["vit_base_patch16_224", "convnext_base", "efficientnet_b4", "resnet50"]


def preprocessing_image():
    return np.random.default_rng(0).integers(0, 256, (2, 16, 16, 3)).astype(np.uint8)


@pytest.mark.parametrize("name", PREPROCESSING_MODELS)
def test_create_preprocessing_equals_reference(name, pins):
    import tfimm

    a = pins[0]["preprocessing"][PREPROCESSING_MODELS.index(name)]
    b = np.asarray(tfimm.create_preprocessing(name, dtype="float32")(preprocessing_image()))
    assert np.abs(a - b).max() < 1e-6
    with pytest.raises(ValueError):
        tfimm.create_preprocessing("not_a_model")


TRANSFER_MODELS = [("resnet18", {"input_size": (32, 32)}),
                   ("vit_tiny_patch16_224", {"input_size": (32, 32), "nb_blocks": 1}),
                   ("convnext_tiny", {"input_size": (32, 32), "nb_blocks": (1, 1, 1, 1)})]
TRANSFER_CHANGES = [{"in_channels": 1}, {"in_channels": 5}, {"nb_classes": 7}]
FAMILY_OF = {"resnet18": "resnet", "vit_tiny_patch16_224": "vit", "convnext_tiny": "convnext"}


def transfer_case_id(name, change):
    return name + "-" + "-".join(f"{k}={v}" for k, v in change.items())


@pytest.mark.parametrize("name,ov", TRANSFER_MODELS)
@pytest.mark.parametrize("change", TRANSFER_CHANGES)
def test_transfer_weights_equals_reference(name, ov, change, pins):
    """in_channels / nb_classes adaptation (tfimm/models/factory.py:174-305; tests/models/test_factory.py:37-90):
    the engine's transfer_weights writes the same values into the same variables as the reference's."""
    import tfimm

    arrays, meta = pins
    case = transfer_case_id(name, change)
    rec = meta["transfer"][case]
    omod = importlib.import_module(f"oracle.{FAMILY_OF[name]}")
    w = params.random_params(omod.param_shapes(_engine_cfg(name, ov)), seed=17)
    src = tfimm.create_model(name, device="cpu", **ov)
    src.load_weights_dict(w)
    dst = tfimm.create_model(name, device="cpu", **ov, **change)
    init = dst.weights_dict()
    tfimm.models.transfer_weights(src, dst)
    got = dst.weights_dict()
    for k in rec["unchanged"]:
        if not np.array_equal(got[k], init[k]):
            raise AssertionError(f"{k}: the reference left it at its initial value, the engine overwrote it")
    off = rec["offset"]
    for k, shape in rec["changed"]:   # a fixed sample of each variable the reference's transfer wrote
        assert list(np.shape(got[k])) == shape, k
        flat = np.asarray(got[k], dtype=np.float32).reshape(-1)
        idx = sample_index(flat.size, TRANSFER_SAMPLE)
        assert np.abs(flat[idx] - arrays["transfer_values"][off:off + len(idx)]).max() < 1e-6, k
        off += len(idx)


STATE_DICT_ARCHS = ["resnet50", "vit_b_16"]


def state_dict_case(arch):
    """(registered name, overrides, seeded timm-style state dict) of a torchvision architecture."""
    import torchvision

    if arch == "resnet50":
        tv = torchvision.models.resnet50(weights=None)
        name, ov = "resnet50", {"input_size": (32, 32)}
        sd = {k: v for k, v in tv.state_dict().items()}
    else:
        tv = torchvision.models.VisionTransformer(image_size=32, patch_size=8, num_layers=2, num_heads=2, hidden_dim=16,
                                                  mlp_dim=64, num_classes=10)
        name, ov = "vit_tiny_patch16_224", {"input_size": (32, 32), "patch_size": 8, "embed_dim": 16, "nb_blocks": 2,
                                             "nb_heads": 2, "nb_classes": 10}
        # torchvision -> timm key names (the reference converts timm checkpoints)
        sd = {}
        for k, v in tv.state_dict().items():
            k = (k.replace("encoder.layers.encoder_layer_", "blocks.").replace("ln_1", "norm1").replace("ln_2", "norm2")
                 .replace("self_attention.in_proj_", "attn.qkv.").replace("self_attention.out_proj", "attn.proj")
                 .replace("mlp.0", "mlp.fc1").replace("mlp.3", "mlp.fc2").replace("encoder.ln", "norm")
                 .replace("conv_proj", "patch_embed.proj").replace("heads.head", "head")
                 .replace("class_token", "cls_token").replace("encoder.pos_embedding", "pos_embed"))
            sd[k] = v
    g = torch.Generator().manual_seed(0)
    sd = {k: (torch.randn(v.shape, generator=g) if v.is_floating_point() else v) for k, v in sd.items()}
    return name, ov, sd


@pytest.mark.parametrize("arch", STATE_DICT_ARCHS)
def test_pytorch_state_dict_conversion_equals_reference(arch, pins):
    """N1: tfimm.utils.timm.convert_state_dict produces exactly what the reference's
    load_pytorch_weights_in_tf2_model (tfimm/utils/timm.py:109-229) writes into its variables."""
    import tfimm
    from tfimm.utils import timm as etimm

    name, ov, sd = state_dict_case(arch)
    eng = tfimm.create_model(name, device="cpu", **ov)
    got, missing, unexpected = etimm.convert_state_dict(eng, sd)
    assert not missing
    # names and exact float32 values of every variable the reference loads (digest of the recorded set)
    assert params_digest(got) == pins[1]["state_dict"][arch]
