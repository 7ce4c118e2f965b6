"""Pins the CaiT oracle (oracle/cait.py) and the engine's CaiT surface to the REFERENCE ITSELF.

``tools/make_cait_pins.py`` ran the unmodified reference ``tfimm/architectures/cait.py`` on the TensorFlow shim
(``oracle/cait_ref.py``) and recorded in ``tests/golden/reference/cait_pins.npz``: the ten registrations and their
configs, the ordered variable table of every registration and pinned configuration (the model's cls_token and
pos_embed, then its layers in the order its __init__ assigns them: a block's gamma_1 / gamma_2 first, the attention's
qkv and proj before proj_l and proj_w), the initial values of the constant-initialised variables (gamma_1 / gamma_2
at init_scale 1e-5 and 1e-6, zero tokens), the SHA-256 of what the reference's PyTorch converter makes of a timm-layout
state dict, and the logits and a fixed sample of every feature in float64 on weights randomised away from their
initial values (non-symmetric proj_l / proj_w with non-zero biases, gamma_1 != gamma_2, a non-zero class token):
cait_xxs24_224 at 224 px, an H = 6 model with interpolate_input on a 208 x 272 image, and a headless model.
Everything compares against that recording; where the reference sources are present, the oracle is also compared with
the reference run live.
"""
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tensorflow-image-models_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import params  # noqa: E402
from oracle import ref_runner as rr  # noqa: E402
from test_reference_pin_cpu import sample_index, table_digest  # noqa: E402,F401

PINS = ROOT / "tests" / "golden" / "reference" / "cait_pins.npz"
FEATURE_SAMPLE = 64
CASES = {
    # H = 6 at head dim 48 (cait_xs's heads), two blocks; a 208 x 272 image: 13 x 17 patches from a 14 x 14 table
    "pin_cait_h6_interp": dict(embed_dim=288, nb_heads=6, nb_blocks=2, nb_classes=7, interpolate_input=True),
    # 2 x 3 patches, H = 2, no head: the logits are the normalised class row
    "pin_cait_noclass": dict(input_size=(32, 48), embed_dim=96, nb_heads=2, nb_blocks=2, nb_classes=0),
}
IMAGE_SIZES = {"pin_cait_h6_interp": (208, 272)}
OUTPUT_CASES = tuple(CASES) + ("cait_xxs24_224",)
INIT_CASES = ("cait_xxs24_224", "cait_s36_384")
CONVERT_CASES = ("pin_cait_noclass",)
_CONST = ("gamma", "beta", "bias", "gamma_1", "gamma_2", "cls_token", "pos_embed")


def weight_seed(name):
    return 31 + sorted(OUTPUT_CASES).index(name)


def weights_for(shapes, name):
    from cait_oracle import randomise

    w = randomise(params.random_params(shapes, seed=weight_seed(name)), weight_seed(name) + 100)
    return {k: v.double() for k, v in w.items()}


def images_for(name):
    size = IMAGE_SIZES.get(name, CASES[name].get("input_size", (224, 224))) if name in CASES else (224, 224)
    return params.test_images(2 if name in CASES else 1, *size).double()


def array_digest(a):
    """SHA-256 of an array's float32 bytes: the converted weights are compared bit for bit without storing them."""
    import hashlib

    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def is_constant_init(key):
    return key.rsplit("/", 1)[-1] in _CONST


def state_dict_for(table, seed):
    """A timm-layout CaiT state dict for a variable table: PyTorch names, (out, in) Linear weights, (out, in, kh, kw)
    convolution weights."""
    from tfimm.utils.timm import pytorch_key

    rng = np.random.default_rng(seed)
    sd = {}
    for k, shape in table.items():
        if k.endswith("/kernel"):
            shape = (shape[3], shape[2], shape[0], shape[1]) if len(shape) == 4 else tuple(reversed(shape))
        sd[pytorch_key(k)] = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    return sd


@pytest.fixture(scope="module")
def pins():
    with np.load(PINS) as z:
        arrays = {k: z[k] for k in z.files}
    return arrays, json.loads(arrays.pop("meta").tobytes())


@pytest.fixture
def cait():
    from cait_oracle import cait_registered

    with cait_registered() as mod:
        yield mod


def _cfg(cait, name):
    import tfimm

    if name in CASES:
        return cait.CaiTConfig(name=name, **CASES[name])
    return tfimm.models.registry.model_config(name)


def test_registrations_and_configs(pins, cait):
    import dataclasses

    import tfimm

    _, meta = pins
    assert sorted(tfimm.list_models(module="cait")) == sorted(meta["registry"]) and len(meta["registry"]) == 10
    for name, ref in meta["configs"].items():
        got = json.loads(json.dumps(dataclasses.asdict(tfimm.models.registry.model_config(name))))
        assert got == ref, name


def test_variable_tables(pins, cait):
    """Names, shapes and order of every registration and pinned configuration."""
    _, meta = pins
    assert set(meta["registry"]) | set(CASES) <= set(meta["tables"])
    for name, digest in meta["tables"].items():
        cfg = _cfg(cait, name)
        engine = {k: tuple(v.shape) for k, v in cait.CaiT(cfg, precision="fp32", device="meta").params.items()}
        assert table_digest(engine, ordered=True) == digest, name


def _oracle_outputs(cait, name, shapes):
    from oracle import cait as oc

    cfg = _cfg(cait, name)
    return oc.forward(cfg, weights_for(shapes, name), images_for(name), return_features=True)


@pytest.mark.parametrize("name", OUTPUT_CASES)
def test_oracle_matches_reference(pins, cait, name):
    """The float64 oracle equals the recorded reference to 1e-12 (relative to the largest value), logits and every
    feature."""
    arrays, meta = pins
    shapes = {k: tuple(v) for k, v in meta["order"][name]}
    w = weights_for(shapes, name)
    wl = w["blocks/0/attn/proj_l/kernel"]
    assert not torch.equal(wl, wl.t()) and w["blocks/0/attn/proj_w/bias"].abs().min() > 0
    assert not torch.equal(w["blocks/0/gamma_1"], w["blocks/0/gamma_2"]) and w["cls_token"].abs().max() > 0
    y, feats = _oracle_outputs(cait, name, shapes)
    ref = arrays[f"out/{name}"]
    assert np.abs(y.numpy() - ref).max() <= 1e-12 * np.abs(ref).max()
    rec = meta["outputs"][name]
    assert list(feats) == rec["features"]
    off = rec["feature_offset"]
    for v, amax in zip(feats.values(), rec["feature_absmax"]):
        flat = v.reshape(-1).numpy()
        s = flat[sample_index(flat.size, FEATURE_SAMPLE)]
        assert np.abs(s - arrays["feature_samples"][off:off + s.size]).max() <= 1e-12 * amax
        assert abs(np.abs(flat).max() - amax) <= 1e-12 * amax
        off += s.size


@pytest.mark.skipif(not rr.available(), reason="the reference sources are not present")
@pytest.mark.parametrize("name", tuple(CASES))
def test_oracle_matches_live_reference(cait, name):
    """Where the reference sources are present: the oracle against the reference run now, to 1e-12."""
    from oracle import cait_ref

    cait_ref.register_test_model(name, **CASES[name])
    rr.set_floatx("float64")
    try:
        ref = cait_ref.create_model(name)
        with rr._reference_modules(), torch.no_grad():
            ref.model(ref.model.dummy_inputs, training=False)
        shapes = ref.weight_shapes()
        ref.assign(weights_for(shapes, name))
        ry, rfeats = ref(images_for(name), return_features=True)
    finally:
        rr.set_floatx("float32")
    y, feats = _oracle_outputs(cait, name, shapes)
    assert list(feats) == list(rfeats)
    for k in feats:
        assert (feats[k] - rfeats[k]).abs().max().item() <= 1e-12 * rfeats[k].abs().max().item(), k


@pytest.mark.parametrize("name", INIT_CASES)
def test_initial_values(pins, cait, name):
    """The constant-initialised variables start where the reference's do: gamma_1 / gamma_2 at the registration's
    init_scale, LayerNorm 1 / 0, zero biases and tokens."""
    arrays, meta = pins
    m = cait.CaiT(_cfg(cait, name), device="cpu")
    keys = meta["init"][name]
    assert "blocks/0/gamma_1" in keys and "blocks_token_only/1/gamma_2" in keys and "cls_token" in keys
    for k in keys:
        np.testing.assert_array_equal(m.params[k].numpy(), arrays[f"init/{name}/{k}"], err_msg=k)


@pytest.mark.parametrize("name", CONVERT_CASES)
def test_state_dict_conversion(pins, cait, name):
    """tfimm.utils.timm.load_pytorch_weights_in_model turns a timm-layout state dict into exactly what the reference's
    converter does, the (H, H) proj_l / proj_w Linear weights and gamma_1 / gamma_2 included."""
    from tfimm.utils.timm import load_pytorch_weights_in_model

    arrays, meta = pins
    m = cait.CaiT(_cfg(cait, name), precision="fp32", device="cpu")
    table = {k: tuple(v) for k, v in meta["order"][name]}
    assert "blocks/0/attn/proj_l/kernel" in table and "blocks/1/gamma_2" in table
    missing, unexpected = load_pytorch_weights_in_model(m, state_dict_for(table, seed=weight_seed(name)))
    assert not missing and not unexpected
    assert set(table) == set(meta["convert"][name])
    for k in table:
        assert array_digest(m.params[k].numpy()) == meta["convert"][name][k], k
