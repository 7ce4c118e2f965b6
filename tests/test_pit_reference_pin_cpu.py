"""Pins the PiT oracle (oracle/pit.py) and the engine's PiT surface to the REFERENCE ITSELF.

``tools/make_pit_pins.py`` ran the unmodified reference ``tfimm/architectures/pit.py`` on the TensorFlow shim
(``oracle/pit_ref.py``) and recorded in ``tests/golden/reference/pit_pins.npz``: the eight registrations and their
configs, the ordered variable table of every registration and pinned configuration, the logits and a fixed sample of
every feature in float64 on seeded weights and images (a plain and a distilled configuration at their native input, at
head dims 32 and 48; an ``interpolate_input`` configuration fed a non-square image whose grids are 7 x 4, 4 x 2 and
2 x 1; a distilled configuration with ``nb_classes = 0``; pit_ti_224 at 224 px), the reference's initial values of its
constant-initialised variables, and the SHA-256 of what the reference's PyTorch converter makes of a timm-layout
state dict.
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

PINS = ROOT / "tests" / "golden" / "reference" / "pit_pins.npz"
FEATURE_SAMPLE = 64
CASES = {
    # grid 5 x 5 -> 3 x 3 -> 2 x 2, head dim 32
    "pin_pit_plain": dict(input_size=(48, 48), embed_dim=(32, 64, 128), nb_heads=(1, 2, 4), nb_blocks=(1, 2, 1),
                          nb_classes=5),
    # patch 8 / stride 4: grid 9 x 13 -> 5 x 7 -> 3 x 4, head dim 48, two token rows
    "pin_pit_dist": dict(input_size=(40, 56), patch_size=8, stride=4, embed_dim=(48, 96, 192), nb_heads=(1, 2, 4),
                         nb_blocks=(1, 1, 2), distilled=True, classifier=("head", "head_dist"), nb_classes=3),
    # pos_embed made for 5 x 5, resized to the 7 x 4 grid of a 64 x 40 image (IMAGE_SIZES); then 4 x 2 and 2 x 1
    "pin_pit_interp": dict(input_size=(48, 48), embed_dim=(32, 64, 128), nb_heads=(1, 1, 2), nb_blocks=(1, 1, 1),
                           interpolate_input=True, nb_classes=4),
    # grid 3 x 3 -> 2 x 2 -> 1 x 1; no head: the logits are the two normalised token rows
    "pin_pit_noclass": dict(input_size=(32, 32), embed_dim=(32, 64, 128), nb_heads=(1, 2, 2), nb_blocks=(1, 1, 1),
                            distilled=True, classifier=("head", "head_dist"), nb_classes=0),
}
IMAGE_SIZES = {"pin_pit_interp": (64, 40)}
OUTPUT_CASES = tuple(CASES) + ("pit_ti_224",)
INIT_CASES = ("pin_pit_dist",)
CONVERT_CASES = ("pin_pit_dist",)
_CONST_LEAVES = ("gamma", "beta", "bias")


def weight_seed(name):
    return 61 + sorted(OUTPUT_CASES).index(name)


def weights_for(shapes, name):
    return params.random_params(shapes, seed=weight_seed(name), dtype=torch.float64)


def images_for(name):
    size = IMAGE_SIZES.get(name, CASES[name]["input_size"]) if name in CASES else (224, 224)
    return params.test_images(2 if name in CASES else 1, *size).double()


def array_digest(a):
    """SHA-256 of an array's float32 bytes: the converted weights are compared bit for bit without storing them."""
    import hashlib

    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def is_constant_init(key):
    return key.rsplit("/", 1)[-1] in _CONST_LEAVES


def state_dict_for(table, seed):
    """A timm-layout state dict for a variable table: PyTorch names, (out, in, kh, kw) kernels."""
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
def pit():
    import importlib
    from copy import deepcopy

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


def _cfg(pit, name):
    import tfimm

    if name in CASES:
        return pit.PoolingVisionTransformerConfig(name=name, **CASES[name])
    return tfimm.models.registry.model_config(name)


def test_registrations_and_configs(pins, pit):
    import dataclasses

    import tfimm

    _, meta = pins
    assert sorted(tfimm.list_models(module="pit")) == sorted(meta["registry"]) and len(meta["registry"]) == 8
    for name, ref in meta["configs"].items():
        got = json.loads(json.dumps(dataclasses.asdict(tfimm.models.registry.model_config(name))))
        assert got == ref, name


def test_variable_tables(pins, pit):
    """Names, shapes and creation order of every registration and pinned configuration: the engine's and the oracle's."""
    from oracle import pit as op

    _, meta = pins
    for name, digest in meta["tables"].items():
        cfg = _cfg(pit, name)
        engine = {k: tuple(v.shape) for k, v in pit.PoolingVisionTransformer(cfg, device="meta").params.items()}
        assert table_digest(engine, ordered=True) == digest, name
        assert table_digest(op.param_shapes(cfg), ordered=True) == digest, name


def _oracle_outputs(pit, name):
    from oracle import pit as op

    cfg = _cfg(pit, name)
    w = weights_for(op.param_shapes(cfg), name)
    return op.forward(cfg, w, images_for(name), return_features=True)


@pytest.mark.parametrize("name", OUTPUT_CASES)
def test_oracle_matches_reference(pins, pit, name):
    """The float64 oracle equals the recorded reference to 1e-12 (relative to the largest value), logits and every
    feature."""
    arrays, meta = pins
    y, feats = _oracle_outputs(pit, name)
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
def test_oracle_matches_live_reference(pit, name):
    """Where the reference sources are present: the oracle against the reference run now, to 1e-12."""
    from oracle import pit_ref

    pit_ref.register_test_model(name, **CASES[name])
    rr.set_floatx("float64")
    try:
        ref = pit_ref.create_model(name)
        with rr._reference_modules(), torch.no_grad():
            ref.model(ref.model.dummy_inputs, training=False)
        ref.assign(weights_for(ref.weight_shapes(), name))
        ry, rfeats = ref(images_for(name), return_features=True)
    finally:
        rr.set_floatx("float32")
    y, feats = _oracle_outputs(pit, name)
    assert list(feats) == list(rfeats)
    for k in feats:
        assert (feats[k] - rfeats[k]).abs().max().item() <= 1e-12 * rfeats[k].abs().max().item(), k


@pytest.mark.parametrize("name", INIT_CASES)
def test_initial_values(pins, pit, name):
    """The constant-initialised variables start where the reference's do (LayerNorm 1 / 0, zero biases)."""
    arrays, meta = pins
    m = pit.PoolingVisionTransformer(_cfg(pit, name), device="cpu")
    keys = meta["init"][name]
    assert keys
    for k in keys:
        np.testing.assert_array_equal(m.params[k].numpy(), arrays[f"init/{name}/{k}"], err_msg=k)


@pytest.mark.parametrize("name", CONVERT_CASES)
def test_state_dict_conversion(pins, pit, name):
    """tfimm.utils.timm.load_pytorch_weights_in_model turns a timm-layout state dict into exactly what the reference's
    converter does."""
    from tfimm.utils.timm import load_pytorch_weights_in_model

    arrays, meta = pins
    m = pit.PoolingVisionTransformer(_cfg(pit, name), device="cpu")
    table = {k: tuple(v) for k, v in meta["order"][name]}
    missing, unexpected = load_pytorch_weights_in_model(m, state_dict_for(table, seed=weight_seed(name)))
    assert not missing and not unexpected
    assert set(table) == set(meta["convert"][name])
    for k in table:
        assert array_digest(m.params[k].numpy()) == meta["convert"][name][k], k
