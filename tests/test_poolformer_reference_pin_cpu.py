"""Pins the PoolFormer oracle (oracle/poolformer.py) and the engine's PoolFormer surface to the REFERENCE ITSELF.

``tools/make_poolformer_pins.py`` ran the unmodified reference ``tfimm/architectures/poolformer.py`` on the TensorFlow
shim (``oracle/poolformer_ref.py``) and recorded in ``tests/golden/reference/poolformer_pins.npz``: the five
registrations and their configs, the ordered variable table of every registration and pinned configuration, the logits
and a fixed sample of every feature in float64 on seeded weights and images (64 x 64; 61 x 45, whose stem padding and
pool edges are uneven; a configuration whose last stage is 1 x 1, where the pool minus x is exactly 0; poolformer_s12 at
224 px), the reference's initial values of its constant-initialised variables, and what the reference's PyTorch
converter makes of a timm-layout state dict.  Everything compares against that recording; where the reference sources
are present, the oracle is also compared with the reference run live.
"""
import json
import sys
from pathlib import Path
from types import SimpleNamespace

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

PINS = ROOT / "tests" / "golden" / "reference" / "poolformer_pins.npz"
FEATURE_SAMPLE = 64
CASES = {
    "pin_pf_64": dict(input_size=(64, 64), embed_dim=(8, 16, 24, 32), nb_blocks=(1, 1, 2, 1), init_scale=0.3,
                      nb_classes=5),
    "pin_pf_61x45": dict(input_size=(61, 45), embed_dim=(16, 8, 24, 16), nb_blocks=(1, 2, 1, 1), init_scale=0.5,
                         nb_classes=3),
    # stem 8 x 8, then 4 x 4, 2 x 2 and a 1 x 1 last stage
    "pin_pf_last1x1": dict(input_size=(32, 32), embed_dim=(8, 16, 16, 24), nb_blocks=(1, 1, 1, 2), init_scale=0.4,
                           nb_classes=0),
}
OUTPUT_CASES = tuple(CASES) + ("poolformer_s12",)
INIT_CASES = ("pin_pf_64",)
CONVERT_CASES = ("pin_pf_61x45",)
_CONST_LEAVES = ("layer_scale_1", "layer_scale_2", "gamma", "beta", "bias")


def weight_seed(name):
    return 61 + sorted(OUTPUT_CASES).index(name)


def weights_for(shapes, name):
    return params.random_params(shapes, seed=weight_seed(name), dtype=torch.float64)


def images_for(name):
    size = CASES[name]["input_size"] if name in CASES else (224, 224)
    return params.test_images(2 if name in CASES else 1, *size).double()


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
def poolformer():
    import importlib
    from copy import deepcopy

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


def _cfg(poolformer, name):
    import tfimm

    if name in CASES:
        return poolformer.PoolFormerConfig(name=name, **CASES[name])
    return tfimm.models.registry.model_config(name)


def test_registrations_and_configs(pins, poolformer):
    import dataclasses

    import tfimm

    _, meta = pins
    assert sorted(tfimm.list_models(module="poolformer")) == sorted(meta["registry"]) and len(meta["registry"]) == 5
    for name, ref in meta["configs"].items():
        got = json.loads(json.dumps(dataclasses.asdict(tfimm.models.registry.model_config(name))))
        assert got == ref, name


def test_variable_tables(pins, poolformer):
    """Names, shapes and creation order of every registration and pinned configuration: the engine's and the oracle's."""
    from oracle import poolformer as op

    _, meta = pins
    for name, digest in meta["tables"].items():
        cfg = _cfg(poolformer, name)
        engine = {k: tuple(v.shape) for k, v in poolformer.PoolFormer(cfg, device="meta").params.items()}
        assert table_digest(engine, ordered=True) == digest, name
        assert table_digest(op.param_shapes(cfg), ordered=True) == digest, name


def _oracle_outputs(poolformer, name):
    from oracle import poolformer as op

    cfg = _cfg(poolformer, name)
    w = weights_for(op.param_shapes(cfg), name)
    return op.forward(cfg, w, images_for(name), return_features=True)


@pytest.mark.parametrize("name", OUTPUT_CASES)
def test_oracle_matches_reference(pins, poolformer, name):
    """The float64 oracle equals the recorded reference to 1e-12 (relative to the largest value), logits and every
    feature."""
    arrays, meta = pins
    y, feats = _oracle_outputs(poolformer, name)
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
    if name == "pin_pf_last1x1":
        # on a 1 x 1 image the pool is x itself: the token mixer adds exactly nothing
        assert feats["stage_3/block_0"].shape[1:3] == (1, 1)


@pytest.mark.skipif(not rr.available(), reason="the reference sources are not present")
@pytest.mark.parametrize("name", tuple(CASES))
def test_oracle_matches_live_reference(poolformer, name):
    """Where the reference sources are present: the oracle against the reference run now, to 1e-12."""
    from oracle import poolformer_ref

    poolformer_ref.register_test_model(name, **CASES[name])
    rr.set_floatx("float64")
    try:
        ref = poolformer_ref.create_model(name)
        with rr._reference_modules(), torch.no_grad():
            ref.model(ref.model.dummy_inputs, training=False)
        ref.assign(weights_for(ref.weight_shapes(), name))
        ry, rfeats = ref(images_for(name), return_features=True)
    finally:
        rr.set_floatx("float32")
    y, feats = _oracle_outputs(poolformer, name)
    assert list(feats) == list(rfeats)
    for k in feats:
        assert (feats[k] - rfeats[k]).abs().max().item() <= 1e-12 * rfeats[k].abs().max().item(), k


@pytest.mark.parametrize("name", INIT_CASES)
def test_initial_values(pins, poolformer, name):
    """The constant-initialised variables start where the reference's do (layer scales at init_scale, GroupNorm 1 / 0,
    zero biases)."""
    arrays, meta = pins
    m = poolformer.PoolFormer(_cfg(poolformer, name), device="cpu")
    keys = meta["init"][name]
    assert keys
    for k in keys:
        np.testing.assert_array_equal(m.params[k].numpy(), arrays[f"init/{name}/{k}"], err_msg=k)


@pytest.mark.parametrize("name", CONVERT_CASES)
def test_state_dict_conversion(pins, poolformer, name):
    """tfimm.utils.timm.load_pytorch_weights_in_model turns a timm-layout state dict into exactly what the reference's
    converter does."""
    from tfimm.utils.timm import load_pytorch_weights_in_model

    arrays, meta = pins
    m = poolformer.PoolFormer(_cfg(poolformer, name), device="cpu")
    table = {k: tuple(v) for k, v in meta["order"][name]}
    missing, unexpected = load_pytorch_weights_in_model(m, state_dict_for(table, seed=weight_seed(name)))
    assert not missing and not unexpected
    for k in table:
        np.testing.assert_array_equal(m.params[k].numpy(), arrays[f"convert/{name}/{k}"], err_msg=k)
