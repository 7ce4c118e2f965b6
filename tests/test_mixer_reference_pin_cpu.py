"""Pins the MLP-Mixer oracle (oracle/mlp_mixer.py) and the engine's MLP-Mixer surface to the REFERENCE ITSELF.

``tools/make_mixer_pins.py`` ran the unmodified reference ``tfimm/architectures/mlp_mixer.py`` on the TensorFlow shim
(``oracle/mixer_ref.py``) and recorded in ``tests/golden/reference/mixer_pins.npz``: the 26 registrations and their
configs, the variable table (names and shapes, in creation order) of every registration and pinned configuration, the
logits and a fixed sample of every feature in float64 on seeded weights and images for small configurations of every
block type (token grids 7 x 7 and 5 x 6), the reference's initial values of the constant-initialised variables, and
what the reference's PyTorch converter makes of a timm-layout state dict.  Everything below compares against that
recording, so it runs without the reference.
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
from test_reference_pin_cpu import sample_index, table_digest  # noqa: E402

PINS = ROOT / "tests" / "golden" / "reference" / "mixer_pins.npz"
FEATURE_SAMPLE = 64
_SMALL = dict(patch_size=4, embed_dim=16, nb_blocks=2, nb_classes=5)
_IMNET = dict(mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
# name -> config fields (besides the name); inputs are 2 images of the config's input size
CASES = {
    "pin_mixer_7x7": dict(input_size=(28, 28), mlp_ratio=(0.5, 4.0), **_SMALL),
    "pin_mixer_5x6": dict(input_size=(20, 24), mlp_ratio=(1.0, 2.0), **_SMALL),
    "pin_gmixer_7x7": dict(input_size=(28, 28), mlp_ratio=(1.0, 4.0), mlp_layer="glu_mlp", act_layer="swish",
                           **_SMALL, **_IMNET),
    "pin_gmixer_5x6": dict(input_size=(20, 24), mlp_ratio=(1.0, 4.0), mlp_layer="glu_mlp", act_layer="swish",
                           **_SMALL),
    "pin_resmlp_7x7": dict(input_size=(28, 28), mlp_ratio=(4.0, 4.0), block_layer="res_block", norm_layer="affine",
                           init_values=1e-5, **_SMALL),
    "pin_resmlp_5x6": dict(input_size=(20, 24), mlp_ratio=(4.0, 4.0), block_layer="res_block", norm_layer="affine",
                           **_SMALL),
    "pin_gmlp_7x7": dict(input_size=(28, 28), mlp_ratio=(6.0, 6.0), block_layer="spatial_gating_block",
                         mlp_layer="gated_mlp", **_SMALL),
    "pin_gmlp_5x6": dict(input_size=(20, 24), mlp_ratio=(6.0, 6.0), block_layer="spatial_gating_block",
                         mlp_layer="gated_mlp", **_SMALL),
}
# configurations whose reference initial values and PyTorch conversion are recorded
INIT_CASES = ("pin_gmixer_7x7", "pin_resmlp_7x7", "pin_gmlp_5x6")
CONVERT_CASES = ("pin_resmlp_5x6", "pin_gmlp_5x6", "pin_gmixer_5x6")
# variables the reference initialises to constants (and GLU fc1 biases, whose gate half is ones)
_CONST_LEAVES = ("ls1", "ls2", "alpha", "beta", "gamma")


def weight_seed(name):
    return 41 + sorted(CASES).index(name)


def cfg_of(name):
    from tfimm.architectures.mlp_mixer import MLPMixerConfig

    return MLPMixerConfig(name=name, **CASES[name])


def is_constant_init(key, mlp_layer):
    leaf = key.rsplit("/", 1)[-1]
    return (leaf in _CONST_LEAVES or key.endswith("gate/proj/bias")
            or (mlp_layer == "glu_mlp" and key.endswith("fc1/bias")))


def state_dict_for(table, seed):
    """A timm-layout state dict for a variable table: PyTorch names, (out, in[, kh, kw]) kernels, ResMLP's Affine
    alpha / beta as (1, 1, C), as timm's checkpoints store them."""
    from tfimm.utils.timm import pytorch_key

    rng = np.random.default_rng(seed)
    sd = {}
    for k, shape in table.items():
        leaf = k.rsplit("/", 1)[-1]
        if leaf == "kernel":
            shape = (shape[3], shape[2], shape[0], shape[1]) if len(shape) == 4 else tuple(reversed(shape))
        elif leaf in ("alpha", "beta") and k.rsplit("/", 1)[0] + "/alpha" in table:
            shape = (1, 1, shape[0])
        sd[pytorch_key(k)] = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    return sd


@pytest.fixture(scope="module")
def pins():
    with np.load(PINS) as z:
        arrays = {k: z[k] for k in z.files}
    return arrays, json.loads(arrays.pop("meta").tobytes())


@pytest.fixture
def mixer():
    import importlib
    from copy import deepcopy

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


def test_registrations_and_configs(pins, mixer):
    import dataclasses

    import tfimm

    _, meta = pins
    assert sorted(tfimm.list_models(module="mlp_mixer")) == sorted(meta["registry"]) and len(meta["registry"]) == 26
    for name, ref in meta["configs"].items():
        got = json.loads(json.dumps(dataclasses.asdict(tfimm.models.registry.model_config(name))))
        assert got == ref, name


def test_variable_tables(pins, mixer):
    """Names, shapes and creation order of every registration and pinned configuration: the engine's and the oracle's."""
    import tfimm
    from oracle import mlp_mixer as om

    _, meta = pins
    for name, digest in meta["tables"].items():
        cfg = tfimm.models.registry.model_config(name) if name in meta["registry"] else cfg_of(name)
        engine = {k: tuple(v.shape) for k, v in mixer.MLPMixer(cfg, device="meta").params.items()}
        assert table_digest(engine, ordered=True) == digest, name
        assert table_digest(om.param_shapes(cfg), ordered=True) == digest, name


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference(pins, name):
    """The float64 oracle equals the reference to 1e-12 (relative to the largest value), logits and every feature."""
    from oracle import mlp_mixer as om

    arrays, meta = pins
    cfg = SimpleNamespace(name=name, **{**_defaults(), **CASES[name]})
    w = params.random_params(om.param_shapes(cfg), seed=weight_seed(name), dtype=torch.float64)
    x = params.test_images(2, *cfg.input_size).double()
    y, feats = om.forward(cfg, w, x, return_features=True)
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


def _defaults():
    import dataclasses

    from tfimm.architectures.mlp_mixer import MLPMixerConfig

    return {f.name: f.default for f in dataclasses.fields(MLPMixerConfig) if f.name != "name"}


@pytest.mark.parametrize("name", INIT_CASES)
def test_initial_values(pins, mixer, name):
    """The constant-initialised variables start where the reference's do (layer scales, Affine 1 / 0, LayerNorm 1 / 0,
    the gMLP gate's projection bias 1, the gate half of a GLU fc1 bias 1)."""
    arrays, meta = pins
    m = mixer.MLPMixer(cfg_of(name), device="cpu")
    keys = meta["init"][name]
    assert keys
    for k in keys:
        np.testing.assert_array_equal(m.params[k].numpy(), arrays[f"init/{name}/{k}"], err_msg=k)


@pytest.mark.parametrize("name", CONVERT_CASES)
def test_state_dict_conversion(pins, mixer, name):
    """tfimm.utils.timm.load_pytorch_weights_in_model turns a timm-layout state dict into exactly what the reference's
    converter does (ResMLP's (1, 1, C) alpha / beta, ls1 / ls2, the gMLP gate, the GLU fc1)."""
    from tfimm.utils.timm import load_pytorch_weights_in_model

    arrays, meta = pins
    m = mixer.MLPMixer(cfg_of(name), device="cpu")
    table = {k: tuple(v) for k, v in meta["order"][name]}
    sd = state_dict_for(table, seed=weight_seed(name))
    missing, unexpected = load_pytorch_weights_in_model(m, sd)
    assert not missing and not unexpected
    for k in table:
        np.testing.assert_array_equal(m.params[k].numpy(), arrays[f"convert/{name}/{k}"], err_msg=k)
