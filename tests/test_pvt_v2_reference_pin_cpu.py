"""Pins the PVT v2 oracle (oracle/pvt_v2.py) and the engine's PVT v2 surface to the REFERENCE ITSELF.

``tools/make_pvt_v2_pins.py`` ran the unmodified reference ``tfimm/architectures/pvt_v2.py`` on the TensorFlow shim
(``oracle/pvt_v2_ref.py``) and recorded in ``tests/golden/reference/pvt_v2_pins.npz``: the six registrations and their
configs, the ordered variable table of every registration and pinned configuration (the patch embeddings, the blocks,
the stage norms, the head: the lists in the order the model's __init__ assigns them), the logits and a fixed sample of
every feature in float64 on seeded weights and images (a small plain configuration; a pvt_v2_b1-shaped configuration
fed a 200 x 264 image, whose padded convolutions round the grids up to 50 x 66, 25 x 33, 13 x 17 and 7 x 9, which no
spatial-reduction ratio divides; ``nb_classes = 0``; pvt_v2_b0 at 224 px), the reference's initial values of its
constant-initialised variables, and the SHA-256 of what the reference's PyTorch converter makes of a state dict in the
official PVT v2 layout (depthwise (C, 1, 3, 3) kernels included).
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

PINS = ROOT / "tests" / "golden" / "reference" / "pvt_v2_pins.npz"
FEATURE_SAMPLE = 64
_SMALL = dict(embed_dim=(32, 64, 32, 64), nb_heads=(1, 1, 1, 1), nb_blocks=(1, 1, 1, 1), mlp_ratio=(2.0, 2.0, 2.0, 1.0))
CASES = {
    # grids 16 x 16 -> 8 x 8 -> 4 x 4 -> 2 x 2; keys 16, 16, 4, 4; head dims 32 and 64
    "pin_pvt_v2_plain": dict(input_size=(64, 64), sr_ratio=(4, 2, 2, 1), nb_classes=5, **_SMALL),
    # pvt_v2_b1's widths and depths on a 200 x 264 image (IMAGE_SIZES): grids 50 x 66, 25 x 33, 13 x 17, 7 x 9; the sr
    # 8 / 4 / 2 convolutions drop the remainder rows and columns
    "pin_pvt_v2_b1_odd": dict(embed_dim=(64, 128, 320, 512), nb_blocks=(2, 2, 2, 2), nb_classes=7),
    # grids 8 x 8 -> 4 x 4 -> 2 x 2 -> 1 x 1; no head: the logits are the mean of the last stage's normalised tokens
    "pin_pvt_v2_noclass": dict(input_size=(32, 32), sr_ratio=(2, 1, 1, 1), nb_classes=0, **_SMALL),
}
IMAGE_SIZES = {"pin_pvt_v2_b1_odd": (200, 264)}
OUTPUT_CASES = tuple(CASES) + ("pvt_v2_b0",)
INIT_CASES = ("pin_pvt_v2_plain",)
CONVERT_CASES = ("pin_pvt_v2_plain",)
_CONST_LEAVES = ("gamma", "beta", "bias")


def weight_seed(name):
    return 71 + sorted(OUTPUT_CASES).index(name)


def weights_for(shapes, name):
    return params.random_params(shapes, seed=weight_seed(name), dtype=torch.float64)


def images_for(name):
    size = IMAGE_SIZES.get(name, CASES[name].get("input_size", (224, 224))) if name in CASES else (224, 224)
    return params.test_images(2 if name in CASES else 1, *size).double()


def array_digest(a):
    """SHA-256 of an array's float32 bytes: the converted weights are compared bit for bit without storing them."""
    import hashlib

    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def is_constant_init(key):
    return key.rsplit("/", 1)[-1] in _CONST_LEAVES


def state_dict_for(table, seed):
    """A state dict in the official PVT v2 layout for a variable table: PyTorch names, (out, in, kh, kw) kernels and
    (C, 1, kh, kw) depthwise kernels."""
    from tfimm.utils.timm import pytorch_key

    rng = np.random.default_rng(seed)
    sd = {}
    for k, shape in table.items():
        if k.endswith("/kernel") or k.endswith("/depthwise_kernel"):
            shape = (shape[3], shape[2], shape[0], shape[1]) if len(shape) == 4 else tuple(reversed(shape))
            if k.endswith("/depthwise_kernel"):
                shape = (shape[1], shape[0], shape[2], shape[3])
        sd[pytorch_key(k)] = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    return sd


@pytest.fixture(scope="module")
def pins():
    with np.load(PINS) as z:
        arrays = {k: z[k] for k in z.files}
    return arrays, json.loads(arrays.pop("meta").tobytes())


@pytest.fixture
def pvt():
    from pvt_v2_oracle import pvt_v2_registered

    with pvt_v2_registered() as mod:
        yield mod


def _cfg(pvt, name):
    import tfimm

    if name in CASES:
        return pvt.PyramidVisionTransformerV2Config(name=name, **CASES[name])
    return tfimm.models.registry.model_config(name)


def test_registrations_and_configs(pins, pvt):
    import dataclasses

    import tfimm

    _, meta = pins
    assert sorted(tfimm.list_models(module="pvt_v2")) == sorted(meta["registry"]) and len(meta["registry"]) == 6
    for name, ref in meta["configs"].items():
        got = json.loads(json.dumps(dataclasses.asdict(tfimm.models.registry.model_config(name))))
        assert got == ref, name


def test_variable_tables(pins, pvt):
    """Names, shapes and creation order of every registration and pinned configuration: the engine's and the
    oracle's."""
    from oracle import pvt_v2 as op

    _, meta = pins
    for name, digest in meta["tables"].items():
        cfg = _cfg(pvt, name)
        engine = {k: tuple(v.shape) for k, v in pvt.PyramidVisionTransformerV2(cfg, device="meta").params.items()}
        assert table_digest(engine, ordered=True) == digest, name
        assert table_digest(op.param_shapes(cfg), ordered=True) == digest, name


def _oracle_outputs(pvt, name):
    from oracle import pvt_v2 as op

    cfg = _cfg(pvt, name)
    w = weights_for(op.param_shapes(cfg), name)
    return op.forward(cfg, w, images_for(name), return_features=True)


@pytest.mark.parametrize("name", OUTPUT_CASES)
def test_oracle_matches_reference(pins, pvt, name):
    """The float64 oracle equals the recorded reference to 1e-12 (relative to the largest value), logits and every
    feature."""
    arrays, meta = pins
    y, feats = _oracle_outputs(pvt, name)
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
@pytest.mark.parametrize("name", ("pin_pvt_v2_plain", "pin_pvt_v2_noclass"))
def test_oracle_matches_live_reference(pvt, name):
    """Where the reference sources are present: the oracle against the reference run now, to 1e-12."""
    from oracle import pvt_v2_ref

    pvt_v2_ref.register_test_model(name, **CASES[name])
    rr.set_floatx("float64")
    try:
        ref = pvt_v2_ref.create_model(name)
        with rr._reference_modules(), torch.no_grad():
            ref.model(ref.model.dummy_inputs, training=False)
        ref.assign(weights_for(ref.weight_shapes(), name))
        ry, rfeats = ref(images_for(name), return_features=True)
    finally:
        rr.set_floatx("float32")
    y, feats = _oracle_outputs(pvt, name)
    assert list(feats) == list(rfeats)
    for k in feats:
        assert (feats[k] - rfeats[k]).abs().max().item() <= 1e-12 * rfeats[k].abs().max().item(), k


@pytest.mark.parametrize("name", INIT_CASES)
def test_initial_values(pins, pvt, name):
    """The constant-initialised variables start where the reference's do (LayerNorm 1 / 0, zero biases, the depthwise
    convolutions' included)."""
    arrays, meta = pins
    m = pvt.PyramidVisionTransformerV2(_cfg(pvt, name), device="cpu")
    keys = meta["init"][name]
    assert keys and "block1/0/mlp/dwconv/dwconv/bias" in keys and "norm4/gamma" in keys
    for k in keys:
        np.testing.assert_array_equal(m.params[k].numpy(), arrays[f"init/{name}/{k}"], err_msg=k)


@pytest.mark.parametrize("name", CONVERT_CASES)
def test_state_dict_conversion(pins, pvt, name):
    """tfimm.utils.timm.load_pytorch_weights_in_model turns an official PVT v2-layout state dict into exactly what the
    reference's converter does, the sr convolution's (C, C, sr, sr) -> (sr, sr, C, C) and the depthwise convolutions'
    (C, 1, 3, 3) -> (3, 3, C, 1) included."""
    from tfimm.utils.timm import load_pytorch_weights_in_model

    arrays, meta = pins
    m = pvt.PyramidVisionTransformerV2(_cfg(pvt, name), device="cpu")
    table = {k: tuple(v) for k, v in meta["order"][name]}
    assert any(k.endswith("/attn/sr/kernel") for k in table)
    assert any(k.endswith("/mlp/dwconv/dwconv/depthwise_kernel") for k in table)
    missing, unexpected = load_pytorch_weights_in_model(m, state_dict_for(table, seed=weight_seed(name)))
    assert not missing and not unexpected
    assert set(table) == set(meta["convert"][name])
    for k in table:
        assert array_digest(m.params[k].numpy()) == meta["convert"][name][k], k
