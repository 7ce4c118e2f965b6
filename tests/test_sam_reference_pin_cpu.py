"""Pins the Segment Anything oracle (oracle/sam.py) and the engine's SAM surface to the REFERENCE ITSELF.

``tools/make_sam_pins.py`` ran the unmodified reference modules (tfimm/architectures/segment_anything/*.py) on the
TensorFlow shim (``oracle/sam_ref.py``) and recorded in ``tests/golden/reference/sam_pins.npz``: the registrations and
configs of sam_vit_b/l/h, the full variable table (names and shapes) of every model below, the image embeddings and
intermediate features in float64 on seeded weights and images, and the weights ``transfer_weights`` writes when the
input size changes.  Everything below compares against that recording, so it runs without the reference.
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
from test_reference_pin_cpu import sample_index, table_digest  # noqa: E402

PINS = ROOT / "tests" / "golden" / "reference" / "sam_pins.npz"
FEATURE_SAMPLE = 64

# the reference's own test configuration (tests/models/test_segment_anything.py:55-72 of the reference: 32 x 32, patch
# 4, window 2, global block 1, fixed_input_size=False) and variants: name -> (config overrides, input sizes)
CASES = {
    "sam_vit_test_model": ({}, [(32, 32), (24, 40)]),
    # grid 10 with window 4: windows padded to 12 on the right and bottom (and 6 x 10 -> 8 x 12 at the second size)
    "sam_pin_pad": (dict(input_size=(40, 40), encoder_embed_dim=16, encoder_nb_heads=2, encoder_window_size=4,
                         embed_dim=16), [(40, 40), (24, 40)]),
    # head_dim 80 (sam_vit_h's), fixed input size
    "sam_pin_dh80": (dict(input_size=(24, 24), encoder_embed_dim=160, encoder_nb_heads=2, encoder_nb_blocks=2,
                          encoder_window_size=4, embed_dim=16, fixed_input_size=True), [(24, 24)]),
}
REGISTERED = ("sam_vit_b", "sam_vit_l", "sam_vit_h")
# The registered models' variable tables are recorded at this input size: building a Keras model runs it once, and a
# 1024 x 1024 forward of sam_vit_h on the shim takes far too long.  Only pos_embed and the global blocks' tables depend
# on the input size; test_sam_cpu.py::test_variable_table checks the 1024 x 1024 parameter counts.
TABLE_INPUT = (64, 64)
TRANSFER = ("sam_vit_test_model", (48, 48))


def weight_seed(name):
    return 31 + sorted(CASES).index(name)


def engine_overrides(name):
    """create_model overrides of sam_vit_b that give the configuration of a pinned case."""
    from oracle import sam_ref

    base = {k: v for k, v in sam_ref.TEST_MODEL_FIELDS.items() if k != "name"}
    return {**base, **CASES[name][0]}


@pytest.fixture(scope="module")
def pins():
    with np.load(PINS) as z:
        arrays = {k: z[k] for k in z.files}
    return arrays, json.loads(arrays.pop("meta").tobytes())


@pytest.fixture
def sam():
    import importlib
    from copy import deepcopy

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


def _weights(name, meta, dtype):
    """The seeded weights the recording used: ``random_params`` over the reference's variables in the reference's
    order (the draws are sequential)."""
    from oracle import sam as osam

    table = osam.param_shapes(_cfg(name))
    return params.random_params({k: table[k] for k in meta["order"][name]}, seed=weight_seed(name), dtype=dtype)


def _cfg(name):
    import tfimm

    return tfimm.create_model("sam_vit_b", device="meta", **engine_overrides(name)).cfg


def test_registrations_and_configs_equal_the_reference(sam, pins):
    import dataclasses

    from tfimm.models import list_models, model_config

    _, meta = pins
    assert list_models(module="sam") == meta["registry"]
    for name in REGISTERED:
        got = json.loads(json.dumps(dataclasses.asdict(model_config(name))))
        assert got == meta["configs"][name], name


@pytest.mark.parametrize("name", list(CASES) + list(REGISTERED))
def test_variable_tables_equal_the_reference(sam, pins, name):
    """Names and shapes of every variable -- image encoder, prompt encoder, mask decoder -- of the engine's model and of
    the oracle's table equal the reference's."""
    import tfimm
    from oracle import sam as osam

    _, meta = pins
    ov = engine_overrides(name) if name in CASES else {"input_size": TABLE_INPUT}
    model = tfimm.create_model(name if name in REGISTERED else "sam_vit_b", device="meta", **ov)
    assert table_digest({k: tuple(v.shape) for k, v in model.params.items()}) == meta["tables"][name]
    assert table_digest(osam.param_shapes(model.cfg)) == meta["tables"][name]


def _case_index():
    return [(name, size) for name, (_, sizes) in CASES.items() for size in sizes]


@pytest.mark.parametrize("name,size", _case_index())
def test_oracle_equals_the_reference(sam, pins, name, size):
    """oracle/sam.py in float64 reproduces what the reference computed in float64 to 1e-12 (embeddings, every feature)."""
    from oracle import sam as osam

    arrays, meta = pins
    rec = meta["outputs"][f"{name}@{size[0]}x{size[1]}"]
    cfg = _cfg(name)
    w = _weights(name, meta, torch.float64)
    x = params.test_images(2, *size).double()
    y, feats = osam.image_encoder(cfg, w, x, return_features=True)
    assert list(y.shape) == rec["shape"]
    ref = arrays[f"out/{name}@{size[0]}x{size[1]}"]
    assert np.abs(y.numpy() - ref).max() <= 1e-12 * np.abs(ref).max()
    assert list(feats) == rec["features"]
    samples = arrays["feature_samples"][rec["feature_offset"]:]
    off = 0
    for k, absmax in zip(feats, rec["feature_absmax"]):
        flat = feats[k].reshape(-1).numpy()
        idx = sample_index(flat.size, FEATURE_SAMPLE)
        assert np.abs(flat[idx] - samples[off:off + idx.size]).max() <= 1e-12 * absmax, k
        off += idx.size


def test_transform_weights_equal_the_reference(sam, pins, tmp_path):
    """create_model(..., input_size=) resizes pos_embed and the global blocks' tables as the reference's
    transfer_weights does (reference sam.py:158-203); the other variables are copied."""
    import tfimm
    from oracle import sam as osam
    from tfimm.models import register_model, save_weights

    arrays, meta = pins
    name, size = TRANSFER
    fields = engine_overrides(name)

    def sam_vit_test_model():
        return sam.SegmentAnythingModel, sam.SegmentAnythingModelConfig(name="sam_vit_test_model", **fields)

    register_model(sam_vit_test_model)
    src = tfimm.create_model(name, device="cpu", precision="fp32")
    w = _weights(name, meta, torch.float32)
    src.load_weights_dict(w)
    path = str(tmp_path / "w.npz")
    save_weights(src, path)
    dst = tfimm.create_model(name, model_path=path, device="cpu", precision="fp32", input_size=size)
    changed = meta["transfer"]["changed"]
    assert set(changed) | set(meta["transfer"]["unchanged"]) == set(dst.params)
    for k in changed:
        ref = arrays[f"transfer/{k}"]
        got = dst.params[k].cpu().numpy()
        assert got.shape == ref.shape, k
        assert np.abs(got - ref).max() <= 1e-6 * max(np.abs(ref).max(), 1.0), k
    for k in meta["transfer"]["unchanged"]:
        assert torch.equal(dst.params[k].cpu(), w[k]), k
