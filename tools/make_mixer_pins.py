"""Records what the UNMODIFIED reference MLP-Mixer module computes into tests/golden/reference/mixer_pins.npz, for
tests/test_mixer_reference_pin_cpu.py.

    python tools/make_mixer_pins.py      (needs the reference sources, see oracle/ref_runner.py and oracle/mixer_ref.py)

Recorded: the ``mlp_mixer`` registrations and their configs; the digest of the variable table (names, shapes, creation
order) of every registration and pinned configuration; for each pinned configuration, the logits (whole) and a fixed
sample of every feature with its max-abs value, in float64 on seeded weights and images; the reference's initial values
of its constant-initialised variables; and the weights the reference's PyTorch converter makes of a timm-layout state
dict.  The other pin files are not touched.
"""
import dataclasses
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tensorflow-image-models_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import mixer_ref  # noqa: E402
from oracle import params  # noqa: E402
from oracle import ref_runner as rr  # noqa: E402
import test_mixer_reference_pin_cpu as t  # noqa: E402

OUT = ROOT / "tests" / "golden" / "reference" / "mixer_pins.npz"


def build(name, **kw):
    ref = mixer_ref.create_model(name, **kw)
    with rr._reference_modules(), torch.no_grad():
        ref.model(ref.model.dummy_inputs, training=False)   # Keras builds lazily
    return ref


def main():
    assert rr.available(), "the reference sources are needed to record the pins"
    arrays, meta = {}, {"tables": {}, "outputs": {}, "init": {}, "order": {}}
    meta["registry"] = mixer_ref.list_models("mlp_mixer")
    meta["configs"] = {n: json.loads(json.dumps(mixer_ref.model_config(n))) for n in meta["registry"]}
    for name, fields in t.CASES.items():
        mixer_ref.register_test_model(name, **fields)
    for name in meta["registry"]:
        meta["tables"][name] = t.table_digest(build(name).weight_shapes(), ordered=True)
        print(name, flush=True)

    for name in t.INIT_CASES:   # float32, default initialisers
        ref = build(name)
        mlp_layer = t.CASES[name].get("mlp_layer", "mlp")
        keys = [k for k in ref.weight_shapes() if t.is_constant_init(k, mlp_layer)]
        meta["init"][name] = keys
        wd = ref.weights_dict()
        for k in keys:
            arrays[f"init/{name}/{k}"] = np.asarray(wd[k], dtype=np.float32)

    for name in t.CONVERT_CASES:
        ref = build(name)
        table = ref.weight_shapes()
        rr.load_pytorch_weights(ref, t.state_dict_for(table, seed=t.weight_seed(name)))
        for k, v in ref.weights_dict().items():
            arrays[f"convert/{name}/{k}"] = np.asarray(v, dtype=np.float32)

    rr.set_floatx("float64")
    samples = []
    for name in t.CASES:
        ref = build(name)
        shapes = ref.weight_shapes()
        meta["tables"][name] = t.table_digest(shapes, ordered=True)
        meta["order"][name] = [[k, list(v)] for k, v in shapes.items()]
        ref.assign(params.random_params(shapes, seed=t.weight_seed(name), dtype=torch.float64))
        x = params.test_images(2, *t.CASES[name]["input_size"]).double()
        y, feats = ref(x, return_features=True)
        assert y.dtype == torch.float64
        arrays[f"out/{name}"] = y.numpy()
        rec = {"features": list(feats), "feature_absmax": [], "feature_offset": int(sum(len(s) for s in samples))}
        for v in feats.values():
            flat = v.reshape(-1).numpy()
            samples.append(flat[t.sample_index(flat.size, t.FEATURE_SAMPLE)])
            rec["feature_absmax"].append(float(np.abs(flat).max()))
        meta["outputs"][name] = rec
    arrays["feature_samples"] = np.concatenate(samples)
    rr.set_floatx("float32")

    arrays["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **arrays)
    print(OUT, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
