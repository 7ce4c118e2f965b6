"""Records what the UNMODIFIED reference PoolFormer module computes into tests/golden/reference/poolformer_pins.npz, for
tests/test_poolformer_reference_pin_cpu.py.

    python tools/make_poolformer_pins.py      (needs the reference sources, see oracle/ref_runner.py)

Recorded: the ``poolformer`` registrations and their configs; the ordered digest of the variable table of every
registration and pinned configuration; for each pinned configuration the logits and a fixed sample of every feature
with its max-abs value, in float64 on seeded weights and images; the reference's initial values of its constant-
initialised variables; and the weights the reference's PyTorch converter makes of a timm-layout state dict.
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tensorflow-image-models_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import params  # noqa: E402
from oracle import poolformer_ref  # noqa: E402
from oracle import ref_runner as rr  # noqa: E402
import test_poolformer_reference_pin_cpu as t  # noqa: E402

OUT = ROOT / "tests" / "golden" / "reference" / "poolformer_pins.npz"


def build(name, **kw):
    ref = poolformer_ref.create_model(name, **kw)
    with rr._reference_modules(), torch.no_grad():
        ref.model(ref.model.dummy_inputs, training=False)   # Keras builds lazily
    return ref


def main():
    assert rr.available(), "the reference sources are needed to record the pins"
    arrays, meta = {}, {"tables": {}, "outputs": {}, "init": {}, "order": {}}
    meta["registry"] = poolformer_ref.list_models("poolformer")
    meta["configs"] = {n: json.loads(json.dumps(poolformer_ref.model_config(n))) for n in meta["registry"]}
    for name, fields in t.CASES.items():
        poolformer_ref.register_test_model(name, **fields)
    for name in meta["registry"]:
        meta["tables"][name] = t.table_digest(build(name).weight_shapes(), ordered=True)
        print(name, flush=True)

    for name in t.INIT_CASES:
        ref = build(name)
        keys = [k for k in ref.weight_shapes() if t.is_constant_init(k)]
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
    for name in t.OUTPUT_CASES:
        ref = build(name)
        shapes = ref.weight_shapes()
        meta["tables"][name] = t.table_digest(shapes, ordered=True)
        meta["order"][name] = [[k, list(v)] for k, v in shapes.items()]
        ref.assign(t.weights_for(shapes, name))
        x = t.images_for(name)
        y, feats = ref(x, return_features=True)
        assert y.dtype == torch.float64
        arrays[f"out/{name}"] = y.numpy()
        rec = {"features": list(feats), "feature_absmax": [], "feature_offset": int(sum(len(s) for s in samples))}
        for v in feats.values():
            flat = v.reshape(-1).numpy()
            samples.append(flat[t.sample_index(flat.size, t.FEATURE_SAMPLE)])
            rec["feature_absmax"].append(float(np.abs(flat).max()))
        meta["outputs"][name] = rec
        print(name, flush=True)
    arrays["feature_samples"] = np.concatenate(samples)
    rr.set_floatx("float32")

    arrays["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **arrays)
    print(OUT, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
