"""Records what the UNMODIFIED reference Segment Anything model computes into tests/golden/reference/sam_pins.npz, for
tests/test_sam_reference_pin_cpu.py.

    python tools/make_sam_pins.py        (needs the reference sources, see oracle/ref_runner.py and oracle/sam_ref.py)

Recorded: the ``sam`` registrations and the configs of sam_vit_b/l/h; the digest of the full variable table (names and
shapes) of every pinned configuration and of sam_vit_b/l/h; for each pinned configuration and input size, the image
embeddings (whole) and a fixed sample of every intermediate feature with its max-abs value, in float64 on seeded
weights and images; and the variables ``transfer_weights`` changes when the input size of the reference's test model
changes (whole), plus the names it leaves unchanged.  tests/golden/reference/pins.npz is not touched.
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

from oracle import params  # noqa: E402
from oracle import ref_runner as rr  # noqa: E402
from oracle import sam_ref  # noqa: E402
import test_sam_reference_pin_cpu as t  # noqa: E402

OUT = ROOT / "tests" / "golden" / "reference" / "sam_pins.npz"


def main():
    assert rr.available(), "the reference sources are needed to record the pins"
    arrays, meta = {}, {"tables": {}, "outputs": {}}
    feature_samples = []
    meta["registry"] = sam_ref.list_models("sam")
    meta["configs"] = {n: json.loads(json.dumps(sam_ref.model_config(n))) for n in t.REGISTERED}
    for name in t.CASES:
        if name != "sam_vit_test_model":
            sam_ref.register_test_model(name=name, **t.CASES[name][0])
    sam_ref.register_test_model()

    for name in t.REGISTERED:
        ref = sam_ref.create_model(name, input_size=t.TABLE_INPUT).build()
        meta["tables"][name] = t.table_digest(ref.weight_shapes())

    rr.set_floatx("float64")
    for name, (_, sizes) in t.CASES.items():
        ref = sam_ref.create_model(name).build()
        shapes = ref.weight_shapes()
        meta["tables"][name] = t.table_digest(shapes)
        meta.setdefault("order", {})[name] = list(shapes)   # the order random_params draws the weights in
        ref.assign(params.random_params(shapes, seed=t.weight_seed(name), dtype=torch.float64))
        for size in sizes:
            key = f"{name}@{size[0]}x{size[1]}"
            x = params.test_images(2, *size).double()
            y, feats = ref.image_encoder(x, return_features=True)
            assert y.dtype == torch.float64
            arrays[f"out/{key}"] = y.numpy()
            rec = {"shape": list(y.shape), "features": list(feats), "feature_absmax": [],
                   "feature_offset": int(sum(len(s) for s in feature_samples))}
            for v in feats.values():
                flat = v.reshape(-1).numpy()
                feature_samples.append(flat[t.sample_index(flat.size, t.FEATURE_SAMPLE)])
                rec["feature_absmax"].append(float(np.abs(flat).max()))
            meta["outputs"][key] = rec
    arrays["feature_samples"] = np.concatenate(feature_samples)
    rr.set_floatx("float32")

    name, size = t.TRANSFER
    src = sam_ref.create_model(name).build()
    w = params.random_params(src.weight_shapes(), seed=t.weight_seed(name))
    assert list(src.weight_shapes()) == meta["order"][name]
    src.assign(w)
    dst = sam_ref.create_model(name, input_size=size).build()
    rr.transfer_weights(src, dst)
    after = dst.weights_dict()
    meta["transfer"] = {"changed": [], "unchanged": []}
    for k, v in after.items():
        if v.shape == tuple(w[k].shape) and np.array_equal(v, w[k].numpy()):
            meta["transfer"]["unchanged"].append(k)
        else:
            meta["transfer"]["changed"].append(k)
            arrays[f"transfer/{k}"] = np.asarray(v, dtype=np.float32)

    arrays["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **arrays)
    print(OUT, OUT.stat().st_size, "bytes", "changed by transfer:", meta["transfer"]["changed"])


if __name__ == "__main__":
    main()
