"""Records what the UNMODIFIED reference computes for tests/test_reference_pin_cpu.py into tests/golden/reference/pins.npz

    python tools/make_reference_pins.py        (needs the reference sources, see oracle/ref_runner.py)

The tests then compare the oracle / the engine's host-side API against this recording, so they run on any machine.
Large arrays are stored as a fixed, seeded sample of their elements together with their max-abs value (the
denominator of the tests' normalised error); name / shape tables and parameter sets compared for exact equality are
stored as truncated SHA-256 digests.  The small metadata (JSON) travels inside the compressed npz.
"""
import dataclasses
import importlib
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
import test_reference_pin_cpu as t  # noqa: E402

OUT = ROOT / "tests" / "golden" / "reference" / "pins.npz"


def main():
    assert rr.available(), "the reference sources are needed to record the pins"
    arrays, meta = {}, {"shim": [], "initial_values": {}, "transfer": {}, "state_dict": {}}
    logit_samples, feat_samples, feat_absmax, tr_values = [], [], [], []
    count = lambda chunks: int(sum(len(c) for c in chunks))  # noqa: E731

    rr.set_floatx("float64")
    for family, name, overrides in t.CASES:
        omod = importlib.import_module(f"oracle.{family}")
        ref = rr.create_model(name, **overrides)
        cfg = t._engine_cfg(name, overrides)
        w = params.random_params(omod.param_shapes(cfg), seed=31, dtype=torch.float64)
        ref.assign(w, ignore_missing=t.IGNORE)
        x = params.test_images(2, *cfg.input_size, cfg.in_channels).double()
        y_ref, f_ref = ref(x, return_features=True)
        loadable = {k: v for k, v in ref.weight_shapes().items() if not any(p in k for p in t.IGNORE)}
        rec = {"weights": t.table_digest(loadable), "features": t.table_digest({k: v.shape for k, v in f_ref.items()},
                                                                              ordered=True),
               "logits_shape": list(y_ref.shape), "logits_absmax": float(y_ref.abs().max()),
               "logits_offset": count(logit_samples), "feature_offset": count(feat_samples),
               "feature_index": len(feat_absmax)}
        flat = y_ref.reshape(-1)
        logit_samples.append(flat[t.sample_index(flat.numel(), t.LOGIT_SAMPLE)].numpy())
        for v in f_ref.values():
            flat = v.reshape(-1)
            feat_samples.append(flat[t.sample_index(flat.numel(), t.FEATURE_SAMPLE)].numpy())
            feat_absmax.append(float(flat.abs().max()))
        meta["shim"].append(rec)
    arrays["shim_logits"] = np.concatenate(logit_samples)
    arrays["shim_features"] = np.concatenate(feat_samples)
    arrays["shim_feature_absmax"] = np.array(feat_absmax)

    from oracle import vit as ovit

    ov = {"input_size": (64, 64), "nb_blocks": 1, "interpolate_input": True}
    ref = rr.create_model("vit_tiny_patch16_224", **ov)
    ref.assign(params.random_params(ovit.param_shapes(t._engine_cfg("vit_tiny_patch16_224", ov)), seed=4,
                                    dtype=torch.float64))
    arrays["interpolate_logits"] = ref(params.test_images(1, 96, 128).double()).numpy()
    rr.set_floatx("float32")

    ref = rr.create_model("vit_tiny_patch16_224")
    ref.assign(params.random_params(ovit.param_shapes(t._engine_cfg("vit_tiny_patch16_224", {})), seed=3))
    arrays["full_size_logits"] = ref(params.test_images(1, 224, 224)).numpy()

    for name, ov in t.INITIAL_VALUE_CASES:   # variables whose initial value is one constant
        wd = rr.create_model(name, **ov).weights_dict()
        meta["initial_values"][name] = {k: float(np.min(v)) for k, v in wd.items() if np.min(v) == np.max(v)}

    meta["registry"] = {fam: rr.list_models(module=fam) for fam in rr.FAMILIES}
    with rr._reference_modules():
        mods = rr._import_reference()
        meta["configs"] = {n: dataclasses.asdict(mods["registry"].model_config(n)) for n in t.REGISTRY_CONFIGS}

    pre = []
    for name in t.PREPROCESSING_MODELS:
        ref = rr.create_preprocessing(name, dtype="float32")
        with rr._reference_modules():
            a = ref(t.preprocessing_image())
        pre.append(a.numpy() if hasattr(a, "numpy") else np.asarray(a))
    arrays["preprocessing"] = np.stack(pre)

    for name, ov in t.TRANSFER_MODELS:
        for change in t.TRANSFER_CHANGES:
            omod = importlib.import_module(f"oracle.{t.FAMILY_OF[name]}")
            w = params.random_params(omod.param_shapes(t._engine_cfg(name, ov)), seed=17)
            src_ref = rr.create_model(name, **ov)
            src_ref.assign(w, ignore_missing=t.IGNORE)
            dst_ref = rr.create_model(name, **ov, **change)
            before = dst_ref.weights_dict()
            rr.transfer_weights(src_ref, dst_ref)
            after = dst_ref.weights_dict()
            rec = {"offset": count(tr_values), "changed": [], "unchanged": []}
            for k, v in after.items():
                if any(p in k for p in t.IGNORE):
                    continue
                if np.array_equal(v, before[k]):
                    rec["unchanged"].append(k)
                    continue
                flat = np.asarray(v, dtype=np.float32).reshape(-1)
                tr_values.append(flat[t.sample_index(flat.size, t.TRANSFER_SAMPLE)])
                rec["changed"].append([k, list(np.shape(v))])
            meta["transfer"][t.transfer_case_id(name, change)] = rec
    arrays["transfer_values"] = np.concatenate(tr_values)

    for arch in t.STATE_DICT_ARCHS:
        name, ov, sd = t.state_dict_case(arch)
        ref = rr.create_model(name, **ov)
        rr.load_pytorch_weights(ref, {k: v.clone() for k, v in sd.items()})
        meta["state_dict"][arch] = t.params_digest({k: v for k, v in ref.weights_dict().items()
                                                    if not any(p in k for p in t.IGNORE)})

    arrays["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **arrays)
    print(OUT, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
