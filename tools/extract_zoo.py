"""Dumps the reference's model registrations (names + config hyper-parameters) as JSON data.

The reference cannot be imported normally here (TensorFlow is not installed), but its config
dataclasses and ``@register_model`` entry points are plain Python.  This script imports
``/root/reference/tfimm`` against a stub ``tensorflow`` module (every attribute is an inert
class), reads the populated registry and writes, for the in-scope families,

    tensorflow-image-models_b200/tfimm/architectures/zoo/<family>.json
        {"<model name>": {<config field>: <value>, ...}, ...}

Only data leaves the reference: names and hyper-parameters.  Run from the repo root:

    python tools/extract_zoo.py
"""
import dataclasses
import json
import sys
import types
from pathlib import Path

REFERENCE = Path("/root/reference")
OUT = Path(__file__).resolve().parent.parent / "tensorflow-image-models_b200" / "tfimm" / "architectures" / "zoo"
FAMILIES = ["vit", "swin", "convnext", "efficientnet", "resnet", "mlp_mixer", "poolformer", "pit", "convmixer", "pvt",
            "pvt_v2", "cait"]


class _Meta(type):
    def __getattr__(cls, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        return cls

    def __call__(cls, *args, **kwargs):
        # decorator use: @stub(...) / @stub -> identity; otherwise an inert instance
        if cls is _Stub and len(args) == 1 and not kwargs and (isinstance(args[0], type) or callable(args[0])):
            return args[0]
        return super().__call__(*args, **kwargs)


class _Stub(metaclass=_Meta):
    def __init__(self, *args, **kwargs):
        pass

    def __call__(self, *args, **kwargs):
        if len(args) == 1 and not kwargs and (isinstance(args[0], type) or callable(args[0])):
            return args[0]
        return self

    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        return _Stub


class _StubModule(types.ModuleType):
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        return _Stub


def _install_stubs():
    for name in [
        "tensorflow", "tensorflow.python", "tensorflow.python.keras", "tensorflow.python.keras.backend",
        "tensorflow.keras", "tensorflow.keras.layers", "tensorflow_addons", "timm", "timm.models",
        "timm.models.layers", "timm.models.helpers", "timm.models.registry", "timm.data",
        "timm.models.layers.helpers", "timm.models.vision_transformer", "timm.layers",
    ]:
        sys.modules[name] = _StubModule(name)


def _jsonable(v):
    if isinstance(v, (tuple, list)):
        return [_jsonable(x) for x in v]
    if isinstance(v, dict):
        return {k: _jsonable(x) for k, x in v.items()}
    if isinstance(v, (str, int, float, bool)) or v is None:
        return v
    raise TypeError(f"non-data config value {v!r}")


def main():
    _install_stubs()
    sys.path.insert(0, str(REFERENCE))
    # Only the in-scope architecture modules are imported (the package __init__ would pull in
    # every family plus torch-based oracles).
    import importlib

    pkg = types.ModuleType("tfimm")
    pkg.__path__ = [str(REFERENCE / "tfimm")]
    sys.modules["tfimm"] = pkg
    arch = types.ModuleType("tfimm.architectures")
    arch.__path__ = [str(REFERENCE / "tfimm" / "architectures")]
    sys.modules["tfimm.architectures"] = arch
    registry = importlib.import_module("tfimm.models.registry")
    OUT.mkdir(parents=True, exist_ok=True)
    for fam in FAMILIES:
        importlib.import_module(f"tfimm.architectures.{fam}")
        names = sorted(registry._module_to_models[fam])
        table = {}
        for name in names:
            cfg = registry.model_config(name)
            fields = {f.name: _jsonable(getattr(cfg, f.name)) for f in dataclasses.fields(cfg)}
            fields["__class__"] = registry.model_class(name).__name__
            fields["__config__"] = type(cfg).__name__
            table[name] = fields
        (OUT / f"{fam}.json").write_text(json.dumps(table, indent=1, sort_keys=True) + "\n")
        print(fam, len(names))


if __name__ == "__main__":
    main()
