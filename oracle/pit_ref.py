"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference ``tfimm/architectures/pit.py`` on the TensorFlow shim, as
``oracle/ref_runner.py`` does for the classifiers and ``oracle/poolformer_ref.py`` for PoolFormer.  The module runs on
the shim as it is."""
import dataclasses

from . import ref_runner as rr


def _import_pit():
    import importlib

    mods = rr._import_reference()
    mods["pit"] = importlib.import_module("tfimm.architectures.pit")
    return mods


def create_model(model_name: str, **kwargs) -> rr.ReferenceModel:
    with rr._reference_modules():
        mods = _import_pit()
        model = mods["factory"].create_model(model_name, **kwargs)
    return rr.ReferenceModel(model, mods)


def register_test_model(name, **cfg_fields):
    """Registers ``name`` in the reference's registry: a ``PoolingVisionTransformerConfig`` with ``cfg_fields``."""
    with rr._reference_modules():
        mods = _import_pit()
        pm = mods["pit"]

        def entry():
            return pm.PoolingVisionTransformer, pm.PoolingVisionTransformerConfig(name=name, **cfg_fields)

        entry.__name__ = name
        mods["registry"].register_model(entry)


def model_config(model_name: str):
    with rr._reference_modules():
        mods = _import_pit()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "pit"):
    with rr._reference_modules():
        mods = _import_pit()
        return mods["registry"].list_models(module=module)
