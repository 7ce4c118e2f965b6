"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference ``tfimm/architectures/cait.py`` on the TensorFlow shim, as
``oracle/ref_runner.py`` does for the classifiers and ``oracle/poolformer_ref.py`` for PoolFormer.  The module runs on
the shim as it is."""
import dataclasses

from . import ref_runner as rr


def _import_cait():
    import importlib

    mods = rr._import_reference()
    mods["cait"] = importlib.import_module("tfimm.architectures.cait")
    return mods


def create_model(model_name: str, **kwargs) -> rr.ReferenceModel:
    with rr._reference_modules():
        mods = _import_cait()
        model = mods["factory"].create_model(model_name, **kwargs)
    return rr.ReferenceModel(model, mods)


def register_test_model(name, **cfg_fields):
    """Registers ``name`` in the reference's registry: a ``CaiTConfig`` with ``cfg_fields``."""
    with rr._reference_modules():
        mods = _import_cait()
        pm = mods["cait"]

        def entry():
            return pm.CaiT, pm.CaiTConfig(name=name, **cfg_fields)

        entry.__name__ = name
        mods["registry"].register_model(entry)


def model_config(model_name: str):
    with rr._reference_modules():
        mods = _import_cait()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "cait"):
    with rr._reference_modules():
        mods = _import_cait()
        return mods["registry"].list_models(module=module)
