"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference ``tfimm/architectures/poolformer.py`` on the TensorFlow
shim, as ``oracle/ref_runner.py`` does for the classifiers and ``oracle/mixer_ref.py`` for MLP-Mixer.  The module runs
on the shim as it is."""
import dataclasses

from . import ref_runner as rr


def _import_poolformer():
    import importlib

    mods = rr._import_reference()
    mods["poolformer"] = importlib.import_module("tfimm.architectures.poolformer")
    return mods


def create_model(model_name: str, **kwargs) -> rr.ReferenceModel:
    with rr._reference_modules():
        mods = _import_poolformer()
        model = mods["factory"].create_model(model_name, **kwargs)
    return rr.ReferenceModel(model, mods)


def register_test_model(name, **cfg_fields):
    """Registers ``name`` in the reference's registry: a ``PoolFormerConfig`` with ``cfg_fields``."""
    with rr._reference_modules():
        mods = _import_poolformer()
        pf = mods["poolformer"]

        def entry():
            return pf.PoolFormer, pf.PoolFormerConfig(name=name, **cfg_fields)

        entry.__name__ = name
        mods["registry"].register_model(entry)


def model_config(model_name: str):
    with rr._reference_modules():
        mods = _import_poolformer()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "poolformer"):
    with rr._reference_modules():
        mods = _import_poolformer()
        return mods["registry"].list_models(module=module)
