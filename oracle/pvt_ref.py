"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference ``tfimm/architectures/pvt.py`` on the TensorFlow shim, as
``oracle/ref_runner.py`` does for the classifiers and ``oracle/pit_ref.py`` for PiT.  The module runs on the shim as
it is."""
import dataclasses

from . import ref_runner as rr


def _import_pvt():
    import importlib

    mods = rr._import_reference()
    mods["pvt"] = importlib.import_module("tfimm.architectures.pvt")
    return mods


def create_model(model_name: str, **kwargs) -> rr.ReferenceModel:
    with rr._reference_modules():
        mods = _import_pvt()
        model = mods["factory"].create_model(model_name, **kwargs)
    return rr.ReferenceModel(model, mods)


def register_test_model(name, **cfg_fields):
    """Registers ``name`` in the reference's registry: a ``PyramidVisionTransformerConfig`` with ``cfg_fields``."""
    with rr._reference_modules():
        mods = _import_pvt()
        pm = mods["pvt"]

        def entry():
            return pm.PyramidVisionTransformer, pm.PyramidVisionTransformerConfig(name=name, **cfg_fields)

        entry.__name__ = name
        mods["registry"].register_model(entry)


def model_config(model_name: str):
    with rr._reference_modules():
        mods = _import_pvt()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "pvt"):
    with rr._reference_modules():
        mods = _import_pvt()
        return mods["registry"].list_models(module=module)
