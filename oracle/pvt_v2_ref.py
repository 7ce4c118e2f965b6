"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference ``tfimm/architectures/pvt_v2.py`` on the TensorFlow shim, as
``oracle/ref_runner.py`` does for the classifiers and ``oracle/pvt_ref.py`` for PVT v1.  The module runs on the shim as
it is."""
import dataclasses

from . import ref_runner as rr


def _import_pvt_v2():
    import importlib

    mods = rr._import_reference()
    mods["pvt_v2"] = importlib.import_module("tfimm.architectures.pvt_v2")
    return mods


def create_model(model_name: str, **kwargs) -> rr.ReferenceModel:
    with rr._reference_modules():
        mods = _import_pvt_v2()
        model = mods["factory"].create_model(model_name, **kwargs)
    return rr.ReferenceModel(model, mods)


def register_test_model(name, **cfg_fields):
    """Registers ``name`` in the reference's registry: a ``PyramidVisionTransformerV2Config`` with ``cfg_fields``."""
    with rr._reference_modules():
        mods = _import_pvt_v2()
        pm = mods["pvt_v2"]

        def entry():
            return pm.PyramidVisionTransformerV2, pm.PyramidVisionTransformerV2Config(name=name, **cfg_fields)

        entry.__name__ = name
        mods["registry"].register_model(entry)


def model_config(model_name: str):
    with rr._reference_modules():
        mods = _import_pvt_v2()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "pvt_v2"):
    with rr._reference_modules():
        mods = _import_pvt_v2()
        return mods["registry"].list_models(module=module)
