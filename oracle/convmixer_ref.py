"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference ``tfimm/architectures/convmixer.py`` on the TensorFlow
shim, as ``oracle/ref_runner.py`` does for the classifiers and ``oracle/mixer_ref.py`` for MLP-Mixer.  The module runs
on the shim as it is."""
import dataclasses

from . import ref_runner as rr


def _import_convmixer():
    import importlib

    mods = rr._import_reference()
    mods["convmixer"] = importlib.import_module("tfimm.architectures.convmixer")
    return mods


def create_model(model_name: str, **kwargs) -> rr.ReferenceModel:
    with rr._reference_modules():
        mods = _import_convmixer()
        model = mods["factory"].create_model(model_name, **kwargs)
    return rr.ReferenceModel(model, mods)


def register_test_model(name, **cfg_fields):
    """Registers ``name`` in the reference's registry: a ``ConvMixerConfig`` with ``cfg_fields``."""
    with rr._reference_modules():
        mods = _import_convmixer()
        pf = mods["convmixer"]

        def entry():
            return pf.ConvMixer, pf.ConvMixerConfig(name=name, **cfg_fields)

        entry.__name__ = name
        mods["registry"].register_model(entry)


def model_config(model_name: str):
    with rr._reference_modules():
        mods = _import_convmixer()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "convmixer"):
    with rr._reference_modules():
        mods = _import_convmixer()
        return mods["registry"].list_models(module=module)
