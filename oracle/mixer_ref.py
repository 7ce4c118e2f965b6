"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference ``tfimm/architectures/mlp_mixer.py`` (MLP-Mixer, gMixer,
ResMLP, gMLP) on the TensorFlow shim, as ``oracle/ref_runner.py`` does for the classifiers.

The reference's package ``__init__`` is bypassed (``ref_runner._import_reference``); the imported module is the
reference's file.  One incompatibility with the shim is fixed at run time, here rather than in ``oracle/tf_shim`` so that
the classifier pins keep running on exactly the shim they were recorded with: ``GatedBiasInitializer`` /
``GatedKernelInitializer`` (tfimm/layers/transformers.py:265-313) compute ``shape[:-1] + [...]``, which needs the list
shape TensorFlow passes; the shim passes a tuple, so their ``__call__`` gets the shape as a list.
"""
import dataclasses

from . import ref_runner as rr


def _import_mixer():
    import importlib

    mods = rr._import_reference()
    tr = importlib.import_module("tfimm.layers.transformers")
    for cls in (tr.GatedBiasInitializer, tr.GatedKernelInitializer):
        if not getattr(cls, "_list_shape", False):
            call = cls.__call__

            def list_call(self, shape, *args, _call=call, **kwargs):
                return _call(self, list(shape), *args, **kwargs)

            cls.__call__, cls._list_shape = list_call, True
    mods["mlp_mixer"] = importlib.import_module("tfimm.architectures.mlp_mixer")
    return mods


def create_model(model_name: str, **kwargs) -> rr.ReferenceModel:
    with rr._reference_modules():
        mods = _import_mixer()
        model = mods["factory"].create_model(model_name, **kwargs)
    return rr.ReferenceModel(model, mods)


def register_test_model(name, **cfg_fields):
    """Registers ``name`` in the reference's registry: an ``MLPMixerConfig`` with ``cfg_fields``."""
    with rr._reference_modules():
        mods = _import_mixer()
        mm = mods["mlp_mixer"]

        def entry():
            return mm.MLPMixer, mm.MLPMixerConfig(name=name, **cfg_fields)

        entry.__name__ = name
        mods["registry"].register_model(entry)


def model_config(model_name: str):
    with rr._reference_modules():
        mods = _import_mixer()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "mlp_mixer"):
    with rr._reference_modules():
        mods = _import_mixer()
        return mods["registry"].list_models(module=module)
