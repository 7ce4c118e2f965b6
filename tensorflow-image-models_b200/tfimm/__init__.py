"""tfimm_b200: a H100-native (sm_90a) inference engine behind tfimm's public API.

Drop-in for the image-classifier forward path of martinsbruveris/tensorflow-image-models
(reference ``tfimm/__init__.py:1-12``): ``create_model``, ``create_preprocessing``,
``list_models`` and the ``ModelConfig`` registry keep their names, arguments and error
behaviour; the returned models run hand-written CUDA kernels instead of Keras layers.
"""
from . import architectures  # noqa: F401  (runs every model registration)
from .models.factory import create_model, create_preprocessing  # noqa: F401
from .models.registry import list_models  # noqa: F401
from .utils import (  # noqa: F401
    cached_model_path,
    clear_model_cache,
    get_dir,
    list_cached_models,
    set_dir,
    set_model_cache,
)
from . import parallel, serving  # noqa: F401
from .version import __version__  # noqa: F401
