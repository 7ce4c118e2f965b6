"""``create_model`` / ``create_preprocessing`` / ``transfer_weights``.

Behavioural contract: reference tfimm/models/factory.py:18-305 (see SURVEY.md 8b):
  * unknown model -> ``RuntimeError`` (create_model) / ``ValueError`` (create_preprocessing)
  * kwargs that name config fields override a deep copy of the registered config, other kwargs
    only log a warning; ``name=`` is also forwarded to the model object
  * ``in_channels`` / ``nb_classes`` override the config; when weights were loaded first they are
    carried over by ``transfer_weights`` (first conv adapted, classifier kept only if the class
    count is unchanged, per-weight ``cfg.transform_weights`` hooks applied)
  * ``create_preprocessing`` returns ``f(img) = (img / 255 - mean) / std`` with mean / std tiled
    cyclically to ``in_channels``.

Engine-specific keyword arguments (not config fields): ``precision`` ("bf16" default | "fp32" |
"tf32", see ``tfimm.models.model.PRECISIONS``), ``device`` and ``seed``.  Weight sources available offline: a ``model_path`` / cache entry that is
a ``.npz`` / ``.pt`` flat dict in reference names, or a PyTorch ``state_dict`` converted by
``tfimm.utils.timm`` rules.  Downloading needs a network and raises ``NotImplementedError``.
"""
import logging
import os
import re
from copy import deepcopy
from typing import Callable, List, Optional

import numpy as np
import torch

from ..utils import cached_model_path
from .registry import is_model, model_class, model_config

_ENGINE_KWARGS = ("precision", "device", "seed")


def _load_flat_dict(path: str):
    if os.path.isdir(path):
        for cand in ("weights.npz", "weights.pt"):
            if os.path.exists(os.path.join(path, cand)):
                path = os.path.join(path, cand)
                break
        else:
            raise NotImplementedError(
                f"{path}: Keras SavedModel directories cannot be read without TensorFlow; "
                "save weights with `tfimm.models.save_weights(model, path)` (npz) instead."
            )
    if path.endswith(".npz"):
        with np.load(path) as data:
            return {k: data[k] for k in data.files}
    return torch.load(path, map_location="cpu")


def save_weights(model, path: str):
    """Writes the model's weights as a flat npz in reference names/layouts plus nothing else."""
    np.savez(path, **model.weights_dict())


def create_model(
    model_name: str,
    pretrained: bool = False,
    model_path: str = "",
    *,
    in_channels: Optional[int] = None,
    nb_classes: Optional[int] = None,
    **kwargs,
):
    if not is_model(model_name):
        raise RuntimeError(f"Unknown model {model_name}.")
    cls = model_class(model_name)
    registered_cfg = model_config(model_name)
    engine_kwargs = {k: kwargs.pop(k) for k in _ENGINE_KWARGS if k in kwargs}

    loaded_model = None
    if model_path or pretrained:
        source = model_path or cached_model_path(model_name)
        if not source:
            if registered_cfg.url.startswith(("[timm]", "[pytorch]", "[hf-pytorch]")):
                raise NotImplementedError(
                    f"No cached weights for {model_name} and downloading ({registered_cfg.url}) needs a "
                    "network. Convert a local PyTorch state_dict with "
                    "`tfimm.utils.timm.load_pytorch_weights_in_model` or pass `model_path=`."
                )
            raise NotImplementedError(
                "Model not found in cache. Download of weights only implemented for PyTorch models."
            )
        loaded_model = cls(deepcopy(registered_cfg), **engine_kwargs)
        loaded_model.load_weights_dict(_load_flat_dict(source), strict=True)

    cfg = deepcopy(registered_cfg)
    for key, value in kwargs.items():
        if hasattr(cfg, key):
            setattr(cfg, key, value)
        else:
            logging.warning(f"Config for {model_name} does not have field `{key}`. Ignoring field.")
    if in_channels is not None:
        setattr(cfg, "in_channels", in_channels)
    if nb_classes is not None:
        setattr(cfg, "nb_classes", nb_classes)

    model_kwargs = dict(engine_kwargs)
    if "name" in kwargs:
        model_kwargs["name"] = kwargs["name"]

    if loaded_model is not None and loaded_model.cfg == cfg:
        return loaded_model
    model = cls(cfg, **model_kwargs)
    if loaded_model is not None:
        transfer_weights(loaded_model, model)
    return model


def create_preprocessing(model_name: str, *, in_channels: Optional[int] = None, dtype=None) -> Callable:
    if not is_model(model_name):
        raise ValueError(f"Unknown model: {model_name}.")
    cfg = model_config(model_name)
    n = in_channels or cfg.in_channels

    def _cycled(values):
        reps = n // len(values) + 1
        return np.asarray((list(values) * reps)[:n], dtype=np.float32)

    mean, std = _cycled(cfg.mean), _cycled(cfg.std)

    def _preprocess(img):
        """Works on single images and batches; numpy in -> numpy out, torch in -> torch out
        (CUDA tensors stay on the device)."""
        if isinstance(img, torch.Tensor):
            tdtype = dtype if isinstance(dtype, torch.dtype) else getattr(torch, str(dtype or "float32"))
            m = torch.as_tensor(mean, device=img.device, dtype=tdtype)
            s = torch.as_tensor(std, device=img.device, dtype=tdtype)
            return (img.to(tdtype) / 255.0 - m) / s
        ndtype = np.dtype(dtype or "float32")
        out = np.asarray(img).astype(ndtype) / ndtype.type(255.0)
        return (out - mean.astype(ndtype)) / std.astype(ndtype)

    # Raw statistics, so callers can hand uint8 pixels to the fused patchify/stem kernels.
    _preprocess.mean = mean
    _preprocess.std = std
    return _preprocess


def _layer_of(key: str) -> str:
    """``"remove/fc/kernel"`` -> ``"fc"`` (layer name as used by cfg.first_conv / cfg.classifier)."""
    key = ("/" + key).replace("/remove/", "/")[1:]
    return key.rsplit("/", 1)[0] if "/" in key else key


def _adapt_first_conv(weight: torch.Tensor, in_channels: int) -> torch.Tensor:
    if weight.dim() != 4:
        return weight  # biases do not depend on the input channels
    src = weight.shape[2]
    if in_channels == src:
        return weight
    if in_channels == 1:
        return weight.sum(dim=2, keepdim=True)  # summed, not averaged: keeps weight statistics
    reps = in_channels // src + 1
    tiled = weight.repeat(1, 1, reps, 1)[:, :, :in_channels, :]
    return tiled * (src / in_channels)


def transfer_weights(src_model, dst_model, weights_to_ignore: Optional[List[str]] = None):
    """Name-matched copy ``src_model -> dst_model`` (in place), with the reference's special cases
    (tfimm/models/factory.py:174-250, 282-305)."""
    ignore = list(weights_to_ignore or [])
    ignore += list(getattr(dst_model, "keys_to_ignore_on_load_missing", []))
    first_conv = getattr(dst_model.cfg, "first_conv", None)
    if hasattr(src_model.cfg, "nb_classes") and hasattr(dst_model.cfg, "nb_classes"):
        keep_classifier = src_model.cfg.nb_classes == dst_model.cfg.nb_classes
    else:
        keep_classifier = True
    classifier = getattr(dst_model.cfg, "classifier", [])
    classifier = [classifier] if isinstance(classifier, str) else list(classifier)
    transforms = getattr(src_model.cfg, "transform_weights", dict())

    update = {}
    for key in dst_model.params:
        layer = _layer_of(key)
        if any(re.search(pat, key) is not None for pat in ignore):
            continue
        if layer in classifier:
            if keep_classifier:
                update[key] = src_model.params[key]
        elif layer == first_conv:
            update[key] = _adapt_first_conv(src_model.params[key], dst_model.cfg.in_channels)
        elif key in transforms:
            update[key] = transforms[key](src_model, src_model.params[key], dst_model.cfg)
        else:
            update[key] = src_model.params[key]
    dst_model.load_weights_dict(update, strict=False)
