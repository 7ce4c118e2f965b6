"""Base class of every engine model: owns the weights, mirrors the reference's model-object contract.

Contract kept from the reference (SURVEY.md 8b; e.g. tfimm/architectures/vit.py:298-478):
  * constructor takes the config object (or a dict of its fields, the ``keras_serializable``
    convention, tfimm/models/serialization.py:50-70) and an optional ``name``
  * ``model(x, training=False, return_features=False)`` -> logits, or ``(logits, features)``
  * ``forward_features``, ``cfg``, ``name``, ``dummy_inputs``, ``feature_names``
  * ``model.weights``: objects with ``.name`` (``"<model name>/<path>:0"``), ``.shape``,
    ``.numpy()``; names and layouts are the reference's TF variable names and layouts, so a
    flat ``{path: array}`` dict converted by the reference's own rules loads unchanged.

What is different by design: weights live in HBM as torch CUDA tensors; the forward pass is a
sequence of hand-written sm_90a kernels (tfimm.backend.ops); inference only.
"""
import functools
import math
from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from ..backend import lib as _lib


@dataclass(frozen=True)
class ParamSpec:
    shape: Tuple[int, ...]
    init: str = "zeros"  # zeros | ones | glorot_uniform | const:<v> | normal:<std> | uniform:<a>
    trainable: bool = True


class Weight:
    """Read/write view of one model parameter under its reference (TF) variable name."""

    def __init__(self, model: "Model", key: str):
        self._model = model
        self.key = key

    @property
    def name(self) -> str:
        return f"{self._model.name}/{self.key}:0"

    @property
    def shape(self):
        return tuple(self._model.params[self.key].shape)

    @property
    def trainable(self) -> bool:
        return self._model.param_specs()[self.key].trainable

    def numpy(self) -> np.ndarray:
        return self._model.params[self.key].detach().float().cpu().numpy()

    def assign(self, value):
        self._model.load_weights_dict({self.key: value}, strict=False)

    def __repr__(self):
        return f"<Weight {self.name} shape={self.shape}>"


def _init_tensor(spec: ParamSpec, gen: torch.Generator) -> torch.Tensor:
    shape = tuple(spec.shape)
    kind, _, arg = spec.init.partition(":")
    if kind == "zeros":
        return torch.zeros(shape)
    if kind == "ones":
        return torch.ones(shape)
    if kind == "const":
        return torch.full(shape, float(arg))
    if kind == "normal":
        return torch.randn(shape, generator=gen) * float(arg)
    if kind == "uniform":
        a = float(arg)
        return (torch.rand(shape, generator=gen) * 2 - 1) * a
    if kind == "glorot_uniform":
        # Keras default for Dense / Conv kernels: receptive field * in, receptive field * out
        rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
        fan_in = shape[-2] * rf if len(shape) >= 2 else shape[0]
        fan_out = shape[-1] * rf if len(shape) >= 2 else shape[0]
        limit = math.sqrt(6.0 / (fan_in + fan_out))
        return (torch.rand(shape, generator=gen) * 2 - 1) * limit
    raise ValueError(f"Unknown initializer {spec.init}")


# bf16: bf16 GEMM operands / activations, fp32 accumulation and residual stream (the fast default).
# fp32: fp32 everywhere on CUDA cores (parity with the reference's arithmetic).
# tf32: fp32 storage, every contraction (GEMMs, k x k convolutions, ViT self-attention) on the TF32 tensor cores, operands
#       rounded to TF32 (round to nearest, ties away) -- what TensorFlow runs for fp32 models on Ampere and newer GPUs.
PRECISIONS = ("bf16", "fp32", "tf32")


def _in_precision_mode(forward):
    """Wraps a public forward entry point (``call``, ``forward_features``): while it runs, the launchers' TF32 switch
    (``lib.tf32_mode``) is on exactly when the model is a tf32 model -- reset afterwards, also when it raises, and
    independent of the caller's context."""

    @functools.wraps(forward)
    def wrapped(self, *args, **kwargs):
        token = _lib.tf32_mode.set(self.precision == "tf32")
        try:
            return forward(self, *args, **kwargs)
        finally:
            _lib.tf32_mode.reset(token)

    return wrapped


class Model:
    cfg_class = None
    # regexes of weights created at build time that need not be present when loading
    keys_to_ignore_on_load_missing: List[str] = []

    def __init_subclass__(cls, **kwargs):
        # every public forward entry point of an architecture -- ``model(x)``, ``model.call``,
        # ``model.forward_features``, and through them ``cuda_graph`` and the serving / parallel paths -- runs its
        # launches in the model's precision mode
        super().__init_subclass__(**kwargs)
        for name in ("call", "forward_features"):
            if name in cls.__dict__:
                setattr(cls, name, _in_precision_mode(cls.__dict__[name]))

    def __init__(self, cfg, *args, name: Optional[str] = None, precision: str = "bf16",
                 device=None, seed: int = 0, **kwargs):
        if isinstance(cfg, dict):
            cfg = self.cfg_class(**cfg)
        if self.cfg_class is not None and not isinstance(cfg, self.cfg_class):
            raise ValueError("Must pass either `cfg` (ModelConfig) or `cfg` (dict)")
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {', '.join(map(repr, PRECISIONS))}, got {precision!r}")
        self.cfg = cfg
        self.name = name or cfg.name
        self.precision = precision
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        self.device = torch.device(device)
        self.params: "OrderedDict[str, torch.Tensor]" = OrderedDict()
        self._specs = None
        self._plan = None  # engine-layout tensors derived from params (see _compile)
        self._plan_version = 0  # bumped whenever the weights / device change (captured CUDA graphs check it)
        self._seed = seed
        self._build()

    # ------------------------------------------------------------------ parameters
    def param_specs(self) -> "OrderedDict[str, ParamSpec]":
        if self._specs is None:
            self._specs = self._param_specs()
        return self._specs

    def _param_specs(self) -> "OrderedDict[str, ParamSpec]":
        raise NotImplementedError

    def _build(self):
        gen = torch.Generator().manual_seed(self._seed)
        for key, spec in self.param_specs().items():
            if self.device.type == "meta":  # shapes only (used to enumerate variables cheaply)
                self.params[key] = torch.empty(tuple(spec.shape), device="meta")
            else:
                self.params[key] = _init_tensor(spec, gen).to(self.device)
        self._plan = None
        self._plan_version += 1

    @property
    def weights(self) -> List[Weight]:
        return [Weight(self, k) for k in self.params]

    @property
    def trainable_weights(self) -> List[Weight]:
        return [w for w in self.weights if w.trainable]

    def count_params(self) -> int:
        return int(sum(p.numel() for p in self.params.values()))

    def weights_dict(self) -> Dict[str, np.ndarray]:
        """Flat ``{path: fp32 array}`` in reference (TF) names and layouts."""
        return {k: v.detach().float().cpu().numpy() for k, v in self.params.items()}

    def load_weights_dict(self, weights: Dict[str, object], strict: bool = True):
        """Loads reference-layout weights.  ``strict``: every parameter of the model must be given
        (except ``keys_to_ignore_on_load_missing``) and no unknown key may be present."""
        import re

        missing = []
        for key, cur in self.params.items():
            if key not in weights:
                if strict and not any(re.search(p, key) for p in self.keys_to_ignore_on_load_missing):
                    missing.append(key)
                continue
            val = weights[key]
            val = val.detach().cpu() if isinstance(val, torch.Tensor) else torch.from_numpy(np.asarray(val))
            val = val.to(torch.float32)
            if tuple(val.shape) != tuple(cur.shape):
                raise ValueError(f"Shape mismatch for {key}: model {tuple(cur.shape)}, given {tuple(val.shape)}")
            self.params[key] = val.contiguous().to(self.device)
        if strict:
            unknown = [k for k in weights if k not in self.params]
            if missing or unknown:
                raise AttributeError(f"load_weights_dict: missing={missing[:5]} unknown={unknown[:5]}")
        self._plan = None
        self._plan_version += 1

    def to(self, device):
        self.device = torch.device(device)
        for k in self.params:
            self.params[k] = self.params[k].to(self.device)
        self._plan = None
        self._plan_version += 1
        return self

    # ------------------------------------------------------------------ engine helpers
    @property
    def act_dtype(self) -> torch.dtype:
        return torch.bfloat16 if self.precision == "bf16" else torch.float32

    def _gemm_operand(self, w: torch.Tensor) -> torch.Tensor:
        """A GEMM / convolution weight matrix as the kernels take it: in the activation dtype and, for tf32 models,
        rounded to TF32 once here (the TF32 kernels round only their activation operand)."""
        w = w.to(self.act_dtype)
        if self.precision == "tf32":
            w = _lib.round_tf32(w)
        return w.contiguous()

    def _dense_weight(self, key: str, pad_k_to: int = 8) -> torch.Tensor:
        """TF Dense/Conv kernel ``(..., in, out)`` -> engine layout ``W[out][K]`` (K contiguous,
        K = prod(leading dims), zero-padded to a multiple of ``pad_k_to``), a GEMM operand (``_gemm_operand``)."""
        w = self.params[key]
        out = w.shape[-1]
        w2 = w.reshape(-1, out).t().contiguous()  # (out, K)
        K = w2.shape[1]
        Kpad = (K + pad_k_to - 1) // pad_k_to * pad_k_to
        if Kpad != K:
            w2 = torch.nn.functional.pad(w2, (0, Kpad - K))
        return self._gemm_operand(w2)

    def _vec(self, key: str) -> torch.Tensor:
        return self.params[key].reshape(-1).float().contiguous()

    def _compile(self):
        raise NotImplementedError

    def _ensure_plan(self):
        if self.device.type != "cuda":
            raise _lib.KernelLibraryError(
                "tfimm_b200 models only run on a CUDA device (sm_90a); there is no CPU fallback. "
                "The model was created on device '%s'." % self.device
            )
        if self._plan is None:
            _lib.load()
            self._plan = self._compile()
        return self._plan

    def _input(self, x) -> torch.Tensor:
        if not isinstance(x, torch.Tensor):
            x = torch.from_numpy(np.ascontiguousarray(x))
        if x.dim() == 3:
            x = x[None]
        if x.dtype == torch.uint8:
            # raw pixels: create_preprocessing's (x/255 - mean)/std is fused into the first kernel
            # (reference tfimm/models/factory.py:153-169); see _patchify.
            if not self.accepts_uint8:
                raise TypeError(f"{type(self).__name__} takes preprocessed float images "
                                "(fused uint8 preprocessing is implemented for the patchify and conv-stem families).")
            return x.to(self.device, non_blocking=True).contiguous()
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.float()
        if self.precision != "bf16" and x.dtype != torch.float32:
            x = x.float()
        return x.to(self.device, non_blocking=True).contiguous()

    accepts_uint8 = False

    def _patchify(self, x, patch_size):
        """Non-overlapping patch gather; uint8 input gets the model's preprocessing fused in."""
        from ..backend import ops

        if x.dtype != torch.uint8:
            return ops.patchify(x, patch_size, self.act_dtype)
        mean, inv_std, scale = self._pixel_stats(x.device)
        return ops.patchify(x, patch_size, self.act_dtype, mean=mean, inv_std=inv_std, scale=scale)

    def _pixel_stats(self, device):
        """(mean, 1 / std, 1 / 255) of create_preprocessing (reference tfimm/models/factory.py:153-169) as device
        tensors, for the kernels that take raw uint8 pixels (patchify, the im2col of the convolutional stems)."""
        if getattr(self, "_pre_stats", None) is None or self._pre_stats[0].device != device:
            n = self.cfg.in_channels

            def cyc(v):
                return torch.tensor((list(v) * (n // len(v) + 1))[:n], dtype=torch.float32, device=device)

            self._pre_stats = (cyc(self.cfg.mean), 1.0 / cyc(self.cfg.std))
        return self._pre_stats[0], self._pre_stats[1], 1.0 / 255.0

    # ------------------------------------------------------------------ public forward API
    @property
    def dummy_inputs(self) -> torch.Tensor:
        return torch.zeros((1, *self.cfg.input_size, self.cfg.in_channels), device=self.device)

    @property
    def feature_names(self) -> List[str]:
        _, features = self(self.dummy_inputs, return_features=True)
        return list(features.keys())

    def forward_features(self, x, training=False, return_features=False):
        raise NotImplementedError

    def call(self, x, training=False, return_features=False):
        raise NotImplementedError

    def __call__(self, x, training=False, return_features=False):
        if training:
            raise NotImplementedError("tfimm_b200 is an inference engine: training=True is not supported.")
        return self.call(x, training=False, return_features=return_features)

    def cuda_graph(self, batch_size: int, input_size=None, dtype=torch.float32):
        """Captures one forward pass (fixed batch / input size) into a CUDA graph and returns a callable
        ``f(x) -> logits`` that copies ``x`` into the graph's static input and replays it: the ~90-400 kernel
        launches of a forward become one graph launch, which removes the host-side launch gaps (this is the
        H100-native replacement for the reference's ``tf.function(jit_compile=True)`` wrapper,
        tfimm/utils/profile.py:88-90).  The returned tensor is overwritten by the next call."""
        from ..backend import ops

        self._ensure_plan()
        h, w = input_size or self.cfg.input_size
        static_in = torch.zeros((batch_size, h, w, self.cfg.in_channels), device=self.device, dtype=dtype)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):  # warm-up: function attributes, allocator pools, tensor-map driver entry point
                self(static_in)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        before = ops.launch_count
        with torch.cuda.graph(graph):
            static_out = self(static_in)
        launches = ops.launch_count - before

        version = self._plan_version

        def run(x):
            if x.dtype != static_in.dtype or tuple(x.shape) != tuple(static_in.shape):
                # copy_ would silently CAST: uint8 pixels replayed through a float capture skip the fused
                # (x/255 - mean)/std of the eager uint8 path.  Capture with dtype=torch.uint8 for raw pixels.
                raise TypeError(f"cuda_graph captured for {tuple(static_in.shape)} {static_in.dtype}, "
                                f"got {tuple(x.shape)} {x.dtype}")
            if self._plan_version != version:
                raise RuntimeError("the model's weights / device changed after cuda_graph() captured them; "
                                   "capture a new graph")
            static_in.copy_(x, non_blocking=True)
            graph.replay()
            ops.launch_count += launches
            return static_out

        run.graph, run.static_input, run.static_output, run.launches = graph, static_in, static_out, launches
        return run

    def get_config(self):
        import dataclasses

        return dataclasses.asdict(self.cfg)

    @classmethod
    def from_config(cls, config):
        return cls(config)
