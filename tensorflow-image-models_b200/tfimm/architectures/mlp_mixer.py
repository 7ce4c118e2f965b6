"""MLP-Mixer, gMixer, ResMLP and gMLP forward path as a chain of sm_90a kernels.

Registered on import (``import tfimm.architectures.mlp_mixer``, module name ``mlp_mixer``); ``import tfimm`` alone does
not import it.

What the reference computes (tfimm/architectures/mlp_mixer.py): PatchEmbeddings (k = s = patch) -> nb_blocks blocks ->
norm over all tokens -> mean over tokens -> head Dense.  Blocks (mlp_mixer.py:115-223, layers/transformers.py):
  mixer_block           x += T(mlp_tokens(T(norm1(x))));  x += mlp_channels(norm2(x))        (T: swap tokens/channels)
  mixer_block, glu_mlp  the same with GluMLP (fc1 -> split -> value * act(gate) -> fc2) in both MLPs (gMixer)
  res_block             x += ls1 * T(linear_tokens(T(affine1(x))));  x += ls2 * mlp_channels(affine2(x))
  spatial_gating_block  x += fc2(u * T(proj(T(LN_1e-5(v)))))  with u | v = act(fc1(norm(x)))   (gMLP)

How it runs here (bf16: fp32 residual stream, bf16 GEMM operands, fp32 accumulation):
  patchify -> stem GEMM (fp32 out: the residual stream)
  token mixing: one wgmma GEMM per Dense (mixer_ops.token_gemm) that reads the activation where it is stored as an
                MN-major operand -- no transpose copies; bias per output row, GLU on row pairs, ls1 as gamma[c], the
                gMLP gate's u as an elementwise multiplier and the residual in its epilogue
  channel MLPs: ops.gemm (ls2 as gamma), or mixer_ops.gemm_glu for gMixer (the full-width hidden never exists)
  norms:        ops.layernorm, mixer_ops.affine
  head:         final norm over all tokens (fp32) -> global_avg_pool -> head GEMM
``precision="fp32"`` runs the same graph on the CUDA-core kernels.  tf32 is refused: TF32 wgmma takes no transpose
immediates, so the token GEMM's MN-major operand has no TF32 form.
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Tuple

import torch

from ..backend import mixer_ops, ops
from ..models import Model, ModelConfig, ParamSpec
from ._zoo import register_zoo

__all__ = ["MLPMixer", "MLPMixerConfig", "param_specs"]

_NORMS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6, "affine": None}
_BLOCKS = ("mixer_block", "res_block", "spatial_gating_block")
_MLPS = ("mlp", "glu_mlp", "gated_mlp")


@dataclass
class MLPMixerConfig(ModelConfig):
    """Hyper-parameters (same fields and defaults as the reference's ``MLPMixerConfig``, mlp_mixer.py:47-80)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_size: int = 16
    embed_dim: int = 512
    nb_blocks: int = 16
    mlp_ratio: Tuple[float, float] = (0.5, 4.0)
    block_layer: str = "mixer_block"
    mlp_layer: str = "mlp"
    drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    norm_layer: str = "layer_norm_eps_1e-6"
    act_layer: str = "gelu"
    init_values: float = 1e-4
    nlhb: bool = False
    stem_norm: bool = False
    crop_pct: float = 0.875
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = (0.5, 0.5, 0.5)
    std: Tuple[float, float, float] = (0.5, 0.5, 0.5)
    first_conv: str = "stem/proj"
    classifier: str = "head"

    @property
    def grid_size(self) -> Tuple[int, int]:
        return (self.input_size[0] // self.patch_size, self.input_size[1] // self.patch_size)

    @property
    def nb_patches(self) -> int:
        return self.grid_size[0] * self.grid_size[1]

    @property
    def hidden_dims(self) -> Tuple[int, int]:
        """(token MLP hidden, channel MLP hidden) as the reference computes them (mlp_mixer.py:95, 154, 209)."""
        if self.block_layer == "mixer_block":
            t, c = (int(x * self.embed_dim) for x in self.mlp_ratio)
            return t, c
        return 0, int(self.embed_dim * self.mlp_ratio[1])


def param_specs(c: MLPMixerConfig) -> "OrderedDict[str, ParamSpec]":
    """The reference's variables (names, shapes, initial values) in creation order."""
    D, N = c.embed_dim, c.nb_patches
    Ht, Hc = c.hidden_dims
    s = OrderedDict()

    def dense(prefix, n_in, n_out, kinit="glorot_uniform", binit="zeros"):
        s[f"{prefix}/kernel"] = ParamSpec((n_in, n_out), kinit)
        s[f"{prefix}/bias"] = ParamSpec((n_out,), binit)

    def norm(prefix, n, kind=c.norm_layer):
        if kind == "affine":
            s[f"{prefix}/alpha"] = ParamSpec((n,), "ones")
            s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")
        else:
            s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
            s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

    def mlp(prefix, hidden, dim):
        dense(f"{prefix}/fc1", dim, hidden)
        out_in = hidden // 2 if c.mlp_layer in ("glu_mlp", "gated_mlp") else hidden
        if c.mlp_layer == "gated_mlp":
            norm(f"{prefix}/gate/norm", hidden // 2, "layer_norm")
            dense(f"{prefix}/gate/proj", N, N, kinit="normal:1e-6", binit="ones")
        dense(f"{prefix}/fc2", out_in, dim)

    s["stem/proj/kernel"] = ParamSpec((c.patch_size, c.patch_size, c.in_channels, D), "glorot_uniform")
    s["stem/proj/bias"] = ParamSpec((D,), "zeros")
    if c.stem_norm:
        norm("stem/norm", D)
    for j in range(c.nb_blocks):
        p = f"blocks/{j}"
        if c.block_layer == "mixer_block":
            norm(f"{p}/norm1", D)
            mlp(f"{p}/mlp_tokens", Ht, N)
            norm(f"{p}/norm2", D)
            mlp(f"{p}/mlp_channels", Hc, D)
        elif c.block_layer == "res_block":
            # ResBlock.build creates the layer scales before its sublayers are built on the first call
            s[f"{p}/ls1"] = ParamSpec((D,), f"const:{c.init_values}")
            s[f"{p}/ls2"] = ParamSpec((D,), f"const:{c.init_values}")
            norm(f"{p}/norm1", D)
            dense(f"{p}/linear_tokens", N, N)
            norm(f"{p}/norm2", D)
            mlp(f"{p}/mlp_channels", Hc, D)
        else:
            norm(f"{p}/norm", D)
            mlp(f"{p}/mlp_channels", Hc, D)
    norm("norm", D)
    if c.nb_classes > 0:
        dense("head", D, c.nb_classes)
    return s


class MLPMixer(Model):
    cfg_class = MLPMixerConfig
    accepts_uint8 = True

    def __init__(self, cfg: MLPMixerConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = MLPMixerConfig(**cfg)
        if kwargs.get("precision", "bf16") == "tf32":
            raise ValueError("MLP-Mixer models run in precision 'bf16' or 'fp32'; tf32 is not implemented for them "
                             "(TF32 wgmma has no transposed operand form for the token-mixing GEMM).")
        if cfg.norm_layer not in _NORMS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        if cfg.block_layer not in _BLOCKS:
            raise ValueError(f"Unknown block layer: {cfg.block_layer}")
        if cfg.mlp_layer not in _MLPS:
            raise ValueError(f"Unknown MLP layer: {cfg.mlp_layer}")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        Ht, Hc = cfg.hidden_dims
        glu = cfg.mlp_layer == "glu_mlp"
        ch_in = Hc // 2 if cfg.mlp_layer in ("glu_mlp", "gated_mlp") else Hc
        if cfg.embed_dim % 8 or ch_in % 8 or (glu and (Hc % 2 or Ht % 2)):
            raise ValueError(f"the kernels need embed_dim and the channel MLP's fc2 width to be multiples of 8 "
                             f"(got {cfg.embed_dim}, {ch_in})")
        self.nb_features = cfg.embed_dim
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        return param_specs(self.cfg)

    def _build(self):
        """The ParamSpec initialisers, then GluMLP's fc1 as the reference initialises it (GatedKernelInitializer /
        GatedBiasInitializer, layers/transformers.py:265-313): the value half of the kernel glorot-uniform over its own
        shape, the gate half normal with std 1e-6; the bias zeros, then ones for the gate half."""
        super()._build()
        if self.cfg.mlp_layer != "glu_mlp" or self.device.type == "meta":
            return
        import math

        gen = torch.Generator().manual_seed(self._seed + 1)
        for key in [k for k in self.params if k.endswith("/fc1/kernel")]:
            k = self.params[key]
            n_in, half = k.shape[0], k.shape[1] // 2
            limit = math.sqrt(6.0 / (n_in + half))
            value = (torch.rand((n_in, half), generator=gen) * 2 - 1) * limit
            gate = torch.randn((n_in, half), generator=gen) * 1e-6
            self.params[key] = torch.cat((value, gate), 1).to(self.device)
            b = torch.zeros(2 * half)
            b[half:] = 1.0
            self.params[key[:-len("kernel")] + "bias"] = b.to(self.device)

    @property
    def feature_names(self) -> List[str]:
        return ["stem"] + [f"block_{j}" for j in range(self.cfg.nb_blocks)] + ["features_all", "features", "logits"]

    # ------------------------------------------------------------------ engine plan
    def _norm_plan(self, prefix, kind):
        if kind == "affine":
            return ("affine", self._vec(f"{prefix}/alpha"), self._vec(f"{prefix}/beta"), None)
        return ("ln", self._vec(f"{prefix}/gamma"), self._vec(f"{prefix}/beta"), _NORMS[kind])

    def _glu_fc1(self, prefix, rows):
        """GLU fc1 in the interleaved order of mixer_ops.glu_interleave (rows=True: token GLU / fp32 channel GLU)."""
        w = self.params[f"{prefix}/kernel"]
        w = w.reshape(-1, w.shape[-1]).t().float()
        K = w.shape[1]
        w = torch.nn.functional.pad(w, (0, (-K) % 8))
        wi, bi = mixer_ops.glu_interleave(w, self._vec(f"{prefix}/bias"), rows)
        return self._gemm_operand(wi), bi

    def _compile(self):
        c = self.cfg
        Ht, Hc = c.hidden_dims
        glu = c.mlp_layer == "glu_mlp"
        P = {"blocks": []}
        P["stem_w"] = self._dense_weight("stem/proj/kernel")
        P["stem_b"] = self._vec("stem/proj/bias")
        P["stem_norm"] = self._norm_plan("stem/norm", c.norm_layer) if c.stem_norm else None
        for j in range(c.nb_blocks):
            p = f"blocks/{j}"
            b = {}
            if c.block_layer == "mixer_block":
                b["n1"], b["n2"] = self._norm_plan(f"{p}/norm1", c.norm_layer), self._norm_plan(f"{p}/norm2", c.norm_layer)
                if glu:
                    b["t1_w"], b["t1_b"] = self._glu_fc1(f"{p}/mlp_tokens/fc1", True)
                else:
                    b["t1_w"], b["t1_b"] = self._dense_weight(f"{p}/mlp_tokens/fc1/kernel"), self._vec(f"{p}/mlp_tokens/fc1/bias")
                b["t2_w"], b["t2_b"] = self._dense_weight(f"{p}/mlp_tokens/fc2/kernel"), self._vec(f"{p}/mlp_tokens/fc2/bias")
            elif c.block_layer == "res_block":
                b["n1"], b["n2"] = self._norm_plan(f"{p}/norm1", c.norm_layer), self._norm_plan(f"{p}/norm2", c.norm_layer)
                b["lt_w"], b["lt_b"] = self._dense_weight(f"{p}/linear_tokens/kernel"), self._vec(f"{p}/linear_tokens/bias")
                b["ls1"], b["ls2"] = self._vec(f"{p}/ls1"), self._vec(f"{p}/ls2")
            else:
                b["n1"] = self._norm_plan(f"{p}/norm", c.norm_layer)
                # the gate's own norm is norm_layer_factory("layer_norm"), eps 1e-5 (layers/transformers.py:364)
                b["gn"] = self._norm_plan(f"{p}/mlp_channels/gate/norm", "layer_norm")
                b["gp_w"], b["gp_b"] = (self._dense_weight(f"{p}/mlp_channels/gate/proj/kernel"),
                                        self._vec(f"{p}/mlp_channels/gate/proj/bias"))
            q = f"{p}/mlp_channels"
            if glu:
                b["c1_w"], b["c1_b"] = self._glu_fc1(f"{q}/fc1", self.precision != "bf16")
            else:
                b["c1_w"], b["c1_b"] = self._dense_weight(f"{q}/fc1/kernel"), self._vec(f"{q}/fc1/bias")
            b["c2_w"], b["c2_b"] = self._dense_weight(f"{q}/fc2/kernel"), self._vec(f"{q}/fc2/bias")
            P["blocks"].append(b)
        P["norm"] = self._norm_plan("norm", c.norm_layer)
        if c.nb_classes > 0:
            P["head_w"], P["head_b"] = self._dense_weight("head/kernel"), self._vec("head/bias")
        return P

    # ------------------------------------------------------------------ forward
    @staticmethod
    def _apply_norm(x, prm, out_dtype):
        kind, a, b, eps = prm
        if kind == "affine":
            return mixer_ops.affine(x, a, b, out_dtype)
        return ops.layernorm(x, a, b, eps, out_dtype)

    def _block(self, b, xs, B, N):
        """One block, in place on the fp32 (B*N, D) residual stream xs."""
        c = self.cfg
        D, adt, act = c.embed_dim, self.act_dtype, c.act_layer
        Ht, Hc = c.hidden_dims
        xs3 = xs.view(B, N, D)
        if c.block_layer == "mixer_block":
            glu = c.mlp_layer == "glu_mlp"
            h = self._apply_norm(xs, b["n1"], adt)
            t = mixer_ops.token_gemm(b["t1_w"][:, :N], h.view(B, N, D), bias=b["t1_b"], act=act, glu=glu,
                                     m_out=Ht // 2 if glu else Ht)
            mixer_ops.token_gemm(b["t2_w"][:, :t.shape[1]], t, bias=b["t2_b"], residual=xs3, out=xs3)
            h = self._apply_norm(xs, b["n2"], adt)
            if glu:
                hid = mixer_ops.gemm_glu(h, b["c1_w"], b["c1_b"], Hc // 2, act)
            else:
                hid = ops.gemm(h, b["c1_w"], bias=b["c1_b"], act=act)
            ops.gemm(hid, b["c2_w"], bias=b["c2_b"], residual=xs, out=xs)
        elif c.block_layer == "res_block":
            a = self._apply_norm(xs, b["n1"], adt)
            mixer_ops.token_gemm(b["lt_w"][:, :N], a.view(B, N, D), bias=b["lt_b"], gamma=b["ls1"], residual=xs3, out=xs3)
            a = self._apply_norm(xs, b["n2"], adt)
            hid = ops.gemm(a, b["c1_w"], bias=b["c1_b"], act=act)
            ops.gemm(hid, b["c2_w"], bias=b["c2_b"], gamma=b["ls2"], residual=xs, out=xs)
        else:
            half = Hc // 2
            h = self._apply_norm(xs, b["n1"], adt)
            z = ops.gemm(h, b["c1_w"], bias=b["c1_b"], act=act)          # u | v, (B*N, Hc)
            v = self._apply_norm(z[:, half:], b["gn"], adt)
            g = mixer_ops.token_gemm(b["gp_w"][:, :N], v.view(B, N, half), bias=b["gp_b"],
                                     mul=z.view(B, N, z.stride(0))[:, :, :half])
            ops.gemm(g.view(B * N, half), b["c2_w"], bias=b["c2_b"], residual=xs, out=xs)

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        x = self._input(x)
        B, H, W, _ = x.shape
        if (H, W) != tuple(c.input_size):
            raise ValueError(f"Input size {(H, W)} does not match the model's {tuple(c.input_size)}: the token count "
                             "of an MLP-Mixer is fixed by its input size.")
        P = self._ensure_plan()
        N, D = c.nb_patches, c.embed_dim
        features = OrderedDict()
        patches = self._patchify(x, c.patch_size)
        xs = ops.gemm(patches, P["stem_w"], bias=P["stem_b"], out_dtype=torch.float32)
        if P["stem_norm"] is not None:
            xs = self._apply_norm(xs, P["stem_norm"], torch.float32)
        if xs.stride(0) != D:
            xs = xs.contiguous()
        if return_features:
            features["stem"] = xs.view(B, N, D).clone()
        for j, b in enumerate(P["blocks"]):
            self._block(b, xs, B, N)
            if return_features:
                features[f"block_{j}"] = xs.view(B, N, D).clone()
        full = self._apply_norm(xs, P["norm"], torch.float32).view(B, N, D)
        out = ops.global_avg_pool(full)
        if return_features:
            features["features_all"] = full
            features["features"] = out
            return out, features
        return out

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        features = {}
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        if c.nb_classes > 0:
            P = self._ensure_plan()
            x = ops.gemm(ops.cast(x, self.act_dtype), P["head_w"], bias=P["head_b"], out_dtype=torch.float32)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "mlp_mixer", MLPMixer, MLPMixerConfig)
