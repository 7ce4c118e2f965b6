"""PVT (Pyramid Vision Transformer, v1) forward path as a chain of sm_90a kernels.

Registered on import (``import tfimm.architectures.pvt``, module name ``pvt``); ``import tfimm`` alone does not import
it.

What the reference computes (tfimm/architectures/pvt.py), per stage j:
  embed   PatchEmbeddings: Conv2D(embed_dim[j], kernel = stride = patch_size[j], VALID) + bias, then LayerNorm eps 1e-5;
          the last stage prepends cls_token; then + pos_embed{j+1} (1, ntok + gh * gw, D), resized bicubically on the
          grid with interpolate_input (the class row kept as it is)                                (pvt.py:366-384)
  blocks  nb_blocks[j] pre-norm blocks (LayerNorm eps 1e-6): spatial-reduction attention -- q = Dense(x); when
          sr_ratio[j] > 1 the keys and values come from x (B, gh, gw, D) through a VALID sr x sr / sr Conv2D + bias and
          a LayerNorm eps 1e-5, else from x itself; kv = Dense(2D) read as (B, N', 2, H, dh); softmax(q k^T / sqrt(dh)) v;
          proj -- then the GELU MLP of width D mlp_ratio[j]                                           (pvt.py:111-247)
  between stages the stream is reshaped to (B, gh, gw, D) for the next patch embedding
  head    LayerNorm eps 1e-6 of the whole stream (features_all), token 0 (features), Dense head   (pvt.py:396-409)

How it runs here (fp32 residual stream (B * T, D) in every precision):
  embed   im2col "valid" (uint8 pixels at stage 0: the preprocessing fused in; after that the stream viewed
          (B, gh, gw, D)) -> GEMM + bias (fp32) -> pvt_ops.pvt_embed_norm: LayerNorm, + the plan-time position table of
          the grid, and the class row at the last stage
  block   layernorm -> q GEMM; sr > 1: im2col(h, sr, sr, "valid") -> GEMM + bias (fp32) -> layernorm (1e-5); -> kv GEMM
          -> pvt_ops.sr_attention -> proj GEMM (+ residual, in place) -> layernorm -> MLP (ops.mlp_fused where
          ops.mlp_fused_supported in bf16, else fc1 + GELU GEMM and fc2 GEMM, + residual)
  head    layernorm of row 0 (of every row when features are asked for) -> head GEMM
Attention: bf16 -> the tensor-core kernel, fp32 and tf32 -> the fp32 kernel (head dim 64 only).
"""
from collections import OrderedDict
from dataclasses import dataclass
from functools import partial
from typing import List, Tuple

import torch

from ..backend import ops, pvt_ops
from ..layers.resize import interpolate_pos_embeddings
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["PyramidVisionTransformer", "PyramidVisionTransformerConfig", "param_specs"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}
_EMBED_EPS = 1e-5   # the patch embeddings' and the spatial reduction's "layer_norm"


@dataclass
class PyramidVisionTransformerConfig(ModelConfig):
    """Hyper-parameters (same fields and defaults as the reference's ``PyramidVisionTransformerConfig``,
    pvt.py:33-108)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_size: Tuple = (4, 2, 2, 2)
    embed_dim: Tuple = (64, 128, 256, 512)
    nb_blocks: Tuple = (3, 4, 6, 3)
    nb_heads: Tuple = (1, 2, 5, 8)
    mlp_ratio: Tuple = (8.0, 8.0, 4.0, 4.0)
    sr_ratio: Tuple = (8, 4, 2, 1)
    qkv_bias: bool = True
    drop_rate: float = 0.0
    attn_drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    norm_layer: str = "layer_norm_eps_1e-6"
    act_layer: str = "gelu"
    interpolate_input: bool = False
    crop_pct: float = 0.9
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "patch_embed1/proj"
    classifier: str = "head"

    @property
    def nb_tokens(self) -> Tuple:
        """Special tokens per stage: the class token joins at the last stage."""
        return (0,) * (len(self.nb_blocks) - 1) + (1,)

    @property
    def grid_size(self) -> Tuple:
        return grids(self.input_size, self.patch_size)

    @property
    def nb_patches(self) -> Tuple:
        return tuple(h * w for h, w in self.grid_size)

    @property
    def transform_weights(self):
        return {f"pos_embed{j + 1}": partial(PyramidVisionTransformer.transform_pos_embed, stage=j)
                for j in range(len(self.nb_blocks))}


def grids(size, patch_size):
    """The grid of every stage: each VALID patch embedding floors, dropping the remainder rows and columns."""
    out = []
    h, w = size
    for p in patch_size:
        h, w = h // p, w // p
        out.append((h, w))
    return tuple(out)


def param_specs(c: PyramidVisionTransformerConfig) -> "OrderedDict[str, ParamSpec]":
    """The reference's variables (names, shapes, initial values) in the order of its ``weights``: pos_embed1 .. and
    cls_token first (zeros, added by the model's build()), then the layers in the order Keras tracks them -- the four
    patch embeddings, then the blocks (in each, the attention's q, kv, proj, then sr and its norm, as its __init__
    assigns them), the norm and the head -- with Keras' default initialisers (glorot_uniform kernels, zero biases,
    LayerNorm 1 / 0)."""
    s = OrderedDict()

    def dense(prefix, shape, bias=True):
        s[f"{prefix}/kernel"] = ParamSpec(shape, "glorot_uniform")
        if bias:
            s[f"{prefix}/bias"] = ParamSpec((shape[-1],), "zeros")

    def norm(prefix, n):
        s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
        s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

    for j, D in enumerate(c.embed_dim):
        s[f"pos_embed{j + 1}"] = ParamSpec((1, c.nb_patches[j] + c.nb_tokens[j], D), "zeros")
    s["cls_token"] = ParamSpec((1, 1, c.embed_dim[-1]), "zeros")
    cin = c.in_channels
    for j, D in enumerate(c.embed_dim):
        p = c.patch_size[j]
        dense(f"patch_embed{j + 1}/proj", (p, p, cin, D))
        norm(f"patch_embed{j + 1}/norm", D)
        cin = D
    for j, (D, depth) in enumerate(zip(c.embed_dim, c.nb_blocks)):
        sr, hid = c.sr_ratio[j], int(D * c.mlp_ratio[j])
        for k in range(depth):
            b = f"block{j + 1}/{k}"
            norm(f"{b}/norm1", D)
            dense(f"{b}/attn/q", (D, D), bias=c.qkv_bias)
            dense(f"{b}/attn/kv", (D, 2 * D), bias=c.qkv_bias)
            dense(f"{b}/attn/proj", (D, D))
            if sr > 1:
                dense(f"{b}/attn/sr", (sr, sr, D, D))
                norm(f"{b}/attn/norm", D)
            norm(f"{b}/norm2", D)
            dense(f"{b}/mlp/fc1", (D, hid))
            dense(f"{b}/mlp/fc2", (hid, D))
    norm("norm", c.embed_dim[-1])
    if c.nb_classes > 0:
        dense("head", (c.embed_dim[-1], c.nb_classes))
    return s


class PyramidVisionTransformer(Model):
    cfg_class = PyramidVisionTransformerConfig
    accepts_uint8 = True

    def __init__(self, cfg: PyramidVisionTransformerConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = PyramidVisionTransformerConfig(**cfg)
        if cfg.norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        fields = (cfg.patch_size, cfg.embed_dim, cfg.nb_blocks, cfg.nb_heads, cfg.mlp_ratio, cfg.sr_ratio)
        if len({len(f) for f in fields}) != 1:
            raise ValueError("patch_size, embed_dim, nb_blocks, nb_heads, mlp_ratio and sr_ratio must have one entry "
                             "per stage")
        for j, (D, H) in enumerate(zip(cfg.embed_dim, cfg.nb_heads)):
            if D % H or D // H != pvt_ops.HEAD_DIM:
                raise ValueError(f"stage {j}: head_dim {D}/{H} must be {pvt_ops.HEAD_DIM}")
            if int(D * cfg.mlp_ratio[j]) % 8:
                raise ValueError(f"stage {j}: the kernels need the MLP width to be a multiple of 8 "
                                 f"(mlp_ratio {cfg.mlp_ratio[j]})")
        if cfg.sr_ratio[-1] != 1:
            raise ValueError(f"sr_ratio[-1] must be 1: the last stage carries the class token (got {cfg.sr_ratio})")
        self.nb_features = cfg.embed_dim[-1]
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        return param_specs(self.cfg)

    def transform_pos_embed(self, src_weights, target_cfg: PyramidVisionTransformerConfig, stage: int):
        """pos_embed{stage + 1} resized bicubically on its grid to ``target_cfg``'s (pvt.py:350-358)."""
        return interpolate_pos_embeddings(self.params[f"pos_embed{stage + 1}"], self.cfg.grid_size[stage],
                                          target_cfg.grid_size[stage], self.cfg.nb_tokens[stage])

    @property
    def feature_names(self) -> List[str]:
        names, k = [], 0
        for j, depth in enumerate(self.cfg.nb_blocks):
            names += [f"patch_embedding_{j}", f"pos_embedding_{j}"]
            names += [f"block_{k + i}" for i in range(depth)]
            k += depth
            names.append(f"stage_{j}")
        return names + ["features_all", "features", "logits"]

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        P = {"eps": _LN_EPS[c.norm_layer], "stages": [], "pos": {}}
        for j, depth in enumerate(c.nb_blocks):
            pe = f"patch_embed{j + 1}"
            st = {"pe_w": self._dense_weight(f"{pe}/proj/kernel"), "pe_b": self._vec(f"{pe}/proj/bias"),
                  "pe_n": (self._vec(f"{pe}/norm/gamma"), self._vec(f"{pe}/norm/beta")), "blocks": []}
            for k in range(depth):
                b = f"block{j + 1}/{k}"
                bias = (lambda key: self._vec(key)) if c.qkv_bias else (lambda key: None)
                blk = dict(
                    n1=(self._vec(f"{b}/norm1/gamma"), self._vec(f"{b}/norm1/beta")),
                    q_w=self._dense_weight(f"{b}/attn/q/kernel"), q_b=bias(f"{b}/attn/q/bias"),
                    kv_w=self._dense_weight(f"{b}/attn/kv/kernel"), kv_b=bias(f"{b}/attn/kv/bias"),
                    proj_w=self._dense_weight(f"{b}/attn/proj/kernel"), proj_b=self._vec(f"{b}/attn/proj/bias"),
                    n2=(self._vec(f"{b}/norm2/gamma"), self._vec(f"{b}/norm2/beta")),
                    fc1_w=self._dense_weight(f"{b}/mlp/fc1/kernel"), fc1_b=self._vec(f"{b}/mlp/fc1/bias"),
                    fc2_w=self._dense_weight(f"{b}/mlp/fc2/kernel"), fc2_b=self._vec(f"{b}/mlp/fc2/bias"),
                )
                if c.sr_ratio[j] > 1:
                    blk["sr_w"], blk["sr_b"] = self._dense_weight(f"{b}/attn/sr/kernel"), self._vec(f"{b}/attn/sr/bias")
                    blk["srn"] = (self._vec(f"{b}/attn/norm/gamma"), self._vec(f"{b}/attn/norm/beta"))
                st["blocks"].append(blk)
            P["stages"].append(st)
        P["cls"] = self._vec("cls_token")
        P["norm"] = (self._vec("norm/gamma"), self._vec("norm/beta"))
        if c.nb_classes > 0:
            P["head_w"], P["head_b"] = self._dense_weight("head/kernel"), self._vec("head/bias")
        return P

    def _pos_table(self, P, j, grid):
        """(ntok + gh * gw, D) fp32: pos_embed{j+1} on ``grid`` (built once per stage and grid size)."""
        if (j, grid) not in P["pos"]:
            c = self.cfg
            pos = interpolate_pos_embeddings(self.params[f"pos_embed{j + 1}"].float(), c.grid_size[j], grid,
                                             c.nb_tokens[j])
            P["pos"][(j, grid)] = pos[0].contiguous()
        return P["pos"][(j, grid)]

    def _check_input(self, H, W):
        """The stage grids of an (H, W) input; ValueError, before any launch, for inputs the model cannot run."""
        c = self.cfg
        if not c.interpolate_input and (H, W) != tuple(c.input_size):
            raise ValueError(f"Input size {(H, W)} does not match the model's {tuple(c.input_size)}; "
                             "create the model with interpolate_input=True to allow this.")
        gs = grids((H, W), c.patch_size)
        for j, ((gh, gw), sr) in enumerate(zip(gs, c.sr_ratio)):
            if gh < max(1, sr) or gw < max(1, sr):
                raise ValueError(f"Input size {(H, W)}: stage {j}'s grid {gh} x {gw} is smaller than its patch "
                                 f"or spatial-reduction ratio {sr}, which leaves no tokens or no keys")
        return gs

    # ------------------------------------------------------------------ forward
    def _block(self, blk, xs, B, T, gh, gw, D, Hh, sr):
        c = self.cfg
        eps, adt = self._plan["eps"], self.act_dtype
        dh = D // Hh
        h = ops.layernorm(xs, *blk["n1"], eps, adt)
        q = ops.gemm(h, blk["q_w"], bias=blk["q_b"])
        if sr > 1:
            cols, rh, rw = ops.im2col(h.view(B, gh, gw, D), sr, sr, "valid", adt)
            r = ops.gemm(cols, blk["sr_w"], bias=blk["sr_b"], out_dtype=torch.float32)
            src, Nk = ops.layernorm(r, *blk["srn"], _EMBED_EPS, adt), rh * rw
        else:
            src, Nk = h, T
        kv = ops.gemm(src, blk["kv_w"], bias=blk["kv_b"])
        a = pvt_ops.sr_attention(q, kv, B, T, Nk, Hh, dh, dh ** -0.5)
        ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], residual=xs, out=xs)
        h = ops.layernorm(xs, *blk["n2"], eps, adt)
        if adt == torch.bfloat16 and ops.mlp_fused_supported(D, blk["fc1_w"].shape[0]):
            # one kernel: the (M, hidden) activations stay on the SM (csrc/mlp_sm90.cu)
            ops.mlp_fused(h, blk["fc1_w"], blk["fc1_b"], blk["fc2_w"], blk["fc2_b"], c.act_layer, residual=xs, out=xs)
        else:
            hid = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
            ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], residual=xs, out=xs)

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        x = self._input(x)
        B = x.shape[0]
        gs = self._check_input(x.shape[1], x.shape[2])
        P = self._ensure_plan()
        features = OrderedDict()
        img, k = x, 0
        last = len(c.nb_blocks) - 1
        for j, st in enumerate(P["stages"]):
            D, p, ntok = c.embed_dim[j], c.patch_size[j], c.nb_tokens[j]
            pre = self._pixel_stats(x.device) if img.dtype == torch.uint8 else None
            cols, gh, gw = ops.im2col(img, p, p, "valid", self.act_dtype, pre=pre)
            assert (gh, gw) == gs[j]
            tok = ops.gemm(cols, st["pe_w"], bias=st["pe_b"], out_dtype=torch.float32)
            if return_features:
                features[f"patch_embedding_{j}"] = ops.layernorm(tok, *st["pe_n"], _EMBED_EPS,
                                                                 torch.float32).view(B, gh * gw, D)
            xs = pvt_ops.pvt_embed_norm(tok, *st["pe_n"], self._pos_table(P, j, (gh, gw)),
                                        P["cls"] if ntok else None, B, gh * gw, _EMBED_EPS)
            T = ntok + gh * gw
            if return_features:
                features[f"pos_embedding_{j}"] = xs.view(B, T, D).clone()
            for blk in st["blocks"]:
                self._block(blk, xs, B, T, gh, gw, D, c.nb_heads[j], c.sr_ratio[j])
                if return_features:
                    features[f"block_{k}"] = xs.view(B, T, D).clone()
                k += 1
            img = xs.view(B, gh, gw, D) if j < last else xs.view(B, T, D)
            if return_features:
                features[f"stage_{j}"] = img
        x3 = img
        D = c.embed_dim[-1]
        if return_features:
            normed = ops.layernorm(xs, *P["norm"], P["eps"], torch.float32).view(B, -1, D)
            out = normed[:, 0]
            features["features_all"] = normed
            features["features"] = out
            return out, features
        return ops.layernorm(x3[:, 0], *P["norm"], P["eps"], torch.float32)

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        features = OrderedDict()
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        if c.nb_classes > 0:
            P = self._ensure_plan()
            x = ops.gemm(ops.cast(x.contiguous(), self.act_dtype), P["head_w"], bias=P["head_b"],
                         out_dtype=torch.float32)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "pvt", PyramidVisionTransformer, PyramidVisionTransformerConfig)
