"""PiT (pooling-based vision transformer) forward path as a chain of sm_90a kernels.

Registered on import (``import tfimm.architectures.pit``, module name ``pit``); ``import tfimm`` alone does not import
it.

What the reference computes (tfimm/architectures/pit.py, reusing vit.ViTBlock):
  stem    Conv2D(embed_dim[0], kernel patch_size, stride, VALID): overlapping patches (16 / 8, or 14 / 7 for pit_b),
          + pos_embed (stored NCHW (1, D0, gh, gw); resized bicubically on the grid with interpolate_input), then
          prepend cls_token (1, nb_tokens, D0): the special tokens get no position embedding     (pit.py:331-349)
  stage j nb_blocks[j] ViT blocks: pre-norm LayerNorm eps 1e-6, qkv with bias, GELU MLP, no layer scale
  pool    between stages (ConvHeadPooling, pit.py:172-188): the grid rows, ZeroPadding2D(1), a 3 x 3 / 2 Conv2D with
          groups = C and 2C filters (output channel o reads input o // 2) + bias; the token rows through Dense(2C);
          concat([tokens, grid])
  head    features_all = the stream before the norm; norm on the token rows; token 0, or both token rows when
          distilled; head (and head_dist, stacked on axis 1)                                   (pit.py:358-395)

How it runs here (fp32 residual stream (B * T, C) in every precision):
  stem    im2col "valid" (uint8 pixels: the preprocessing fused in) -> GEMM + bias -> ops.assemble_tokens with a
          plan-time position table whose first nb_tokens rows are zero, cls / dist = rows 0 / 1 of cls_token
  block   layernorm -> qkv GEMM -> pit_ops.attention -> proj GEMM (+ residual, in place) -> layernorm -> MLP
          (ops.mlp_fused where ops.mlp_fused_supported in bf16, else fc1 + GELU GEMM and fc2 GEMM, + residual)
  pool    pit_ops.pit_pool writes the new stream's grid rows (and, in bf16, the token rows as the bf16 operand);
          the token Dense is one GEMM per token row, written through a row-strided view into the new stream
  head    layernorm of each token row -> head GEMM(s)
Attention: bf16 -> pit_ops.pit_attention_bf16 (head dims 32 / 48 / 64, any T); fp32 -> the fp32 SIMT kernel; tf32 ->
the TF32 kernel at head dim 64, the fp32 SIMT kernel at 32 and 48.
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Tuple, Union

import torch

from ..backend import ops, pit_ops
from ..layers.resize import tf_bicubic_resize
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["PoolingVisionTransformer", "PoolingVisionTransformerConfig", "param_specs"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}


@dataclass
class PoolingVisionTransformerConfig(ModelConfig):
    """Hyper-parameters (same fields and defaults as the reference's ``PoolingVisionTransformerConfig``,
    pit.py:51-144)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_size: int = 16
    stride: int = 8
    embed_dim: Tuple = (64, 128, 256)
    nb_blocks: Tuple = (2, 6, 4)
    nb_heads: Tuple = (2, 4, 8)
    mlp_ratio: float = 4.0
    distilled: bool = False
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
    first_conv: str = "patch_embed/conv"
    classifier: Union[str, Tuple[str, str]] = "head"

    @property
    def nb_tokens(self) -> int:
        return 2 if self.distilled else 1

    @property
    def grid_size(self) -> Tuple[int, int]:
        return ((self.input_size[0] - self.patch_size) // self.stride + 1,
                (self.input_size[1] - self.patch_size) // self.stride + 1)

    @property
    def transform_weights(self):
        return {"pos_embed": PoolingVisionTransformer.transform_pos_embed}


def param_specs(c: PoolingVisionTransformerConfig) -> "OrderedDict[str, ParamSpec]":
    """The reference's variables (names, shapes, initial values) in creation order: pos_embed and cls_token first
    (TruncatedNormal(0.02), created by the model's build()), then the layers in call order with Keras' default
    initialisers (glorot_uniform kernels, zero biases, LayerNorm 1 / 0)."""
    s = OrderedDict()
    gh, gw = c.grid_size

    def dense(prefix, shape, bias=True):
        s[f"{prefix}/kernel"] = ParamSpec(shape, "glorot_uniform")
        if bias:
            s[f"{prefix}/bias"] = ParamSpec((shape[-1],), "zeros")

    def norm(prefix, n):
        s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
        s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

    s["pos_embed"] = ParamSpec((1, c.embed_dim[0], gh, gw), "normal:0.02")
    s["cls_token"] = ParamSpec((1, c.nb_tokens, c.embed_dim[0]), "normal:0.02")
    dense("patch_embed/conv", (c.patch_size, c.patch_size, c.in_channels, c.embed_dim[0]))
    for j, (D, depth) in enumerate(zip(c.embed_dim, c.nb_blocks)):
        hid = int(D * c.mlp_ratio)
        for k in range(depth):
            p = f"transformers/{j}/blocks/{k}"
            norm(f"{p}/norm1", D)
            dense(f"{p}/attn/qkv", (D, 3 * D))
            dense(f"{p}/attn/proj", (D, D))
            norm(f"{p}/norm2", D)
            dense(f"{p}/mlp/fc1", (D, hid))
            dense(f"{p}/mlp/fc2", (hid, D))
        if j < len(c.nb_blocks) - 1:
            p = f"transformers/{j + 1}/pool"
            dense(f"{p}/conv", (3, 3, 1, c.embed_dim[j + 1]))
            dense(f"{p}/fc", (D, c.embed_dim[j + 1]))
    norm("norm", c.embed_dim[-1])
    if c.nb_classes > 0:
        dense("head", (c.embed_dim[-1], c.nb_classes))
        if c.distilled:
            dense("head_dist", (c.embed_dim[-1], c.nb_classes))
    return s


class PoolingVisionTransformer(Model):
    cfg_class = PoolingVisionTransformerConfig
    accepts_uint8 = True

    def __init__(self, cfg: PoolingVisionTransformerConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = PoolingVisionTransformerConfig(**cfg)
        if cfg.norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        if len({len(cfg.embed_dim), len(cfg.nb_blocks), len(cfg.nb_heads)}) != 1:
            raise ValueError("embed_dim, nb_blocks and nb_heads must have one entry per stage")
        for j, (D, H) in enumerate(zip(cfg.embed_dim, cfg.nb_heads)):
            if D % H or D // H not in pit_ops.HEAD_DIMS:
                raise ValueError(f"stage {j}: head_dim {D}/{H} must be one of {pit_ops.HEAD_DIMS}")
            if j + 1 < len(cfg.embed_dim) and cfg.embed_dim[j + 1] != 2 * D:
                raise ValueError("the pooling layer doubles the width: embed_dim[j + 1] must be 2 embed_dim[j] "
                                 f"(got {cfg.embed_dim})")
        if int(cfg.embed_dim[0] * cfg.mlp_ratio) % 8:
            raise ValueError(f"the kernels need the MLP width to be a multiple of 8 (mlp_ratio {cfg.mlp_ratio})")
        self.nb_features = cfg.embed_dim[-1]
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        return param_specs(self.cfg)

    def transform_pos_embed(self, src_weights, target_cfg: PoolingVisionTransformerConfig):
        """pos_embed resized bicubically on its grid to ``target_cfg``'s (pit.py:296-308)."""
        return self._resized_pos(self.params["pos_embed"], target_cfg.grid_size).permute(0, 3, 1, 2).contiguous()

    @staticmethod
    def _resized_pos(pos_embed, grid):
        """NCHW pos_embed -> (1, gh, gw, D) at ``grid``."""
        pos = pos_embed.permute(0, 2, 3, 1)
        if tuple(grid) != tuple(pos.shape[1:3]):
            pos = tf_bicubic_resize(pos, tuple(grid))
        return pos

    @property
    def feature_names(self) -> List[str]:
        c = self.cfg
        names = ["patch_embedding"]
        for j, depth in enumerate(c.nb_blocks):
            names += [f"stage_{j}/block_{k}" for k in range(depth)]
            if j < len(c.nb_blocks) - 1:
                names.append(f"stage_{j}/pool")
        return names + ["features_all", "features", "logits"]

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        P = {"eps": _LN_EPS[c.norm_layer], "stages": [], "pos": {}}
        P["pe_w"], P["pe_b"] = self._dense_weight("patch_embed/conv/kernel"), self._vec("patch_embed/conv/bias")
        cls = self.params["cls_token"][0].float()
        P["cls"] = cls[0].contiguous()
        P["dist"] = cls[1].contiguous() if c.distilled else None
        for j, depth in enumerate(c.nb_blocks):
            st = {"blocks": []}
            for k in range(depth):
                p = f"transformers/{j}/blocks/{k}"
                st["blocks"].append(dict(
                    n1=(self._vec(f"{p}/norm1/gamma"), self._vec(f"{p}/norm1/beta")),
                    qkv_w=self._dense_weight(f"{p}/attn/qkv/kernel"), qkv_b=self._vec(f"{p}/attn/qkv/bias"),
                    proj_w=self._dense_weight(f"{p}/attn/proj/kernel"), proj_b=self._vec(f"{p}/attn/proj/bias"),
                    n2=(self._vec(f"{p}/norm2/gamma"), self._vec(f"{p}/norm2/beta")),
                    fc1_w=self._dense_weight(f"{p}/mlp/fc1/kernel"), fc1_b=self._vec(f"{p}/mlp/fc1/bias"),
                    fc2_w=self._dense_weight(f"{p}/mlp/fc2/kernel"), fc2_b=self._vec(f"{p}/mlp/fc2/bias"),
                ))
            if j < len(c.nb_blocks) - 1:
                p = f"transformers/{j + 1}/pool"
                st["pool_w"] = self.params[f"{p}/conv/kernel"].float().reshape(9, -1).contiguous()
                st["pool_b"] = self._vec(f"{p}/conv/bias")
                st["fc_w"], st["fc_b"] = self._dense_weight(f"{p}/fc/kernel"), self._vec(f"{p}/fc/bias")
            P["stages"].append(st)
        P["norm"] = (self._vec("norm/gamma"), self._vec("norm/beta"))
        if c.nb_classes > 0:
            P["head_w"], P["head_b"] = self._dense_weight("head/kernel"), self._vec("head/bias")
            if c.distilled:
                P["headd_w"], P["headd_b"] = self._dense_weight("head_dist/kernel"), self._vec("head_dist/bias")
        return P

    def _pos_table(self, P, grid):
        """(nb_tokens + gh * gw, D0) fp32: zero rows for the special tokens, then pos_embed on ``grid`` (built once per
        grid size)."""
        if grid not in P["pos"]:
            pos = self._resized_pos(self.params["pos_embed"].float(), grid)[0].reshape(grid[0] * grid[1], -1)
            zeros = torch.zeros((self.cfg.nb_tokens, pos.shape[1]), dtype=torch.float32, device=pos.device)
            P["pos"][grid] = torch.cat((zeros, pos), dim=0).contiguous()
        return P["pos"][grid]

    # ------------------------------------------------------------------ forward
    def _tokens(self, x, P):
        """Image batch -> (stream (B * T, D0) fp32, gh, gw)."""
        c = self.cfg
        B, H, W, _ = x.shape
        if not c.interpolate_input and (H, W) != tuple(c.input_size):
            raise ValueError(f"Input size {(H, W)} does not match the model's {tuple(c.input_size)}; "
                             "create the model with interpolate_input=True to allow this.")
        pre = self._pixel_stats(x.device) if x.dtype == torch.uint8 else None
        cols, gh, gw = ops.im2col(x, c.patch_size, c.stride, "valid", self.act_dtype, pre=pre)
        if gh < 1 or gw < 1:
            raise ValueError(f"Input size {(H, W)} is smaller than the patch size {c.patch_size}")
        tok = ops.gemm(cols, P["pe_w"], bias=P["pe_b"], out_dtype=torch.float32)
        if tok.stride(0) != tok.shape[1]:
            tok = tok.contiguous()
        xs = ops.assemble_tokens(tok, P["cls"], P["dist"], self._pos_table(P, (gh, gw)), B, gh * gw, torch.float32)
        return xs, gh, gw

    def _block(self, blk, xs, B, T, D, Hh):
        c = self.cfg
        eps, adt = self._plan["eps"], self.act_dtype
        dh = D // Hh
        h = ops.layernorm(xs, *blk["n1"], eps, adt)
        qkv = ops.gemm(h, blk["qkv_w"], bias=blk["qkv_b"])
        a = pit_ops.attention(qkv, B, T, Hh, dh, dh ** -0.5)
        ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], residual=xs, out=xs)
        h = ops.layernorm(xs, *blk["n2"], eps, adt)
        if adt == torch.bfloat16 and ops.mlp_fused_supported(D, blk["fc1_w"].shape[0]):
            # one kernel: the (M, 4D) hidden activations stay on the SM (csrc/mlp_sm90.cu)
            ops.mlp_fused(h, blk["fc1_w"], blk["fc1_b"], blk["fc2_w"], blk["fc2_b"], c.act_layer, residual=xs, out=xs)
        else:
            hid = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
            ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], residual=xs, out=xs)

    def _pool(self, st, xs, B, gh, gw):
        """ConvHeadPooling: the grid rows by pit_pool, the token rows by the token Dense, into a new stream."""
        nb = self.cfg.nb_tokens
        bf16 = self.act_dtype == torch.bfloat16
        y, tokens = pit_ops.pit_pool(xs, st["pool_w"], st["pool_b"], B, nb, gh, gw, tokens_bf16=bf16)
        gh, gw = pit_ops.pool_geometry(gh, gw)
        C = xs.shape[1]
        x3, y3 = xs.view(B, -1, C), y.view(B, nb + gh * gw, 2 * C)
        for i in range(nb):
            a = tokens.view(B, nb, C)[:, i] if bf16 else x3[:, i]
            ops.gemm(a, st["fc_w"], bias=st["fc_b"], out=y3[:, i])
        return y, gh, gw

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        features = OrderedDict()
        xs, gh, gw = self._tokens(x, P)
        B, nb = x.shape[0], c.nb_tokens
        if return_features:
            features["patch_embedding"] = xs.view(B, nb + gh * gw, -1).clone()
        for j, st in enumerate(P["stages"]):
            D, T = c.embed_dim[j], nb + gh * gw
            for k, blk in enumerate(st["blocks"]):
                self._block(blk, xs, B, T, D, c.nb_heads[j])
                if return_features:
                    features[f"stage_{j}/block_{k}"] = xs.view(B, T, D).clone()
            if "pool_w" in st:
                xs, gh, gw = self._pool(st, xs, B, gh, gw)
                if return_features:
                    features[f"stage_{j}/pool"] = xs.view(B, nb + gh * gw, -1).clone()
        D = c.embed_dim[-1]
        x3 = xs.view(B, -1, D)
        rows = [ops.layernorm(x3[:, i], *P["norm"], P["eps"], torch.float32) for i in range(nb)]
        out = torch.stack(rows, dim=1) if c.distilled else rows[0]
        if return_features:
            features["features_all"] = x3
            features["features"] = out
            return out, features
        return out

    def _head(self, feats, w, b):
        return ops.gemm(ops.cast(feats.contiguous(), self.act_dtype), w, bias=b, out_dtype=torch.float32)

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        features = OrderedDict()
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        if c.nb_classes > 0:
            P = self._ensure_plan()
            if not c.distilled:
                x = self._head(x, P["head_w"], P["head_b"])
            else:
                x = torch.stack((self._head(x[:, 0], P["head_w"], P["head_b"]),
                                 self._head(x[:, 1], P["headd_w"], P["headd_b"])), dim=1)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "pit", PoolingVisionTransformer, PoolingVisionTransformerConfig)
