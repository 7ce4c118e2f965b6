"""PoolFormer forward path as a chain of sm_90a kernels.

Registered on import (``import tfimm.architectures.poolformer``, module name ``poolformer``); ``import tfimm`` alone does
not import it.

What the reference computes (tfimm/architectures/poolformer.py, layers/transformers.py, layers/norm.py):
  stem        ZeroPadding2D(2) -> Conv2D 7 x 7 / 4 with bias (PatchEmbeddings, poolformer.py:227-237)
  block       x += ls1 * (AvgPool3x3_same(GN(x)) - GN(x));  x += ls2 * fc2(GELU(fc1(GN(x))))       (poolformer.py:188-202)
              GN: GroupNormalization with one group -- moments over the whole (H, W, C) image, eps 1e-5, biased
              variance, per-channel gamma / beta; the pool excludes padded cells from its count (TF "same")
  downsample  ZeroPadding2D(1) -> Conv2D 3 x 3 / 2 with bias between stages (poolformer.py:256-267)
  head        GN -> GlobalAveragePooling2D -> Dense (poolformer.py:270-276, 320-325, 349)

How it runs here (fp32 residual stream (B, H, W, C) in every precision):
  stem / downsample   im2col (uint8 pixels: create_preprocessing fused in, the padding stays 0 after it) -> GEMM
  block               poolformer_ops.gn1_partials(x)   norm1's statistics (x is a stem, downsample or MLP output)
                      poolformer_ops.poolformer_mixer  token mixer, out of place, + the partials of its output
                      poolformer_ops.gn1_apply         norm2 -> the fc1 operand (bf16, or fp32 for fp32 / tf32)
                      ops.mlp_fused where ops.mlp_fused_supported(C, 4C) in bf16, else fc1 + GELU GEMM, then fc2 GEMM
                      with ls2 as gamma and the stream as the residual, in place
  head                gn1_partials -> gn1_apply (fp32: features_all) -> global_avg_pool -> head GEMM
precision "tf32" runs the GEMMs on the TF32 tensor cores; the PoolFormer kernels are fp32 in every precision.
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Tuple

import torch

from ..backend import ops, poolformer_ops
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["PoolFormer", "PoolFormerConfig", "param_specs"]

_GN_EPS = 1e-5  # GroupNormalization's default epsilon (layers/norm.py)


@dataclass
class PoolFormerConfig(ModelConfig):
    """Hyper-parameters (same fields and defaults as the reference's ``PoolFormerConfig``, poolformer.py:48-107)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    embed_dim: Tuple = (64, 128, 320, 512)
    nb_blocks: Tuple = (2, 2, 6, 2)
    mlp_ratio: Tuple = (4.0, 4.0, 4.0, 4.0)
    drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    norm_layer: str = "group_norm_1grp"
    act_layer: str = "gelu"
    init_scale: float = 1e-5
    crop_pct: float = 0.95
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "patch_embed/proj"
    classifier: str = "head"


def param_specs(c: PoolFormerConfig) -> "OrderedDict[str, ParamSpec]":
    """The reference's variables (names, shapes, initial values) in creation order: TruncatedNormal(0.02) kernels and
    zero biases (poolformer.py:110-116), the layer scales at init_scale, created by the block's build() before its
    sublayers (poolformer.py:174-186)."""
    s = OrderedDict()
    kinit = "normal:0.02"

    def conv(prefix, k, n_in, n_out):
        s[f"{prefix}/kernel"] = ParamSpec((k, k, n_in, n_out), kinit)
        s[f"{prefix}/bias"] = ParamSpec((n_out,), "zeros")

    def norm(prefix, n):
        s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
        s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

    conv("patch_embed/proj", 7, c.in_channels, c.embed_dim[0])
    for j, (dim, depth) in enumerate(zip(c.embed_dim, c.nb_blocks)):
        hid = int(dim * c.mlp_ratio[j])
        for k in range(depth):
            p = f"network/{2 * j}/{k}"
            s[f"{p}/layer_scale_1"] = ParamSpec((dim,), f"const:{c.init_scale}")
            s[f"{p}/layer_scale_2"] = ParamSpec((dim,), f"const:{c.init_scale}")
            norm(f"{p}/norm1", dim)
            norm(f"{p}/norm2", dim)
            conv(f"{p}/mlp/fc1", 1, dim, hid)
            conv(f"{p}/mlp/fc2", 1, hid, dim)
        if j < len(c.nb_blocks) - 1:
            conv(f"network/{2 * j + 1}/proj", 3, dim, c.embed_dim[j + 1])
    norm("norm", c.embed_dim[-1])
    if c.nb_classes > 0:
        s["head/kernel"] = ParamSpec((c.embed_dim[-1], c.nb_classes), kinit)
        s["head/bias"] = ParamSpec((c.nb_classes,), "zeros")
    return s


class PoolFormer(Model):
    cfg_class = PoolFormerConfig
    accepts_uint8 = True

    def __init__(self, cfg: PoolFormerConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = PoolFormerConfig(**cfg)
        if cfg.norm_layer != "group_norm_1grp":
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        if any(d % 8 for d in cfg.embed_dim) or any(int(d * r) % 8 for d, r in zip(cfg.embed_dim, cfg.mlp_ratio)):
            raise ValueError(f"the kernels need every width and MLP width to be a multiple of 8 (got {cfg.embed_dim}, "
                             f"mlp_ratio {cfg.mlp_ratio})")
        self.nb_features = cfg.embed_dim[-1]
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        return param_specs(self.cfg)

    @property
    def feature_names(self) -> List[str]:
        c = self.cfg
        names = ["patch_embedding"]
        for j, depth in enumerate(c.nb_blocks):
            names += [f"stage_{j}/block_{k}" for k in range(depth)]
            if j < len(c.nb_blocks) - 1:
                names.append(f"stage_{j}/downsample")
        return names + ["features_all", "features", "logits"]

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        P = {"stem_w": self._dense_weight("patch_embed/proj/kernel"), "stem_b": self._vec("patch_embed/proj/bias"),
             "stages": []}
        for j, depth in enumerate(c.nb_blocks):
            st = {"blocks": []}
            for k in range(depth):
                p = f"network/{2 * j}/{k}"
                st["blocks"].append(dict(
                    ls1=self._vec(f"{p}/layer_scale_1"), ls2=self._vec(f"{p}/layer_scale_2"),
                    n1=(self._vec(f"{p}/norm1/gamma"), self._vec(f"{p}/norm1/beta")),
                    n2=(self._vec(f"{p}/norm2/gamma"), self._vec(f"{p}/norm2/beta")),
                    fc1_w=self._dense_weight(f"{p}/mlp/fc1/kernel"), fc1_b=self._vec(f"{p}/mlp/fc1/bias"),
                    fc2_w=self._dense_weight(f"{p}/mlp/fc2/kernel"), fc2_b=self._vec(f"{p}/mlp/fc2/bias"),
                ))
            if j < len(c.nb_blocks) - 1:
                st["ds_w"] = self._dense_weight(f"network/{2 * j + 1}/proj/kernel")
                st["ds_b"] = self._vec(f"network/{2 * j + 1}/proj/bias")
            P["stages"].append(st)
        P["norm"] = (self._vec("norm/gamma"), self._vec("norm/beta"))
        if c.nb_classes > 0:
            P["head_w"], P["head_b"] = self._dense_weight("head/kernel"), self._vec("head/bias")
        return P

    # ------------------------------------------------------------------ forward
    def _conv(self, x, w, b, ks, stride, pad):
        """Zero padding + k x k / stride Conv2D with bias into a new fp32 stream (B, Ho, Wo, N)."""
        pre = self._pixel_stats(x.device) if x.dtype == torch.uint8 else None
        cols, Ho, Wo = ops.im2col(x, ks, stride, pad, self.act_dtype, pre=pre)
        y = ops.gemm(cols, w, bias=b, out_dtype=torch.float32)
        if y.stride(0) != y.shape[1]:
            y = y.contiguous()
        return y.view(x.shape[0], Ho, Wo, -1)

    def _block(self, blk, x):
        """One PoolFormerBlock on the fp32 stream x (B, H, W, C) -> the new stream (the MLP adds into the mixer's
        output in place).  x is a stem, downsample or MLP output, so its partials are computed here; norm2's come
        with the mixer's output."""
        c = self.cfg
        B, H, W, C = x.shape
        partials = poolformer_ops.gn1_partials(x)
        y, p2 = poolformer_ops.poolformer_mixer(x, partials, *blk["n1"], blk["ls1"], _GN_EPS)
        h = poolformer_ops.gn1_apply(y, p2, *blk["n2"], _GN_EPS, self.act_dtype)
        y2 = y.view(B * H * W, C)
        if self.act_dtype == torch.bfloat16 and ops.mlp_fused_supported(C, blk["fc1_w"].shape[0]):
            # one kernel: the (M, 4C) hidden activations stay on the SM (csrc/mlp_sm90.cu)
            ops.mlp_fused(h, blk["fc1_w"], blk["fc1_b"], blk["fc2_w"], blk["fc2_b"], c.act_layer, gamma=blk["ls2"],
                          residual=y2, out=y2)
        else:
            hid = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
            ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], gamma=blk["ls2"], residual=y2, out=y2)
        return y

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        features = OrderedDict()
        x = self._conv(x, P["stem_w"], P["stem_b"], 7, 4, 2)
        if return_features:
            features["patch_embedding"] = x.clone()
        for j, st in enumerate(P["stages"]):
            for k, blk in enumerate(st["blocks"]):
                x = self._block(blk, x)
                if return_features:
                    features[f"stage_{j}/block_{k}"] = x.clone()
            if "ds_w" in st:
                x = self._conv(x, st["ds_w"], st["ds_b"], 3, 2, 1)
                if return_features:
                    features[f"stage_{j}/downsample"] = x.clone()
        B, H, W, C = x.shape
        full = poolformer_ops.gn1_apply(x, poolformer_ops.gn1_partials(x), *P["norm"], _GN_EPS, torch.float32)
        full = full.view(B, H, W, C)
        out = ops.global_avg_pool(full)
        if return_features:
            features["features_all"] = full
            features["features"] = out
            return out, features
        return out

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        features = OrderedDict()
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        if c.nb_classes > 0:
            P = self._ensure_plan()
            x = ops.gemm(ops.cast(x, self.act_dtype), P["head_w"], bias=P["head_b"], out_dtype=torch.float32)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "poolformer", PoolFormer, PoolFormerConfig)
