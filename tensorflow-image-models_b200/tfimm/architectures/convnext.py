"""ConvNeXt forward path as a chain of sm_90a kernels.

What the reference computes (tfimm/architectures/convnext.py):
  stem Conv2D(k = s = patch) + LN -> 4 stages; stage s>0 starts with LN + Conv2D(k = s = 2);
  block: ZeroPad(3) -> depthwise 7x7 -> LN -> Dense(C,4C) -> GELU -> Dense(4C,C) -> * gamma -> + shortcut
  head: global average pool -> LN -> Dense                              [convnext.py:219-228, 286-295, 375-440]

How it runs here:
  stem: patchify gather + wgmma GEMM (K = 48) + LN into the residual stream
  downsample: ONE kernel does LN per pixel and writes the 2x2 im2col layout, then a wgmma GEMM
  block: [dw7x7 + bias + LN] (one CUDA-core kernel, bf16 out) -> [fc1 + bias + GELU] ->
         [fc2 + bias, * gamma, + shortcut, in place]   (the last two are the wgmma GEMM epilogues)
  head: pool kernel -> LN -> GEMM
"""
import os
from collections import OrderedDict
from dataclasses import dataclass
from typing import Tuple

import torch

from ..backend import ops
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["ConvNeXt", "ConvNeXtConfig"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}


@dataclass
class ConvNeXtConfig(ModelConfig):
    """Same fields and defaults as the reference's ``ConvNeXtConfig`` (convnext.py:66-134)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_size: int = 4
    embed_dim: Tuple = (96, 192, 384, 768)
    nb_blocks: Tuple = (3, 3, 9, 3)
    mlp_ratio: float = 4.0
    conv_mlp_block: bool = False
    drop_rate: float = 0.0
    drop_path_rate: float = 0.1
    norm_layer: str = "layer_norm_eps_1e-6"
    act_layer: str = "gelu"
    init_scale: float = 1e-6
    crop_pct: float = 0.875
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "stem/0"
    classifier: str = "head/fc"


class ConvNeXt(Model):
    cfg_class = ConvNeXtConfig
    accepts_uint8 = True

    def __init__(self, cfg: ConvNeXtConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = ConvNeXtConfig(**cfg)
        if cfg.norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        c = self.cfg
        s = OrderedDict()
        # tf.keras.initializers.TruncatedNormal(0.02) kernels, zero biases (convnext.py:137-143)
        kinit = "normal:0.02"

        def norm(prefix, n):
            s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
            s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

        s["stem/0/kernel"] = ParamSpec((c.patch_size, c.patch_size, c.in_channels, c.embed_dim[0]), kinit)
        s["stem/0/bias"] = ParamSpec((c.embed_dim[0],), "zeros")
        norm("stem/1", c.embed_dim[0])
        for j, (dim, depth) in enumerate(zip(c.embed_dim, c.nb_blocks)):
            if j > 0:
                norm(f"stages/{j}/downsample/0", c.embed_dim[j - 1])
                s[f"stages/{j}/downsample/1/kernel"] = ParamSpec((2, 2, c.embed_dim[j - 1], dim), kinit)
                s[f"stages/{j}/downsample/1/bias"] = ParamSpec((dim,), "zeros")
            hid = int(c.mlp_ratio * dim)
            lead = (1, 1) if c.conv_mlp_block else ()
            for k in range(depth):
                p = f"stages/{j}/blocks/{k}"
                s[f"{p}/conv_dw/depthwise_kernel"] = ParamSpec((7, 7, dim, 1), kinit)
                s[f"{p}/conv_dw/bias"] = ParamSpec((dim,), "zeros")
                norm(f"{p}/norm", dim)
                s[f"{p}/mlp/fc1/kernel"] = ParamSpec((*lead, dim, hid), kinit)
                s[f"{p}/mlp/fc1/bias"] = ParamSpec((hid,), "zeros")
                s[f"{p}/mlp/fc2/kernel"] = ParamSpec((*lead, hid, dim), kinit)
                s[f"{p}/mlp/fc2/bias"] = ParamSpec((dim,), "zeros")
                s[f"{p}/gamma"] = ParamSpec((dim,), f"const:{c.init_scale}")
        norm("head/norm", c.embed_dim[-1])
        if c.nb_classes > 0:
            s["head/fc/kernel"] = ParamSpec((c.embed_dim[-1], c.nb_classes), kinit)
            s["head/fc/bias"] = ParamSpec((c.nb_classes,), "zeros")
        return s

    def _compile(self):
        c = self.cfg
        P = {"eps": _LN_EPS[c.norm_layer], "stages": []}
        P["stem_w"] = self._dense_weight("stem/0/kernel")
        P["stem_b"] = self._vec("stem/0/bias")
        P["stem_n"] = (self._vec("stem/1/gamma"), self._vec("stem/1/beta"))
        for j, (dim, depth) in enumerate(zip(c.embed_dim, c.nb_blocks)):
            st = {"dim": dim, "blocks": []}
            if j > 0:
                pre = f"stages/{j}/downsample"
                st["ds_n"] = (self._vec(f"{pre}/0/gamma"), self._vec(f"{pre}/0/beta"))
                st["ds_w"] = self._dense_weight(f"{pre}/1/kernel")
                st["ds_b"] = self._vec(f"{pre}/1/bias")
            for k in range(depth):
                p = f"stages/{j}/blocks/{k}"
                st["blocks"].append(dict(
                    dw_w=self.params[f"{p}/conv_dw/depthwise_kernel"].reshape(49, dim).float().contiguous(),
                    dw_b=self._vec(f"{p}/conv_dw/bias"),
                    n=(self._vec(f"{p}/norm/gamma"), self._vec(f"{p}/norm/beta")),
                    fc1_w=self._dense_weight(f"{p}/mlp/fc1/kernel"),
                    fc1_b=self._vec(f"{p}/mlp/fc1/bias"),
                    fc2_w=self._dense_weight(f"{p}/mlp/fc2/kernel"),
                    fc2_b=self._vec(f"{p}/mlp/fc2/bias"),
                    ls=self._vec(f"{p}/gamma"),
                ))
            P["stages"].append(st)
        P["head_n"] = (self._vec("head/norm/gamma"), self._vec("head/norm/beta"))
        if c.nb_classes > 0:
            P["head_w"] = self._dense_weight("head/fc/kernel")
            P["head_b"] = self._vec("head/fc/bias")
        return P

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        features = OrderedDict()
        B, H, W, _ = x.shape
        adt, rdt, eps = self.act_dtype, torch.float32, P["eps"]
        H, W = H // c.patch_size, W // c.patch_size
        patches = self._patchify(x, c.patch_size)
        y = ops.gemm(patches, P["stem_w"], bias=P["stem_b"])
        xs = ops.layernorm(y, *P["stem_n"], eps, rdt)  # residual stream (B*H*W, C) fp32
        if return_features:
            features["stem"] = xs.view(B, H, W, -1).clone()
        for j, st in enumerate(P["stages"]):
            dim = st["dim"]
            if j > 0:
                cols = ops.layernorm_patch2x2(xs.view(B, H, W, -1), *st["ds_n"], eps, adt)
                H, W = H // 2, W // 2
                xs = ops.gemm(cols, st["ds_w"], bias=st["ds_b"], out_dtype=rdt)
                if return_features:
                    features[f"stage_{j}/downsample"] = xs.view(B, H, W, dim).clone()
            for k, blk in enumerate(st["blocks"]):
                h = ops.dwconv_ln(xs.view(B, H, W, dim), blk["dw_w"], blk["dw_b"], *blk["n"], eps, adt)
                if adt == torch.bfloat16 and ops.mlp_fused_supported(dim, blk["fc1_w"].shape[0]):
                    # one kernel: the (M, 4 dim) hidden activations stay on the SM (csrc/mlp_sm90.cu)
                    ops.mlp_fused(h.view(-1, dim), blk["fc1_w"], blk["fc1_b"], blk["fc2_w"], blk["fc2_b"], c.act_layer,
                                  gamma=blk["ls"], residual=xs, out=xs)
                else:
                    hid = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
                    ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], gamma=blk["ls"], residual=xs, out=xs)
                if return_features:
                    features[f"stage_{j}/block_{k}"] = xs.view(B, H, W, dim).clone()
        out = xs.view(B, H, W, -1)
        features["conv_features"] = out
        return (out, features) if return_features else out

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        features = OrderedDict()
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        pooled = ops.global_avg_pool(x)
        x = ops.layernorm(pooled, *P["head_n"], P["eps"], torch.float32)
        features["features"] = x
        if c.nb_classes > 0:
            x = ops.gemm(ops.cast(x, self.act_dtype), P["head_w"], bias=P["head_b"], out_dtype=torch.float32)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "convnext", ConvNeXt, ConvNeXtConfig)
