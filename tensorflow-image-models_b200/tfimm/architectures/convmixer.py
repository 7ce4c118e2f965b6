"""ConvMixer forward path as a chain of sm_90a kernels.

Registered on import (``import tfimm.architectures.convmixer``, module name ``convmixer``); ``import tfimm`` alone does
not import it.

What the reference computes (tfimm/architectures/convmixer.py):
  stem   Conv2D p x p / p, VALID, with bias -> act -> BN                                      (convmixer.py:88-96)
  block  x = x + BN1(act(DepthwiseConv2D_k_same(x) + b));  x = BN2(act(Conv2D_1x1(x) + b))   (convmixer.py:63-73)
  head   GlobalAveragePooling2D -> Dense (linear when nb_classes = 0)                         (convmixer.py:99-106)
  BN is inference-form BatchNormalization with the moving statistics, eps 1e-5; it comes AFTER the activation.

How it runs here.  The GEMM epilogue computes residual + gamma act(acc + bias); it cannot add a per-column shift after
the activation, so every BN is carried forward to whoever reads the activation a = act(z), as x = s a + t with
s = gamma / sqrt(var + eps) and t = beta - mean s folded in float64 at plan time:
  stem     im2col "valid" (uint8 pixels: the preprocessing fused in) -> GEMM + bias + act -> a (fp32)
  block j  convmixer_ops.dwconv(a, BN of the previous stage, taps, b, BN1) -> y = x + s1 act(dw(x) + b) + t1 in the
           activation dtype (x = s a + t inside the image, 0 in the padding) -> 1 x 1 GEMM + bias + act -> a (fp32)
  head     ops.global_avg_pool(a) -> mixer_ops.affine with the last BN (= features) -> head GEMM
  features stem, block_j and features_all are s a + t materialised by mixer_ops.affine, only when asked for.
Storage points: a is fp32 in every precision; y and the stem patches are in the activation dtype; the weights are GEMM
operands as in the other families.  precision "tf32" runs the GEMMs on the TF32 tensor cores; the depthwise kernel is
fp32 on the CUDA cores in every precision.
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Tuple

import torch

from ..backend import convmixer_ops, mixer_ops, ops
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["ConvMixer", "ConvMixerConfig", "param_specs"]

_BN_EPS = 1e-5  # the reference's "batch_norm" factory (layers/factory.py)


@dataclass
class ConvMixerConfig(ModelConfig):
    """Hyper-parameters (same fields and defaults as the reference's ``ConvMixerConfig``, convmixer.py:21-38)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_size: Tuple[int, int] = (7, 7)
    embed_dim: int = 768
    depth: int = 32
    kernel_size: int = 9
    norm_layer: str = "batch_norm"
    act_layer: str = "gelu"
    crop_pct: float = 0.96
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "stem/0"
    classifier: str = "head"


def param_specs(c: ConvMixerConfig) -> "OrderedDict[str, ParamSpec]":
    """The reference's variables (names, shapes, initial values) in creation order: the trainable ones first (Keras
    glorot_uniform kernels, zero biases, BN gamma 1 / beta 0), then every BN's moving_mean / moving_variance (0 / 1) in
    the order the BNs were built."""
    s = OrderedDict()
    bns = []
    ph, pw = c.patch_size
    C, k = c.embed_dim, c.kernel_size

    def bn(prefix):
        s[f"{prefix}/gamma"] = ParamSpec((C,), "ones")
        s[f"{prefix}/beta"] = ParamSpec((C,), "zeros")
        bns.append(prefix)

    s["stem/0/kernel"] = ParamSpec((ph, pw, c.in_channels, C), "glorot_uniform")
    s["stem/0/bias"] = ParamSpec((C,), "zeros")
    bn("stem/2")
    for j in range(c.depth):
        p = f"blocks/{j}"
        s[f"{p}/0/fn/0/depthwise_kernel"] = ParamSpec((k, k, C, 1), "glorot_uniform")
        s[f"{p}/0/fn/0/bias"] = ParamSpec((C,), "zeros")
        bn(f"{p}/0/fn/2")
        s[f"{p}/1/kernel"] = ParamSpec((1, 1, C, C), "glorot_uniform")
        s[f"{p}/1/bias"] = ParamSpec((C,), "zeros")
        bn(f"{p}/3")
    if c.nb_classes > 0:
        s["head/kernel"] = ParamSpec((C, c.nb_classes), "glorot_uniform")
        s["head/bias"] = ParamSpec((c.nb_classes,), "zeros")
    for prefix in bns:
        s[f"{prefix}/moving_mean"] = ParamSpec((C,), "zeros", trainable=False)
        s[f"{prefix}/moving_variance"] = ParamSpec((C,), "ones", trainable=False)
    return s


class ConvMixer(Model):
    cfg_class = ConvMixerConfig
    accepts_uint8 = True

    def __init__(self, cfg: ConvMixerConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = ConvMixerConfig(**cfg)
        if cfg.norm_layer != "batch_norm":
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer} (ConvMixer here takes 'batch_norm')")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        if cfg.kernel_size not in convmixer_ops.KERNEL_SIZES:
            raise ValueError(f"the depthwise kernel takes kernel_size in {convmixer_ops.KERNEL_SIZES}, "
                             f"got {cfg.kernel_size}")
        if cfg.embed_dim <= 0 or cfg.embed_dim % convmixer_ops.CHANNEL_MULTIPLE:
            raise ValueError(f"the depthwise kernel needs embed_dim to be a multiple of "
                             f"{convmixer_ops.CHANNEL_MULTIPLE}, got {cfg.embed_dim}")
        if len(set(cfg.patch_size)) != 1:
            raise ValueError(f"the stem takes square patches, got patch_size {cfg.patch_size}")
        self.nb_features = cfg.embed_dim
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        return param_specs(self.cfg)

    @property
    def feature_names(self) -> List[str]:
        return ["stem"] + [f"block_{j}" for j in range(self.cfg.depth)] + ["features_all", "features", "logits"]

    # ------------------------------------------------------------------ engine plan
    def _bn(self, prefix):
        """Inference BatchNorm as (s, t), x = s a + t, folded in float64."""
        g, b = self.params[f"{prefix}/gamma"].double(), self.params[f"{prefix}/beta"].double()
        m, v = self.params[f"{prefix}/moving_mean"].double(), self.params[f"{prefix}/moving_variance"].double()
        s = g / torch.sqrt(v + _BN_EPS)
        return s.float().contiguous(), (b - m * s).float().contiguous()

    def _compile(self):
        c = self.cfg
        P = {"stem_w": self._dense_weight("stem/0/kernel"), "stem_b": self._vec("stem/0/bias"),
             "stem_bn": self._bn("stem/2"), "blocks": []}
        for j in range(c.depth):
            p = f"blocks/{j}"
            P["blocks"].append(dict(
                taps=self.params[f"{p}/0/fn/0/depthwise_kernel"].float().reshape(c.kernel_size ** 2,
                                                                                   c.embed_dim).contiguous(),
                dw_b=self._vec(f"{p}/0/fn/0/bias"), bn1=self._bn(f"{p}/0/fn/2"),
                pw_w=self._dense_weight(f"{p}/1/kernel"), pw_b=self._vec(f"{p}/1/bias"), bn2=self._bn(f"{p}/3"),
            ))
        if c.nb_classes > 0:
            P["head_w"], P["head_b"] = self._dense_weight("head/kernel"), self._vec("head/bias")
        return P

    # ------------------------------------------------------------------ forward
    def _affine(self, a, bn):
        """s a + t of the fp32 activation a (B, H, W, C) -> fp32 (B, H, W, C)."""
        return mixer_ops.affine(a.view(-1, a.shape[-1]), *bn, torch.float32).view(a.shape)

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        p = c.patch_size[0]
        B, H, W = x.shape[:3]
        if H < p or W < p:
            raise ValueError(f"ConvMixer needs an input of at least {p} x {p} pixels, got {H} x {W}")
        features = OrderedDict()
        pre = self._pixel_stats(x.device) if x.dtype == torch.uint8 else None
        cols, gh, gw = ops.im2col(x, p, p, "valid", self.act_dtype, pre=pre)
        a = ops.gemm(cols, P["stem_w"], bias=P["stem_b"], act=c.act_layer, out_dtype=torch.float32)
        a = a.view(B, gh, gw, c.embed_dim)
        bn = P["stem_bn"]
        if return_features:
            features["stem"] = self._affine(a, bn)
        for j, blk in enumerate(P["blocks"]):
            y = convmixer_ops.dwconv(a, *bn, blk["taps"], blk["dw_b"], *blk["bn1"], c.act_layer, self.act_dtype)
            a = ops.gemm(y.view(-1, c.embed_dim), blk["pw_w"], bias=blk["pw_b"], act=c.act_layer,
                         out_dtype=torch.float32).view(B, gh, gw, c.embed_dim)
            bn = blk["bn2"]
            if return_features:
                features[f"block_{j}"] = self._affine(a, bn)
        out = mixer_ops.affine(ops.global_avg_pool(a), *bn, torch.float32)
        if return_features:
            features["features_all"] = features[f"block_{c.depth - 1}"] if c.depth else features["stem"]
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


register_zoo(__name__, "convmixer", ConvMixer, ConvMixerConfig)
