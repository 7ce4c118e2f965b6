"""PVT v2 (Pyramid Vision Transformer v2) forward path as a chain of sm_90a kernels.

Registered on import (``import tfimm.architectures.pvt_v2``, module name ``pvt_v2``); ``import tfimm`` alone does not
import it.

What the reference computes (tfimm/architectures/pvt_v2.py), per stage j:
  embed   PatchEmbeddings: zero padding k // 2, Conv2D(embed_dim[j], k, stride) + bias with (k, stride) = (7, 4) at stage
          0 and (3, 2) after it, then LayerNorm eps 1e-5; no position table, no class token  (layers/transformers.py)
  blocks  nb_blocks[j] pre-norm blocks (norm_layer, LayerNorm eps 1e-6): spatial-reduction attention as in PVT v1 --
          q = Dense(x); when sr_ratio[j] > 1 the keys and values come from x (B, gh, gw, D) through a VALID sr x sr / sr
          Conv2D + bias and a LayerNorm eps 1e-5; kv = Dense(2D) read as (B, N', 2, H, dh); softmax(q k^T / sqrt(dh))
          v; proj -- then the ConvFFN: fc1, a 3 x 3 "same" depthwise Conv2D + bias on the (gh, gw) grid, the
          activation, fc2                                                                       (pvt_v2.py:77-297)
  then    the stage's own norm_layer (norm{j+1}), the stream reshaped to (B, gh, gw, D) for the next patch embedding
  head    the mean over the last stage's tokens (features), Dense head                          (pvt_v2.py:381-414)

How it runs here (fp32 residual stream (B * gh * gw, D) in every precision):
  embed   im2col with zero padding k // 2 (uint8 pixels at stage 0: the preprocessing fused in) -> GEMM + bias (fp32)
          -> layernorm (1e-5, fp32)
  block   layernorm -> q GEMM; sr > 1: im2col(h, sr, sr, "valid") -> GEMM + bias (fp32) -> layernorm (1e-5); -> kv GEMM
          -> pvt_v2_ops.sr_attention (head dim 64: PVT v1's kernels, 32: this family's) -> proj GEMM (+ residual, in
          place) -> layernorm -> pvt_v2_ops.conv_mlp (+ residual, in place): in bf16 at C in {32, 64} one fused
          kernel, else fc1 GEMM, dwconv_bias_act, fc2 GEMM
  stage   layernorm (norm_layer, fp32)
  head    global_avg_pool of the last stage -> head GEMM
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Tuple

import torch

from ..backend import ops, pvt_v2_ops
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["PyramidVisionTransformerV2", "PyramidVisionTransformerV2Config", "param_specs"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}
_EMBED_EPS = 1e-5   # the patch embeddings' and the spatial reduction's "layer_norm"


@dataclass
class PyramidVisionTransformerV2Config(ModelConfig):
    """Hyper-parameters (same fields and defaults as the reference's ``PyramidVisionTransformerV2Config``,
    pvt_v2.py:29-74)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    embed_dim: Tuple = (64, 128, 256, 512)
    nb_blocks: Tuple = (3, 4, 6, 3)
    nb_heads: Tuple = (1, 2, 5, 8)
    mlp_ratio: Tuple = (8.0, 8.0, 4.0, 4.0)
    sr_ratio: Tuple = (8, 4, 2, 1)
    linear_sr: bool = False
    qkv_bias: bool = True
    drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    attn_drop_rate: float = 0.0
    norm_layer: str = "layer_norm_eps_1e-6"
    act_layer: str = "gelu"
    crop_pct: float = 0.9
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "patch_embed1/proj"
    classifier: str = "head"


def patch_geometry(j):
    """(kernel size, stride, zero padding) of stage j's overlapping patch embedding (pvt_v2.py:319-326)."""
    k, s = (7, 4) if j == 0 else (3, 2)
    return k, s, k // 2


def grids(size, nb_stages):
    """The grid of every stage: floor((n + 2 p - k) / s) + 1 per padded, strided convolution."""
    out = []
    h, w = size
    for j in range(nb_stages):
        k, s, p = patch_geometry(j)
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        out.append((h, w))
    return tuple(out)


def param_specs(c: PyramidVisionTransformerV2Config) -> "OrderedDict[str, ParamSpec]":
    """The reference's variables (names, shapes, initial values) in the order of its ``weights``: the layers in the
    order Keras tracks them -- the lists patch_embed, blocks and norms in the order __init__ assigns them, then the
    head; in each block norm1, the attention's q, kv, proj, sr and its norm, norm2, the MLP's fc1, depthwise
    convolution and fc2 -- with Keras' default initialisers (glorot_uniform kernels, zero biases, LayerNorm 1 / 0)."""
    s = OrderedDict()

    def dense(prefix, shape, bias=True, leaf="kernel"):
        s[f"{prefix}/{leaf}"] = ParamSpec(shape, "glorot_uniform")
        if bias:
            s[f"{prefix}/bias"] = ParamSpec((shape[-2] if leaf == "depthwise_kernel" else shape[-1],), "zeros")

    def norm(prefix, n):
        s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
        s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

    cin = c.in_channels
    for j, D in enumerate(c.embed_dim):
        k = patch_geometry(j)[0]
        dense(f"patch_embed{j + 1}/proj", (k, k, cin, D))
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
            dense(f"{b}/mlp/dwconv/dwconv", (3, 3, hid, 1), leaf="depthwise_kernel")
            dense(f"{b}/mlp/fc2", (hid, D))
    for j, D in enumerate(c.embed_dim):
        norm(f"norm{j + 1}", D)
    if c.nb_classes > 0:
        dense("head", (c.embed_dim[-1], c.nb_classes))
    return s


class PyramidVisionTransformerV2(Model):
    cfg_class = PyramidVisionTransformerV2Config
    accepts_uint8 = True

    def __init__(self, cfg: PyramidVisionTransformerV2Config, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = PyramidVisionTransformerV2Config(**cfg)
        if cfg.linear_sr:
            raise ValueError("linear_sr=True (pvt_v2_b2_li's adaptive-pooling spatial reduction) is not supported; the "
                             "reference leaves it unregistered as broken")
        if cfg.norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        fields = (cfg.embed_dim, cfg.nb_blocks, cfg.nb_heads, cfg.mlp_ratio, cfg.sr_ratio)
        if len({len(f) for f in fields}) != 1:
            raise ValueError("embed_dim, nb_blocks, nb_heads, mlp_ratio and sr_ratio must have one entry per stage")
        for j, (D, H) in enumerate(zip(cfg.embed_dim, cfg.nb_heads)):
            if D % H or D // H not in pvt_v2_ops.HEAD_DIMS:
                raise ValueError(f"stage {j}: head_dim {D}/{H} must be one of {pvt_v2_ops.HEAD_DIMS}")
            if int(D * cfg.mlp_ratio[j]) % 8:
                raise ValueError(f"stage {j}: the kernels need the MLP width to be a multiple of 8 "
                                 f"(mlp_ratio {cfg.mlp_ratio[j]})")
        self.nb_features = cfg.embed_dim[-1]
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        return param_specs(self.cfg)

    @property
    def feature_names(self) -> List[str]:
        names, k = [], 0
        for j, depth in enumerate(self.cfg.nb_blocks):
            names.append(f"patch_embedding_{j}")
            names += [f"block_{k + i}" for i in range(depth)]
            k += depth
            names.append(f"stage_{j}")
        return names + ["features_all", "features", "logits"]

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        P = {"eps": _LN_EPS[c.norm_layer], "stages": []}
        for j, depth in enumerate(c.nb_blocks):
            pe = f"patch_embed{j + 1}"
            st = {"pe_w": self._dense_weight(f"{pe}/proj/kernel"), "pe_b": self._vec(f"{pe}/proj/bias"),
                  "pe_n": (self._vec(f"{pe}/norm/gamma"), self._vec(f"{pe}/norm/beta")),
                  "norm": (self._vec(f"norm{j + 1}/gamma"), self._vec(f"norm{j + 1}/beta")), "blocks": []}
            for k in range(depth):
                b = f"block{j + 1}/{k}"
                bias = (lambda key: self._vec(key)) if c.qkv_bias else (lambda key: None)
                hid = int(c.embed_dim[j] * c.mlp_ratio[j])
                blk = dict(
                    n1=(self._vec(f"{b}/norm1/gamma"), self._vec(f"{b}/norm1/beta")),
                    q_w=self._dense_weight(f"{b}/attn/q/kernel"), q_b=bias(f"{b}/attn/q/bias"),
                    kv_w=self._dense_weight(f"{b}/attn/kv/kernel"), kv_b=bias(f"{b}/attn/kv/bias"),
                    proj_w=self._dense_weight(f"{b}/attn/proj/kernel"), proj_b=self._vec(f"{b}/attn/proj/bias"),
                    n2=(self._vec(f"{b}/norm2/gamma"), self._vec(f"{b}/norm2/beta")),
                    fc1_w=self._dense_weight(f"{b}/mlp/fc1/kernel"), fc1_b=self._vec(f"{b}/mlp/fc1/bias"),
                    # (3, 3, hidden, 1) -> (9, hidden): taps in (ky, kx) order, as dwconv_bias_act takes them
                    dw_w=self.params[f"{b}/mlp/dwconv/dwconv/depthwise_kernel"].float().reshape(9, hid).contiguous(),
                    dw_b=self._vec(f"{b}/mlp/dwconv/dwconv/bias"),
                    fc2_w=self._dense_weight(f"{b}/mlp/fc2/kernel"), fc2_b=self._vec(f"{b}/mlp/fc2/bias"),
                )
                if c.sr_ratio[j] > 1:
                    blk["sr_w"], blk["sr_b"] = self._dense_weight(f"{b}/attn/sr/kernel"), self._vec(f"{b}/attn/sr/bias")
                    blk["srn"] = (self._vec(f"{b}/attn/norm/gamma"), self._vec(f"{b}/attn/norm/beta"))
                st["blocks"].append(blk)
            P["stages"].append(st)
        if c.nb_classes > 0:
            P["head_w"], P["head_b"] = self._dense_weight("head/kernel"), self._vec("head/bias")
        return P

    def _check_input(self, H, W):
        """The stage grids of an (H, W) input; ValueError, before any launch, for inputs the model cannot run."""
        c = self.cfg
        if H < 1 or W < 1:
            raise ValueError(f"Input size {(H, W)} is empty")
        gs = grids((H, W), len(c.nb_blocks))
        for j, ((gh, gw), sr) in enumerate(zip(gs, c.sr_ratio)):
            if gh < max(1, sr) or gw < max(1, sr):
                raise ValueError(f"Input size {(H, W)}: stage {j}'s grid {gh} x {gw} is smaller than its "
                                 f"spatial-reduction ratio {sr}, which leaves no keys")
        return gs

    # ------------------------------------------------------------------ forward
    def _block(self, blk, xs, B, gh, gw, D, Hh, sr):
        c = self.cfg
        eps, adt = self._plan["eps"], self.act_dtype
        dh, N = D // Hh, gh * gw
        h = ops.layernorm(xs, *blk["n1"], eps, adt)
        q = ops.gemm(h, blk["q_w"], bias=blk["q_b"])
        if sr > 1:
            cols, rh, rw = ops.im2col(h.view(B, gh, gw, D), sr, sr, "valid", adt)
            r = ops.gemm(cols, blk["sr_w"], bias=blk["sr_b"], out_dtype=torch.float32)
            src, Nk = ops.layernorm(r, *blk["srn"], _EMBED_EPS, adt), rh * rw
        else:
            src, Nk = h, N
        kv = ops.gemm(src, blk["kv_w"], bias=blk["kv_b"])
        a = pvt_v2_ops.sr_attention(q, kv, B, N, Nk, Hh, dh, dh ** -0.5)
        ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], residual=xs, out=xs)
        h = ops.layernorm(xs, *blk["n2"], eps, adt)
        pvt_v2_ops.conv_mlp(h, blk["fc1_w"], blk["fc1_b"], blk["dw_w"], blk["dw_b"], blk["fc2_w"], blk["fc2_b"], xs,
                            B, gh, gw, c.act_layer, out=xs)

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        x = self._input(x)
        B = x.shape[0]
        gs = self._check_input(x.shape[1], x.shape[2])
        P = self._ensure_plan()
        features = OrderedDict()
        img, k = x, 0
        for j, st in enumerate(P["stages"]):
            D = c.embed_dim[j]
            ks, stride, pad = patch_geometry(j)
            pre = self._pixel_stats(x.device) if img.dtype == torch.uint8 else None
            cols, gh, gw = ops.im2col(img, ks, stride, pad, self.act_dtype, pre=pre)
            assert (gh, gw) == gs[j]
            tok = ops.gemm(cols, st["pe_w"], bias=st["pe_b"], out_dtype=torch.float32)
            xs = ops.layernorm(tok, *st["pe_n"], _EMBED_EPS, torch.float32)
            if return_features:
                features[f"patch_embedding_{j}"] = xs.view(B, gh * gw, D).clone()
            for blk in st["blocks"]:
                self._block(blk, xs, B, gh, gw, D, c.nb_heads[j], c.sr_ratio[j])
                if return_features:
                    features[f"block_{k}"] = xs.view(B, gh * gw, D).clone()
                k += 1
            img = ops.layernorm(xs, *st["norm"], P["eps"], torch.float32).view(B, gh, gw, D)
            if return_features:
                features[f"stage_{j}"] = img
        D = c.embed_dim[-1]
        out = ops.global_avg_pool(img)
        if return_features:
            features["features_all"] = img.view(B, -1, D)
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


register_zoo(__name__, "pvt_v2", PyramidVisionTransformerV2, PyramidVisionTransformerV2Config)
