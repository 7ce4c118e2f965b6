"""EfficientNet / MobileNet-V2 family forward path as a chain of sm_90a kernels.

What the reference computes (tfimm/architectures/efficientnet.py, efficientnet_blocks.py,
efficientnet_builder.py): stem Conv3x3/s2 + BN + act -> stages of MBConv-style blocks decoded from
strings such as ``ir_r2_k3_s2_e6_c24_se0.25`` -> 1x1 head conv + BN + act -> global pool -> Dense.
                                                   [efficientnet.py:278-345, efficientnet_blocks.py:348-535]

How it runs here (inference, so every BatchNorm is folded into the preceding conv at load time):
  1x1 convs (expand / project / head)   wgmma GEMM, folded-BN bias + act (+ residual) in the epilogue
  depthwise k x k (TF "same" or symmetric pad)  one CUDA-core kernel with bias + act and the squeeze
                                                (per-image channel sums) fused in
  squeeze-excite                        one tiny kernel per block for the two FCs + a channel-scale pass
  dense k x k convs (stem, fused-MBConv) im2col gather + wgmma GEMM
"""
import math
import re
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

from ..backend import ops
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD, make_divisible
from ._zoo import register_zoo

__all__ = ["EfficientNet", "EfficientNetConfig"]

_BN_EPS = {"batch_norm": 1e-5, "batch_norm_tf": 1e-3}


@dataclass
class EfficientNetConfig(ModelConfig):
    """Same fields and defaults as the reference's ``EfficientNetConfig`` (efficientnet.py:119-190)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    stem_size: int = 32
    architecture: Tuple[Tuple[str, ...], ...] = ()
    channel_multiplier: float = 1.0
    depth_multiplier: float = 1.0
    fix_first_last: bool = False
    nb_features: int = 1280
    drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    norm_layer: str = "batch_norm"
    act_layer: str = "swish"
    padding: str = "symmetric"
    crop_pct: float = 0.875
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "conv_stem"
    classifier: str = "classifier"


# ----------------------------------------------------------------------------------------------------
# Architecture strings -> flat list of resolved blocks
# ----------------------------------------------------------------------------------------------------
@dataclass
class BlockSpec:
    """One fully resolved block (channels, strides and SE width already computed)."""

    kind: str            # "ir" | "ds" | "er" | "cn"
    name: str            # weight prefix, "blocks.<stage>.<index>"
    key: str             # feature key, "stage_<stage>/block_<index>"
    c_in: int
    c_mid: int           # expanded width (== c_in for "ds"; unused for "cn")
    c_out: int
    kernel: int          # depthwise (ir/ds) or dense (er/cn) kernel size
    stride: int
    se_rd: int           # squeeze width, 0 = no SE
    act: str
    pw_act: bool
    skip: bool


_ACT_CODES = {"re": "relu", "r6": "relu6", "hs": "hard_swish", "sw": "swish", "mi": "mish"}


def parse_block_string(text: str) -> dict:
    """``ir_r2_k3_s2_e6_c24_se0.25_noskip`` -> option dict (notation: efficientnet_blocks.py:66-186)."""
    head, *opts = text.split("_")
    out = {"type": head, "skip": head != "dsa", "act": None}
    for tok in opts:
        if tok == "noskip":
            out["skip"] = False
        elif tok == "skip":
            out["skip"] = head != "dsa"
        elif tok.startswith("n"):
            out["act"] = _ACT_CODES[tok[1:]]
        else:
            m = re.match(r"([a-z]+)(\d.*)", tok)
            if m:
                out[m.group(1)] = m.group(2)
    return out


def _ksize(v: str) -> int:
    k = v.split(".")
    if len(k) == 2 and k[0] != k[1]:
        raise NotImplementedError(f"Non-square kernel {v} is not supported.")
    return int(k[0])


def scaled_repeats(repeats: List[int], multiplier: float) -> List[int]:
    """Depth scaling of one stage ("ceil" truncation), distributing from the last block definition
    backwards (efficientnet_builder.py:47-93)."""
    total = sum(repeats)
    budget = int(math.ceil(total * multiplier))
    out = []
    for r in reversed(repeats):
        take = max(1, round(r / total * budget))
        out.append(take)
        total -= r
        budget -= take
    return out[::-1]


def resolve_blocks(cfg: EfficientNetConfig) -> List[BlockSpec]:
    """Everything EfficientNetBuilder / decode_architecture decide, as a flat list
    (efficientnet_builder.py:96-144, 173-283)."""
    nb_stages = len(cfg.architecture)
    blocks: List[BlockSpec] = []
    c_prev = cfg.stem_size
    for si, strings in enumerate(cfg.architecture):
        parsed = [parse_block_string(s) for s in strings]
        fixed = cfg.fix_first_last and si in (0, nb_stages - 1)
        reps = scaled_repeats([int(p["r"]) for p in parsed], 1.0 if fixed else cfg.depth_multiplier)
        bi = 0
        for p, rep in zip(parsed, reps):
            for _ in range(rep):
                kind = "ds" if p["type"] == "dsa" else p["type"]
                if kind not in ("ir", "ds", "er", "cn"):
                    raise ValueError(f"Unknown block type {p['type']} while building model.")
                if "cc" in p and int(p["cc"]) > 0:
                    raise NotImplementedError("CondConv blocks are not implemented.")
                if "gs" in p:
                    raise NotImplementedError("Grouped pointwise convolutions are not implemented.")
                if _ksize(p.get("a", "1")) != 1 and kind != "er" or _ksize(p.get("p", "1")) != 1:
                    raise NotImplementedError("Only 1x1 expansion / projection kernels are implemented.")
                exp_ratio = float(p.get("e", 1.0))
                se_ratio = float(p.get("se", 0.0))
                if kind != "cn":
                    se_ratio /= exp_ratio
                c_out = make_divisible(int(p["c"]) * cfg.channel_multiplier, 8)
                if kind == "ir":
                    c_mid = make_divisible(c_prev * exp_ratio, 8)
                elif kind == "er":
                    forced = make_divisible(int(p["fc"]) * cfg.channel_multiplier, 8) if int(p.get("fc", 0)) else c_prev
                    c_mid = make_divisible(forced * exp_ratio, 8)
                else:
                    c_mid = c_prev
                stride = int(p["s"]) if bi == 0 else 1
                if stride not in (1, 2):
                    raise ValueError("stride must be 1 or 2")
                se_in = c_mid if kind in ("ir", "er") else c_prev
                se_rd = round(se_in * se_ratio) if (se_ratio > 0.0 and kind != "cn") else 0
                skip = bool(p["skip"]) and stride == 1 and c_out == c_prev
                blocks.append(BlockSpec(
                    kind=kind, name=f"blocks.{si}.{bi}", key=f"stage_{si}/block_{bi}", c_in=c_prev, c_mid=c_mid,
                    c_out=c_out, kernel=_ksize(p["k"]), stride=stride, se_rd=se_rd,
                    act=p["act"] or cfg.act_layer, pw_act=p["type"] == "dsa", skip=skip))
                c_prev = c_out
                bi += 1
    return blocks


class EfficientNet(Model):
    cfg_class = EfficientNetConfig
    accepts_uint8 = True   # raw pixels: create_preprocessing fused into the stem's im2col gather

    def __init__(self, cfg: EfficientNetConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = EfficientNetConfig(**cfg)
        if cfg.norm_layer not in _BN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        if cfg.padding not in ("same", "symmetric", "valid"):
            raise ValueError(f"Unknown padding: {cfg.padding}")
        ops.act_code(cfg.act_layer)
        self.blocks = resolve_blocks(cfg)
        for b in self.blocks:
            ops.act_code(b.act)
        super().__init__(cfg, *args, **kwargs)

    # ------------------------------------------------------------------ parameters
    def _param_specs(self):
        c = self.cfg
        s = OrderedDict()

        def conv(prefix, k, cin, cout, bias=False):
            s[f"{prefix}/kernel"] = ParamSpec((k, k, cin, cout), "glorot_uniform")
            if bias:
                s[f"{prefix}/bias"] = ParamSpec((cout,), "zeros")

        def dwconv(prefix, k, ch):
            s[f"{prefix}/depthwise_kernel"] = ParamSpec((k, k, ch, 1), "glorot_uniform")

        def bn(prefix, ch):
            s[f"{prefix}/gamma"] = ParamSpec((ch,), "ones")
            s[f"{prefix}/beta"] = ParamSpec((ch,), "zeros")
            s[f"{prefix}/moving_mean"] = ParamSpec((ch,), "zeros", trainable=False)
            s[f"{prefix}/moving_variance"] = ParamSpec((ch,), "ones", trainable=False)

        def se(prefix, ch, rd):
            conv(f"{prefix}/conv_reduce", 1, ch, rd, bias=True)
            conv(f"{prefix}/conv_expand", 1, rd, ch, bias=True)

        conv("conv_stem", 3, c.in_channels, c.stem_size)
        bn("bn1", c.stem_size)
        for b in self.blocks:
            p = b.name
            if b.kind == "ir":
                conv(f"{p}/conv_pw", 1, b.c_in, b.c_mid)
                bn(f"{p}/bn1", b.c_mid)
                dwconv(f"{p}/conv_dw", b.kernel, b.c_mid)
                bn(f"{p}/bn2", b.c_mid)
                if b.se_rd:
                    se(f"{p}/se", b.c_mid, b.se_rd)
                conv(f"{p}/conv_pwl", 1, b.c_mid, b.c_out)
                bn(f"{p}/bn3", b.c_out)
            elif b.kind == "ds":
                dwconv(f"{p}/conv_dw", b.kernel, b.c_in)
                bn(f"{p}/bn1", b.c_in)
                if b.se_rd:
                    se(f"{p}/se", b.c_in, b.se_rd)
                conv(f"{p}/conv_pw", 1, b.c_in, b.c_out)
                bn(f"{p}/bn2", b.c_out)
            elif b.kind == "er":
                conv(f"{p}/conv_exp", b.kernel, b.c_in, b.c_mid)
                bn(f"{p}/bn1", b.c_mid)
                if b.se_rd:
                    se(f"{p}/se", b.c_mid, b.se_rd)
                conv(f"{p}/conv_pwl", 1, b.c_mid, b.c_out)
                bn(f"{p}/bn2", b.c_out)
            else:  # cn
                conv(f"{p}/conv", b.kernel, b.c_in, b.c_out)
                bn(f"{p}/bn1", b.c_out)
        conv("conv_head", 1, self.blocks[-1].c_out if self.blocks else c.stem_size, c.nb_features)
        bn("bn2", c.nb_features)
        if c.nb_classes > 0:
            s["classifier/kernel"] = ParamSpec((c.nb_features, c.nb_classes), "glorot_uniform")
            s["classifier/bias"] = ParamSpec((c.nb_classes,), "zeros")
        return s

    # ------------------------------------------------------------------ engine plan (BN folded)
    def _bn_scale_shift(self, prefix):
        eps = _BN_EPS[self.cfg.norm_layer]
        g, b = self.params[f"{prefix}/gamma"].float(), self.params[f"{prefix}/beta"].float()
        m, v = self.params[f"{prefix}/moving_mean"].float(), self.params[f"{prefix}/moving_variance"].float()
        scale = g * torch.rsqrt(v + eps)
        return scale, b - m * scale

    def _folded_conv(self, conv_prefix, bn_prefix):
        """Dense conv kernel (kh,kw,cin,cout) + BN -> (W[cout][Kpad] in act dtype, bias fp32)."""
        scale, shift = self._bn_scale_shift(bn_prefix)
        w = self.params[f"{conv_prefix}/kernel"].float() * scale  # broadcast over the last (cout) axis
        cout = w.shape[-1]
        w2 = w.reshape(-1, cout).t().contiguous()
        K = w2.shape[1]
        Kpad = (K + 7) // 8 * 8
        if Kpad != K:
            w2 = torch.nn.functional.pad(w2, (0, Kpad - K))
        return self._gemm_operand(w2), shift.contiguous()

    def _folded_dw(self, conv_prefix, bn_prefix):
        scale, shift = self._bn_scale_shift(bn_prefix)
        w = self.params[f"{conv_prefix}/depthwise_kernel"].float()[..., 0] * scale  # (k,k,C)
        return w.reshape(-1, w.shape[-1]).contiguous(), shift.contiguous()

    def _se_weights(self, prefix):
        wr = self.params[f"{prefix}/conv_reduce/kernel"].float()[0, 0].t().contiguous()   # (rd, C)
        we = self.params[f"{prefix}/conv_expand/kernel"].float()[0, 0].contiguous()       # (rd, C): TF layout as is
        return wr, self._vec(f"{prefix}/conv_reduce/bias"), we, self._vec(f"{prefix}/conv_expand/bias")

    def _compile(self):
        c = self.cfg
        P = {"blocks": []}
        P["stem"] = self._folded_conv("conv_stem", "bn1")
        for b in self.blocks:
            p, d = b.name, {}
            if b.kind == "ir":
                d["pw"] = self._folded_conv(f"{p}/conv_pw", f"{p}/bn1")
                d["dw"] = self._folded_dw(f"{p}/conv_dw", f"{p}/bn2")
                d["pwl"] = self._folded_conv(f"{p}/conv_pwl", f"{p}/bn3")
            elif b.kind == "ds":
                d["dw"] = self._folded_dw(f"{p}/conv_dw", f"{p}/bn1")
                d["pw"] = self._folded_conv(f"{p}/conv_pw", f"{p}/bn2")
            elif b.kind == "er":
                d["exp"] = self._folded_conv(f"{p}/conv_exp", f"{p}/bn1")
                d["pwl"] = self._folded_conv(f"{p}/conv_pwl", f"{p}/bn2")
            else:
                d["conv"] = self._folded_conv(f"{p}/conv", f"{p}/bn1")
            if b.se_rd:
                d["se"] = self._se_weights(f"{p}/se")
            P["blocks"].append(d)
        P["head"] = self._folded_conv("conv_head", "bn2")
        if c.nb_classes > 0:
            P["cls_w"] = self._dense_weight("classifier/kernel")
            P["cls_b"] = self._vec("classifier/bias")
        return P

    # ------------------------------------------------------------------ forward
    def _dense_conv(self, x, wb, k, stride, act, residual=None, gate=None):
        """k x k dense conv (+folded BN, +act, +residual) on (B,H,W,C) -> (B,Ho,Wo,Cout).  ``gate`` (B, C): squeeze-excite
        gate of a 1 x 1 projection's input, applied inside the GEMM (ops.gemm_gated)."""
        w, bias = wb
        B = x.shape[0]
        if k == 1 and stride == 1:
            cols, Ho, Wo = x.reshape(-1, x.shape[-1]), x.shape[1], x.shape[2]
        else:
            # raw uint8 pixels (stem): create_preprocessing is fused into the gather
            pre = self._pixel_stats(x.device) if x.dtype == torch.uint8 else None
            cols, Ho, Wo = ops.im2col(x, k, stride, self.cfg.padding, self.act_dtype, pre=pre)
        res2d = residual.reshape(-1, residual.shape[-1]) if residual is not None else None
        if gate is not None:
            y = ops.gemm_gated(cols, gate, Ho * Wo, w, bias=bias, act=act, residual=res2d)
        else:
            y = ops.gemm(cols, w, bias=bias, act=act, residual=res2d)
        return y.view(B, Ho, Wo, w.shape[0])

    def _se_gate(self, x, se, act, pooled_sum=None):
        """SEModule up to the sigmoid: (B, C) fp32 gate.  bf16 models hand it to the projection GEMM; fp32 models scale
        ``x`` in place (the fp32 GEMM has no gated form)."""
        B, H, W, C = x.shape
        if pooled_sum is None:
            return ops.se_gate(ops.global_avg_pool(x), 1, *se, act=act, gate_act="sigmoid")  # already a mean
        return ops.se_gate(pooled_sum, H * W, *se, act=act, gate_act="sigmoid")

    def _project(self, h, wb, act, shortcut, gate):
        """1 x 1 projection after the (optional) squeeze-excite gate.  With >= 256 pixels per image the gate is applied
        inside the GEMM.  Small feature maps (a 128-row tile spans several images) keep the separate pass."""
        if gate is not None and (h.dtype != torch.bfloat16 or h.shape[1] * h.shape[2] < 256):
            h, gate = ops.scale_channels_(h, gate), None
        return self._dense_conv(h, wb, 1, 1, act, residual=shortcut, gate=gate)

    def _block(self, x, b: BlockSpec, d):
        pad = self.cfg.padding
        shortcut = x if b.skip else None
        B = x.shape[0]
        if b.kind == "ir":
            h = self._dense_conv(x, d["pw"], 1, 1, b.act)
            pool = torch.zeros((B, b.c_mid), device=x.device, dtype=torch.float32) if b.se_rd else None
            h = ops.dwconv_bias_act(h, *d["dw"], b.kernel, b.stride, pad, act=b.act, pool_sum=pool)
            gate = self._se_gate(h, d["se"], b.act, pool) if b.se_rd else None
            return self._project(h, d["pwl"], None, shortcut, gate)
        if b.kind == "ds":
            pool = torch.zeros((B, b.c_in), device=x.device, dtype=torch.float32) if b.se_rd else None
            h = ops.dwconv_bias_act(x, *d["dw"], b.kernel, b.stride, pad, act=b.act, pool_sum=pool)
            gate = self._se_gate(h, d["se"], b.act, pool) if b.se_rd else None
            return self._project(h, d["pw"], b.act if b.pw_act else None, shortcut, gate)
        if b.kind == "er":
            h = self._dense_conv(x, d["exp"], b.kernel, b.stride, b.act)
            gate = self._se_gate(h, d["se"], b.act) if b.se_rd else None
            return self._project(h, d["pwl"], None, shortcut, gate)
        return self._dense_conv(x, d["conv"], b.kernel, b.stride, b.act, residual=shortcut)

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        features = OrderedDict()
        x = self._dense_conv(x, P["stem"], 3, 2, c.act_layer)
        features["stem"] = x
        for b, d in zip(self.blocks, P["blocks"]):
            x = self._block(x, b, d)
            features[b.key] = x
        x = self._dense_conv(x, P["head"], 1, 1, c.act_layer)
        features["conv_features"] = x
        return (x, features) if return_features else x

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        features = OrderedDict()
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        x = ops.global_avg_pool(x)
        features["features"] = x
        if c.nb_classes > 0:
            x = ops.gemm(ops.cast(x, self.act_dtype), P["cls_w"], bias=P["cls_b"], out_dtype=torch.float32)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "efficientnet", EfficientNet, EfficientNetConfig)
