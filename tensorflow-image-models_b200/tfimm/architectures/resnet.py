"""ResNet / ResNeXt / SE-ResNet / ECA-ResNet forward path as a chain of sm_90a kernels.

What the reference computes (tfimm/architectures/resnet.py): stem (7x7/s2 conv or three 3x3 convs) + BN
+ ReLU -> 3x3/s2 max-pool (or conv) -> 4 stages of BasicBlock / Bottleneck with projection shortcuts
(conv or avg-pool + 1x1) -> global average pool -> Dense.          [resnet.py:166-189, 266-292, 295-382, 466-593]

How it runs here (BatchNorm folded into the preceding conv at load time):
  1x1 convs                   wgmma GEMM; the last conv of a block adds the shortcut and applies the
                              ReLU in its epilogue (act_after_residual)
  3x3 / 7x7 dense convs       im2col gather + wgmma GEMM
  grouped 3x3 (ResNeXt)       CUDA-core grouped-conv kernel (4..32 channels per group)
  SE / ECA                    pool + tiny gate kernel, then one fused  x = relu(x * gate + shortcut)  pass
Not implemented (raise at construction): BlurPool anti-aliasing (1 registration), GroupNorm (1), groups
wider than 32 channels (resnext 32x8d and wider).
"""
import math
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

from ..backend import ops
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD, make_divisible
from ._zoo import register_zoo

__all__ = ["ResNet", "ResNetConfig"]

_BN_EPS = {"batch_norm": 1e-5, "batch_norm_tf": 1e-3}
_GN_GROUPS = {"group_norm": 32, "group_norm_1grp": 1}  # norm_layer_factory, tfimm/layers/factory.py:49-56; eps 1e-5


@dataclass
class ResNetConfig(ModelConfig):
    """Same fields and defaults as the reference's ``ResNetConfig`` (resnet.py:55-99)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    block: str = "basic_block"
    nb_blocks: Tuple = (2, 2, 2, 2)
    nb_channels: Tuple = (64, 128, 256, 512)
    cardinality: int = 1
    base_width: int = 64
    downsample_mode: str = "conv"
    zero_init_last_bn: bool = True
    stem_width: int = 64
    stem_type: str = ""
    replace_stem_pool: bool = False
    block_reduce_first: int = 1
    down_kernel_size: int = 1
    act_layer: str = "relu"
    norm_layer: str = "batch_norm"
    aa_layer: str = ""
    attn_layer: str = ""
    se_ratio: float = 0.0625
    drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    global_pool: str = "avg"
    test_input_size: Optional[Tuple[int, int]] = None
    pool_size: int = 7
    crop_pct: float = 0.875
    interpolation: str = "bilinear"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "conv1"
    classifier: str = "fc"

    def __post_init__(self):
        if self.test_input_size is None:
            self.test_input_size = self.input_size


@dataclass
class _Block:
    name: str          # "layer{i}/{b}"
    c_in: int
    mid1: int          # channels after conv1
    width: int         # channels after conv2 (== out for basic blocks)
    c_out: int
    stride: int
    groups: int
    shortcut: str      # "" | "conv" | "avg"
    attn: str          # "" | "se" | "eca"
    attn_width: int    # SE squeeze width or ECA kernel size


def eca_kernel_size(channels: int, gamma: int = 2, beta: int = 1) -> int:
    """EcaModule.build, tfimm/layers/attention.py:107-110."""
    t = int(abs(math.log(channels, 2) + beta) / gamma)
    return max(t if t % 2 else t + 1, 3)


def resolve_blocks(cfg: ResNetConfig) -> List[_Block]:
    """make_stage (resnet.py:333-382) for all four stages, plus the widths the blocks derive."""
    if cfg.block not in ("basic_block", "bottleneck"):
        raise ValueError(f"Unknown block {cfg.block}")
    expansion = 1 if cfg.block == "basic_block" else 4
    real_in = cfg.stem_width * 2 if cfg.stem_type in ("deep", "deep_tiered") else 64
    ref_in = real_in  # the `in_channels` bookkeeping variable of make_stage (only feeds the projection test)
    out = []
    for i in range(4):
        ch = cfg.nb_channels[i]
        c_out = ch * expansion
        for b in range(cfg.nb_blocks[i]):
            stride = 1 if (i == 0 or b > 0) else 2
            needs_proj = b == 0 and (stride != 1 or ref_in != c_out)
            in_ch = real_in
            if cfg.block == "basic_block":
                mid1, width, groups = ch // cfg.block_reduce_first, c_out, 1
            else:
                width = int(math.floor(ch * (cfg.base_width / 64)) * cfg.cardinality)
                mid1, groups = width // cfg.block_reduce_first, cfg.cardinality
            if cfg.attn_layer == "se":
                aw = make_divisible(c_out * cfg.se_ratio, 8, round_limit=0.0)
            elif cfg.attn_layer == "eca":
                aw = eca_kernel_size(c_out)
            else:
                aw = 0
            out.append(_Block(f"layer{i + 1}/{b}", in_ch, mid1, width, c_out, stride, groups,
                              cfg.downsample_mode if needs_proj else "", cfg.attn_layer, aw))
            # The reference carries `nb_channels`, not `out_channels`, into the next projection test
            # (resnet.py:379); the convolutions themselves see the real channel count.
            ref_in = ch
            real_in = c_out
    return out


class ResNet(Model):
    cfg_class = ResNetConfig
    accepts_uint8 = True   # raw pixels: create_preprocessing fused into the stem's im2col gather
    keys_to_ignore_on_load_missing = ["blur_kernel"]

    def __init__(self, cfg: ResNetConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = ResNetConfig(**cfg)
        if cfg.norm_layer not in _BN_EPS and cfg.norm_layer not in _GN_GROUPS:
            raise NotImplementedError(f"norm_layer={cfg.norm_layer} is not implemented in this engine.")
        if cfg.aa_layer not in ("", "blur_pool"):
            raise ValueError(f"Unknown anti-aliasing layer {cfg.aa_layer}")
        if cfg.attn_layer not in ("", "se", "eca"):
            raise ValueError(f"Unknown attention layer {cfg.attn_layer}")
        if cfg.global_pool != "avg":
            raise NotImplementedError("Only global average pooling is implemented.")
        if cfg.downsample_mode not in ("avg", "conv"):
            raise ValueError(f"Unknown downsample mode {cfg.downsample_mode}")
        ops.act_code(cfg.act_layer)
        self.blocks = resolve_blocks(cfg)
        if cfg.norm_layer in _GN_GROUPS and cfg.cardinality > 1:
            raise NotImplementedError("GroupNorm with grouped convolutions is not implemented (no registration uses it).")
        super().__init__(cfg, *args, **kwargs)

    # ------------------------------------------------------------------ parameters
    def _stem_layout(self):
        c = self.cfg
        if c.stem_type in ("deep", "deep_tiered"):
            first = 3 * (c.stem_width // 4) if c.stem_type == "deep_tiered" else c.stem_width
            return [("conv1/0", 3, c.in_channels, first, "conv1/1"),
                    ("conv1/3", 3, first, c.stem_width, "conv1/4"),
                    ("conv1/6", 3, c.stem_width, c.stem_width * 2, "bn1")]
        return [("conv1", 7, c.in_channels, 64, "bn1")]

    def _param_specs(self):
        c = self.cfg
        s = OrderedDict()

        def conv(prefix, k, cin, cout, bias=False):
            s[f"{prefix}/kernel"] = ParamSpec((k, k, cin, cout), "glorot_uniform")
            if bias:
                s[f"{prefix}/bias"] = ParamSpec((cout,), "zeros")

        def bn(prefix, ch, last=False):
            zero = last and c.zero_init_last_bn
            s[f"{prefix}/gamma"] = ParamSpec((ch,), "zeros" if zero else "ones")
            s[f"{prefix}/beta"] = ParamSpec((ch,), "zeros")
            if c.norm_layer in _GN_GROUPS:
                return
            s[f"{prefix}/moving_mean"] = ParamSpec((ch,), "zeros", trainable=False)
            s[f"{prefix}/moving_variance"] = ParamSpec((ch,), "zeros" if zero else "ones", trainable=False)

        for name, k, cin, cout, bn_name in self._stem_layout():
            conv(name, k, cin, cout)
            bn(bn_name, cout)
        stem_out = self._stem_layout()[-1][3]
        if c.replace_stem_pool:
            conv("maxpool/0", 3, stem_out, stem_out)
            bn("maxpool/1", stem_out)
        for b in self.blocks:
            p = b.name
            if c.block == "basic_block":
                conv(f"{p}/conv1", 3, b.c_in, b.mid1)
                bn(f"{p}/bn1", b.mid1)
                conv(f"{p}/conv2", 3, b.mid1, b.c_out)
                bn(f"{p}/bn2", b.c_out, last=True)
            else:
                conv(f"{p}/conv1", 1, b.c_in, b.mid1)
                bn(f"{p}/bn1", b.mid1)
                conv(f"{p}/conv2", 3, b.mid1 // b.groups, b.width)
                bn(f"{p}/bn2", b.width)
                conv(f"{p}/conv3", 1, b.width, b.c_out)
                bn(f"{p}/bn3", b.c_out, last=True)
            if b.attn == "se":
                conv(f"{p}/se/fc1", 1, b.c_out, b.attn_width, bias=True)
                conv(f"{p}/se/fc2", 1, b.attn_width, b.c_out, bias=True)
            elif b.attn == "eca":
                s[f"{p}/se/conv/kernel"] = ParamSpec((b.attn_width, 1, 1), "glorot_uniform")
            if b.shortcut == "conv":
                conv(f"{p}/downsample/0", c.down_kernel_size, b.c_in, b.c_out)
                bn(f"{p}/downsample/1", b.c_out)
            elif b.shortcut == "avg":
                conv(f"{p}/downsample/1", 1, b.c_in, b.c_out)
                bn(f"{p}/downsample/2", b.c_out)
        if c.nb_classes > 0:
            s["remove/fc/kernel"] = ParamSpec((self.blocks[-1].c_out, c.nb_classes), "glorot_uniform")
            s["remove/fc/bias"] = ParamSpec((c.nb_classes,), "zeros")
        return s

    # ------------------------------------------------------------------ engine plan (BN folded)
    def _bn_scale_shift(self, prefix):
        eps = _BN_EPS[self.cfg.norm_layer]
        g, b = self.params[f"{prefix}/gamma"].float(), self.params[f"{prefix}/beta"].float()
        m, v = self.params[f"{prefix}/moving_mean"].float(), self.params[f"{prefix}/moving_variance"].float()
        scale = g * torch.rsqrt(v + eps)
        return scale, b - m * scale

    def _folded_conv(self, conv_prefix, bn_prefix):
        """-> (W [out][K] in the activation dtype, bias or None, (gamma, beta) of a GroupNorm or None).
        BatchNorm (inference) is folded into W and the bias; GroupNorm needs the data and runs as its own kernel."""
        w = self.params[f"{conv_prefix}/kernel"].float()
        if self.cfg.norm_layer in _GN_GROUPS:
            shift, gn = None, (self._vec(f"{bn_prefix}/gamma"), self._vec(f"{bn_prefix}/beta"))
        else:
            scale, shift = self._bn_scale_shift(bn_prefix)
            w, shift, gn = w * scale, shift.contiguous(), None
        cout = w.shape[-1]
        w2 = w.reshape(-1, cout).t().contiguous()
        K = w2.shape[1]
        Kpad = (K + 7) // 8 * 8
        if Kpad != K:
            w2 = torch.nn.functional.pad(w2, (0, Kpad - K))
        return self._gemm_operand(w2), shift, gn

    def _folded_grouped_wide(self, conv_prefix, bn_prefix, groups):
        """Grouped 3x3 with >= 48 channels per group: one [cg][Kpad] GEMM weight per group (see _grouped_wide)."""
        scale, shift = self._bn_scale_shift(bn_prefix)
        w = self.params[f"{conv_prefix}/kernel"].float() * scale        # (k, k, cg, C)
        k, _, cg, C = w.shape
        wg = w.reshape(k * k * cg, groups, C // groups).permute(1, 2, 0)  # (G, cg_out, k*k*cg)
        Kpad = (k * k * cg + 7) // 8 * 8
        if Kpad != k * k * cg:
            wg = torch.nn.functional.pad(wg, (0, Kpad - k * k * cg))
        return self._gemm_operand(wg), shift.contiguous()

    def _folded_grouped(self, conv_prefix, bn_prefix):
        scale, shift = self._bn_scale_shift(bn_prefix)
        w = self.params[f"{conv_prefix}/kernel"].float() * scale   # (k, k, cg, C)
        return w.reshape(-1, w.shape[2], w.shape[3]).contiguous(), shift.contiguous()

    def _compile(self):
        c = self.cfg
        P = {"stem": [], "blocks": []}
        for name, k, cin, cout, bn_name in self._stem_layout():
            P["stem"].append((k, self._folded_conv(name, bn_name)))
        if c.replace_stem_pool:
            P["pool_conv"] = self._folded_conv("maxpool/0", "maxpool/1")
        for b in self.blocks:
            p, d = b.name, {}
            d["conv1"] = self._folded_conv(f"{p}/conv1", f"{p}/bn1")
            if b.groups > 1 and b.width // b.groups in (4, 8, 16, 32):
                d["conv2g"] = self._folded_grouped(f"{p}/conv2", f"{p}/bn2")
            elif b.groups > 1:
                d["conv2w"] = self._folded_grouped_wide(f"{p}/conv2", f"{p}/bn2", b.groups)
            else:
                d["conv2"] = self._folded_conv(f"{p}/conv2", f"{p}/bn2")
            if c.block == "bottleneck":
                d["conv3"] = self._folded_conv(f"{p}/conv3", f"{p}/bn3")
            if b.attn == "se":
                d["se"] = (self.params[f"{p}/se/fc1/kernel"].float()[0, 0].t().contiguous(), self._vec(f"{p}/se/fc1/bias"),
                           self.params[f"{p}/se/fc2/kernel"].float()[0, 0].contiguous(), self._vec(f"{p}/se/fc2/bias"))
            elif b.attn == "eca":
                d["eca"] = self._vec(f"{p}/se/conv/kernel")
            if b.shortcut == "conv":
                d["proj"] = self._folded_conv(f"{p}/downsample/0", f"{p}/downsample/1")
            elif b.shortcut == "avg":
                d["proj"] = self._folded_conv(f"{p}/downsample/1", f"{p}/downsample/2")
            P["blocks"].append(d)
        if c.nb_classes > 0:
            P["fc_w"] = self._dense_weight("remove/fc/kernel")
            P["fc_b"] = self._vec("remove/fc/bias")
        return P

    # ------------------------------------------------------------------ forward
    def _conv(self, x, wb, k, stride, pad, act, residual=None, act_after_residual=False):
        w, bias, gn = wb
        B = x.shape[0]
        if (k > 1 and gn is None and self.precision in ("bf16", "tf32") and isinstance(pad, int) and x.shape[-1] % 64 == 0
                and w.shape[1] == k * k * x.shape[-1]):
            # implicit GEMM: the A tiles are 4-D TMA boxes of the feature map, nothing is materialised
            return ops.conv_gemm(x, w, bias=bias, ks=k, stride=stride, pad=pad, act=act,
                                 residual=residual.contiguous() if residual is not None else None,
                                 act_after_residual=act_after_residual)
        if k == 1 and stride == 1:
            cols, Ho, Wo = x.reshape(-1, x.shape[-1]), x.shape[1], x.shape[2]
        else:
            # raw uint8 pixels (first stem conv): create_preprocessing is fused into the gather
            pre = self._pixel_stats(x.device) if x.dtype == torch.uint8 else None
            cols, Ho, Wo = ops.im2col(x, k, stride, pad, self.act_dtype, pre=pre)
        if gn is not None:
            # conv -> GroupNorm (-> + shortcut) -> act: the norm needs the whole (H, W, C/G) extent, so it cannot be
            # an epilogue of the GEMM tile; residual and activation ride on the normalisation pass instead
            assert residual is None or act_after_residual
            y = ops.gemm(cols, w).view(B, Ho, Wo, w.shape[0])
            return ops.group_norm(y, *gn, _GN_GROUPS[self.cfg.norm_layer], 1e-5, act=act,
                                  residual=residual.contiguous() if residual is not None else None)
        res2d = residual.reshape(-1, residual.shape[-1]) if residual is not None else None
        y = ops.gemm(cols, w, bias=bias, act=act, residual=res2d, act_after_residual=act_after_residual)
        return y.view(B, Ho, Wo, w.shape[0])

    def _grouped_wide(self, x, wb, b: _Block, stride, act):
        """Grouped 3x3 convolution with wide groups (ResNeXt 32x8d .. 32x48d: 48-384 channels per group): grouped
        im2col (one [M][9*cg] matrix per group) and one tensor-core GEMM per group, written straight into the
        group's column slice of the output.  Narrow groups (<= 32 channels) use the direct kernel instead."""
        wg, shift = wb
        G, cg = wg.shape[0], wg.shape[1]
        cols, Ho, Wo = ops.im2col(x, 3, stride, 1, self.act_dtype, groups=G)
        out = torch.empty((cols.shape[1], G * cg), device=x.device, dtype=self.act_dtype)
        for g in range(G):
            ops.gemm(cols[g], wg[g], bias=shift[g * cg:(g + 1) * cg], act=act, out=out[:, g * cg:(g + 1) * cg])
        return out.view(x.shape[0], Ho, Wo, G * cg)

    def _shortcut(self, x, b: _Block, d):
        c = self.cfg
        if b.shortcut == "conv":
            k = c.down_kernel_size
            return self._conv(x, d["proj"], k, b.stride, (b.stride + k) // 2 - 1, None)
        if b.shortcut == "avg":
            if b.stride != 1:
                x = ops.pool2d(x, 2, b.stride, "same", "avg")
            return self._conv(x, d["proj"], 1, 1, 0, None)
        return x

    def _block(self, x, b: _Block, d):
        c = self.cfg
        act = c.act_layer
        shortcut = self._shortcut(x, b, d)
        plain = b.attn == ""
        # anti-aliased variants: the strided conv runs at stride 1 and BlurPool2D takes the stride (resnet.py:127-140)
        use_aa = bool(c.aa_layer) and b.stride == 2
        cstride = 1 if use_aa else b.stride
        if c.block == "basic_block":
            h = self._conv(x, d["conv1"], 3, cstride, 1, act)
            if use_aa:
                h = ops.blur_pool(h, b.stride)
            h = self._conv(h, d["conv2"], 3, 1, 1, act if plain else None,
                           residual=shortcut if plain else None, act_after_residual=plain)
        else:
            h = self._conv(x, d["conv1"], 1, 1, 0, act)
            if "conv2g" in d:
                h = ops.grouped_conv(h, *d["conv2g"], b.width // b.groups, 3, cstride, 1, act=act)
            elif "conv2w" in d:
                h = self._grouped_wide(h, d["conv2w"], b, cstride, act)
            else:
                h = self._conv(h, d["conv2"], 3, cstride, 1, act)
            if use_aa:
                h = ops.blur_pool(h, b.stride)
            h = self._conv(h, d["conv3"], 1, 1, 0, act if plain else None,
                           residual=shortcut if plain else None, act_after_residual=plain)
        if not plain:
            mean = ops.global_avg_pool(h)
            gate = ops.se_gate(mean, 1, *d["se"], act="relu", gate_act="sigmoid") if b.attn == "se" \
                else ops.eca_gate(mean, d["eca"])
            h = ops.scale_add_act_(h, gate, shortcut.contiguous(), act)
        return h

    @property
    def feature_names(self) -> List[str]:
        return ["stem"] + [f"block_{j}" for j in range(sum(self.cfg.nb_blocks))] + ["features", "logits"]

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        features = OrderedDict()
        deep = c.stem_type in ("deep", "deep_tiered")
        for i, (k, wb) in enumerate(P["stem"]):
            if deep:
                x = self._conv(x, wb, 3, 2 if i == 0 else 1, 1 if i == 0 else "same", c.act_layer)
            else:
                x = self._conv(x, wb, 7, 2, 3, c.act_layer)
        if c.replace_stem_pool:
            x = self._conv(x, P["pool_conv"], 3, 2, 1, c.act_layer)
        elif c.aa_layer:  # ZeroPadding2D(1) + MaxPool2D(3, strides=1) + BlurPool2D(stride=2), resnet.py:532-536
            x = ops.blur_pool(ops.pool2d(x, 3, 1, 1, "max_zero_pad"), 2)
        else:
            x = ops.pool2d(x, 3, 2, 1, "max_zero_pad")
        features["stem"] = x
        for j, (b, d) in enumerate(zip(self.blocks, P["blocks"])):
            x = self._block(x, b, d)
            features[f"block_{j}"] = x
        features["features"] = x
        return (x, features) if return_features else x

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        features = {}
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        x = ops.global_avg_pool(x)
        if c.nb_classes > 0:
            x = ops.gemm(ops.cast(x, self.act_dtype), P["fc_w"], bias=P["fc_b"], out_dtype=torch.float32)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "resnet", ResNet, ResNetConfig)
