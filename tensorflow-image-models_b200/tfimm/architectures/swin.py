"""Swin Transformer forward path as a chain of sm_90a kernels.

What the reference computes (tfimm/architectures/swin.py): PatchEmbeddings(k = s = 4) + LN -> 4 stages of
SwinTransformerBlocks [LN -> roll(-s) -> window_partition -> WindowAttention(+rel-pos bias, +shift mask)
-> window_reverse -> roll(+s) -> residual; LN -> MLP -> residual] with PatchMerging between stages ->
LN -> mean over tokens -> head.                                          [swin.py:159-198, 287-327, 348-362, 488-517]

How it runs here: tokens stay in raster order for the whole network.  The two rolls, the partition
and the reverse are row permutations, so they are folded into a row-index table consumed by the
window-attention kernel (gather q/k/v rows, scatter output rows); the shift mask is regenerated
from per-token region labels; PatchMerging's strided gather + concat is fused with its LayerNorm.
GEMMs (qkv / proj / fc1 / fc2 / reduction / head) run on wgmma with bias / GELU / residual epilogues.
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np
import torch

from ..backend import ops
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["SwinTransformer", "SwinTransformerConfig"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}


@dataclass
class SwinTransformerConfig(ModelConfig):
    """Same fields and defaults as the reference's ``SwinTransformerConfig`` (swin.py:28-69)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_size: int = 4
    embed_dim: int = 96
    nb_blocks: Tuple = (2, 2, 6, 2)
    nb_heads: Tuple = (3, 6, 12, 24)
    window_size: int = 7
    mlp_ratio: float = 4.0
    qkv_bias: bool = True
    drop_rate: float = 0.0
    attn_drop_rate: float = 0.0
    drop_path_rate: float = 0.1
    norm_layer: str = "layer_norm"
    act_layer: str = "gelu"
    patch_norm: bool = True
    interpolate_input: bool = False
    crop_pct: float = 0.9
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "patch_embed/proj"
    classifier: str = "head"

    @property
    def patch_resolution(self):
        return (self.input_size[0] // self.patch_size, self.input_size[1] // self.patch_size)

    @property
    def nb_patches(self):
        return self.patch_resolution[0] * self.patch_resolution[1]


def relative_position_index(ws: int) -> np.ndarray:
    """(ws^2, ws^2) lookup into the (2ws-1)^2 bias table: entry [i, j] encodes the offset of token i
    from token j inside a window (swin.py:143-157)."""
    yy, xx = np.meshgrid(np.arange(ws), np.arange(ws), indexing="ij")
    flat = np.stack([yy.reshape(-1), xx.reshape(-1)])            # (2, n)
    rel = flat[:, :, None] - flat[:, None, :] + (ws - 1)          # (2, n, n), both in [0, 2ws-2]
    return (rel[0] * (2 * ws - 1) + rel[1]).astype(np.int64)


def window_tables(h: int, w: int, ws: int, shift: int):
    """Row map and region labels of one (shifted-)window layout.
    row_map[wi*n + p]: raster token index that lands at position p of window wi after roll(-shift) and
    window_partition (swin.py:299-303, 72-87); labels: the 9-region ids of swin.py:249-262 (None if
    shift == 0)."""
    sy, sx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")   # coordinates in the shifted frame
    src = ((sy + shift) % h) * w + ((sx + shift) % w)                 # roll(-s): y[i] = x[(i+s) % n]

    def partition(a):
        return a.reshape(h // ws, ws, w // ws, ws).transpose(0, 2, 1, 3).reshape(-1)

    row_map = partition(src).astype(np.int32)
    labels = None
    if shift > 0:
        def region(coord, size):
            return np.where(coord < size - ws, 0, np.where(coord < size - shift, 1, 2))

        labels = partition(3 * region(sy, h) + region(sx, w)).astype(np.int32)
    return row_map, labels


class SwinTransformer(Model):
    cfg_class = SwinTransformerConfig
    accepts_uint8 = True

    def __init__(self, cfg: SwinTransformerConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = SwinTransformerConfig(**cfg)
        if cfg.norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)
        super().__init__(cfg, *args, **kwargs)

    # ------------------------------------------------------------------ geometry
    def _stage_geometry(self):
        """Per stage: (h, w, dim, heads, [(window, shift) per block]) with the reference's clamp
        (swin.py:219-223): if min(input_size) <= window_size then shift = 0, window = min(input_size)."""
        c = self.cfg
        out = []
        for i, depth in enumerate(c.nb_blocks):
            h, w = c.patch_resolution[0] // 2 ** i, c.patch_resolution[1] // 2 ** i
            blocks = []
            for j in range(depth):
                ws, shift = c.window_size, (0 if j % 2 == 0 else c.window_size // 2)
                if min(h, w) <= ws:
                    ws, shift = min(h, w), 0
                blocks.append((ws, shift))
            out.append((h, w, int(c.embed_dim * 2 ** i), c.nb_heads[i], blocks))
        return out

    @property
    def keys_to_ignore_on_load_missing(self) -> List[str]:
        names = []
        for i, depth in enumerate(self.cfg.nb_blocks):
            for j in range(depth):
                names.append(f"layers/{i}/blocks/{j}/attn_mask")
                names.append(f"layers/{i}/blocks/{j}/attn/relative_position_index")
        return names

    @property
    def feature_names(self) -> List[str]:
        names = ["patch_embedding"]
        k = 0
        for j, depth in enumerate(self.cfg.nb_blocks):
            for _ in range(depth):
                names.append(f"block_{k}")
                k += 1
            names.append(f"stage_{j}")
        return names + ["features_all", "features", "logits"]

    # ------------------------------------------------------------------ parameters
    def _param_specs(self):
        c = self.cfg
        s = OrderedDict()

        def dense(prefix, n_in, n_out, bias=True):
            s[f"{prefix}/kernel"] = ParamSpec((n_in, n_out), "glorot_uniform")
            if bias:
                s[f"{prefix}/bias"] = ParamSpec((n_out,), "zeros")

        def norm(prefix, n):
            s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
            s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

        s["patch_embed/proj/kernel"] = ParamSpec((c.patch_size, c.patch_size, c.in_channels, c.embed_dim), "glorot_uniform")
        s["patch_embed/proj/bias"] = ParamSpec((c.embed_dim,), "zeros")
        if c.patch_norm:
            norm("patch_embed/norm", c.embed_dim)
        n_tab = (2 * c.window_size - 1) ** 2
        n_win = c.window_size ** 2
        nb_stages = len(c.nb_blocks)
        for i, (h, w, dim, heads, blocks) in enumerate(self._stage_geometry()):
            for j, (ws, shift) in enumerate(blocks):
                p = f"layers/{i}/blocks/{j}"
                norm(f"{p}/norm1", dim)
                dense(f"{p}/attn/qkv", dim, 3 * dim, bias=c.qkv_bias)
                dense(f"{p}/attn/proj", dim, dim)
                s[f"{p}/attn/relative_position_bias_table"] = ParamSpec((n_tab, heads), "zeros")
                s[f"{p}/attn/relative_position_index"] = ParamSpec((n_win, n_win), "zeros", trainable=False)
                mask_shape = ((h // ws) * (w // ws), ws * ws, ws * ws) if shift > 0 else (1,)
                s[f"{p}/attn_mask"] = ParamSpec(mask_shape, "zeros", trainable=False)
                norm(f"{p}/norm2", dim)
                dense(f"{p}/mlp/fc1", dim, int(dim * c.mlp_ratio))
                dense(f"{p}/mlp/fc2", int(dim * c.mlp_ratio), dim)
            if i < nb_stages - 1:
                norm(f"layers/{i}/downsample/norm", 4 * dim)
                dense(f"layers/{i}/downsample/reduction", 4 * dim, 2 * dim, bias=False)
        norm("norm", int(c.embed_dim * 2 ** (nb_stages - 1)))
        if c.nb_classes > 0:
            dense("head", int(c.embed_dim * 2 ** (nb_stages - 1)), c.nb_classes)
        return s

    def _build(self):
        super()._build()
        if self.device.type == "meta":
            return
        c = self.cfg
        index = torch.from_numpy(relative_position_index(c.window_size))
        for i, (h, w, dim, heads, blocks) in enumerate(self._stage_geometry()):
            for j, (ws, shift) in enumerate(blocks):
                p = f"layers/{i}/blocks/{j}"
                self.params[f"{p}/attn/relative_position_index"] = index.to(self.device)
                if shift > 0:
                    _, labels = window_tables(h, w, ws, shift)
                    lab = torch.from_numpy(labels).view(-1, ws * ws)
                    mask = torch.where(lab[:, None, :] != lab[:, :, None], -100.0, 0.0).float()
                    self.params[f"{p}/attn_mask"] = mask.to(self.device)

    def load_weights_dict(self, weights, strict=True):
        ignore = set(self.keys_to_ignore_on_load_missing)
        weights = {k: v for k, v in weights.items() if k not in ignore}
        super().load_weights_dict(weights, strict=strict)

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        dev = self.device
        P = {"eps": _LN_EPS[c.norm_layer], "stages": []}
        P["pe_w"] = self._dense_weight("patch_embed/proj/kernel")
        P["pe_b"] = self._vec("patch_embed/proj/bias")
        P["pe_n"] = (self._vec("patch_embed/norm/gamma"), self._vec("patch_embed/norm/beta")) if c.patch_norm else None
        index = torch.from_numpy(relative_position_index(c.window_size)).to(dev).reshape(-1)
        nb_stages = len(c.nb_blocks)
        for i, (h, w, dim, heads, blocks) in enumerate(self._stage_geometry()):
            st = {"h": h, "w": w, "dim": dim, "heads": heads, "blocks": []}
            tables = {}
            for j, (ws, shift) in enumerate(blocks):
                if ws != c.window_size:
                    # the reference's bias reshape (swin.py:179-182) needs window_size**2 tokens per window
                    raise ValueError(f"Stage {i} resolution {(h, w)} is smaller than window_size={c.window_size}.")
                p = f"layers/{i}/blocks/{j}"
                if (ws, shift) not in tables:
                    row_map, labels = window_tables(h, w, ws, shift)
                    mask = None
                    if labels is not None:
                        lab = torch.from_numpy(labels).view(-1, ws * ws)
                        mask = torch.where(lab[:, None, :] != lab[:, :, None], -100.0, 0.0).float().contiguous().to(dev)
                    bits = None
                    if labels is not None and ws * ws <= 52:
                        # bit j of (window w, token i): tokens i and j lie in different shift regions (the -100 entries)
                        diff = (lab[:, :, None] != lab[:, None, :]).to(torch.int64)              # (nW, n, n)
                        packed = (diff << torch.arange(ws * ws, dtype=torch.int64)[None, None, :]).sum(dim=-1)
                        bits = torch.zeros((lab.shape[0], 64), dtype=torch.int64)
                        bits[:, :ws * ws] = packed
                        bits = bits.contiguous().to(dev)
                    tables[(ws, shift)] = (
                        torch.from_numpy(row_map).to(dev),
                        torch.from_numpy(labels).to(dev) if labels is not None else None,
                        mask,
                        bits,
                    )
                n = ws * ws
                table = self.params[f"{p}/attn/relative_position_bias_table"].float()
                bias = table[index].view(n, n, heads).permute(2, 0, 1).contiguous()  # tf.gather + transpose
                bias_pad = None
                if n <= 52:  # padded-table window-attention entry: 16-byte aligned rows of 64
                    bias_pad = torch.zeros((heads, 64, 64), device=dev, dtype=torch.float32)
                    bias_pad[:, :n, :n] = bias
                st["blocks"].append(dict(
                    ws=ws, shift=shift, tables=tables[(ws, shift)], bias=bias, bias_pad=bias_pad,
                    n1=(self._vec(f"{p}/norm1/gamma"), self._vec(f"{p}/norm1/beta")),
                    qkv_w=self._dense_weight(f"{p}/attn/qkv/kernel"),
                    qkv_b=self._vec(f"{p}/attn/qkv/bias") if c.qkv_bias else None,
                    proj_w=self._dense_weight(f"{p}/attn/proj/kernel"),
                    proj_b=self._vec(f"{p}/attn/proj/bias"),
                    n2=(self._vec(f"{p}/norm2/gamma"), self._vec(f"{p}/norm2/beta")),
                    fc1_w=self._dense_weight(f"{p}/mlp/fc1/kernel"),
                    fc1_b=self._vec(f"{p}/mlp/fc1/bias"),
                    fc2_w=self._dense_weight(f"{p}/mlp/fc2/kernel"),
                    fc2_b=self._vec(f"{p}/mlp/fc2/bias"),
                ))
            if i < nb_stages - 1:
                q = f"layers/{i}/downsample"
                st["ds_n"] = (self._vec(f"{q}/norm/gamma"), self._vec(f"{q}/norm/beta"))
                st["ds_w"] = self._dense_weight(f"{q}/reduction/kernel")
            P["stages"].append(st)
        P["norm"] = (self._vec("norm/gamma"), self._vec("norm/beta"))
        if c.nb_classes > 0:
            P["head_w"] = self._dense_weight("head/kernel")
            P["head_b"] = self._vec("head/bias")
        return P

    # ------------------------------------------------------------------ forward
    def _window_attention(self, qkv, blk, B, nw, n, heads, dh):
        row_map, labels, mask, bits = blk["tables"]
        scale = dh ** -0.5
        if qkv.dtype == torch.bfloat16 and dh == 32 and n <= 52:
            return ops.window_attention_tc(qkv, blk["bias_pad"], row_map, bits, B, nw, n, heads, dh, scale)
        if qkv.dtype == torch.bfloat16 and dh == 32 and n <= 144:
            # mma.sync kernel: 8 x 8 windows, and the 12 x 12 windows of the *_window12_384 models
            return ops.window_attention(qkv, blk["bias"], row_map, labels, B, nw, n, heads, dh, scale)
        # generic path: fp32 SIMT kernel (precision="fp32", other head dims, windows larger than 144 tokens)
        out = ops.attention(ops.cast(qkv, torch.float32), B * nw, n, heads, dh, scale, bias=blk["bias"], mask=mask,
                            row_map=row_map, nw_img=nw)
        return ops.cast(out, qkv.dtype)

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        if tuple(x.shape[1:3]) != tuple(c.input_size):
            raise ValueError(f"Swin needs the input size it was built for {tuple(c.input_size)}, got {tuple(x.shape[1:3])}.")
        features = OrderedDict()
        B = x.shape[0]
        adt, rdt, eps = self.act_dtype, torch.float32, P["eps"]
        patches = self._patchify(x, c.patch_size)
        y = ops.gemm(patches, P["pe_w"], bias=P["pe_b"])
        xs = ops.layernorm(y, *P["pe_n"], eps, rdt) if P["pe_n"] is not None else ops.cast(y, rdt)
        if return_features:
            features["patch_embedding"] = xs.view(B, -1, c.embed_dim).clone()
        block_idx = 0
        for i, st in enumerate(P["stages"]):
            h, w, dim, heads = st["h"], st["w"], st["dim"], st["heads"]
            dh = dim // heads
            for blk in st["blocks"]:
                ws = blk["ws"]
                nw, n = (h // ws) * (w // ws), ws * ws
                t = ops.layernorm(xs, *blk["n1"], eps, adt)
                qkv = ops.gemm(t, blk["qkv_w"], bias=blk["qkv_b"])
                a = self._window_attention(qkv, blk, B, nw, n, heads, dh)
                ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], residual=xs, out=xs)
                t = ops.layernorm(xs, *blk["n2"], eps, adt)
                if adt == torch.bfloat16 and ops.mlp_fused_supported(dim, blk["fc1_w"].shape[0]):
                    # one kernel: the (M, 4 dim) hidden activations stay on the SM (csrc/mlp_sm90.cu)
                    ops.mlp_fused(t, blk["fc1_w"], blk["fc1_b"], blk["fc2_w"], blk["fc2_b"], c.act_layer, residual=xs,
                                  out=xs)
                else:
                    hid = ops.gemm(t, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
                    ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], residual=xs, out=xs)
                if return_features:
                    features[f"block_{block_idx}"] = xs.view(B, h * w, dim).clone()
                block_idx += 1
            if "ds_w" in st:
                cols = ops.patch_merge_ln(xs.view(B, h, w, dim), *st["ds_n"], eps, adt)
                xs = ops.gemm(cols, st["ds_w"], out_dtype=rdt)
            if return_features:
                features[f"stage_{i}"] = xs.view(B, -1, xs.shape[1]).clone()
        full = ops.layernorm(xs, *P["norm"], eps, torch.float32)
        features["features_all"] = full.view(B, -1, full.shape[1])
        out = ops.global_avg_pool(features["features_all"])
        features["features"] = out
        return (out, features) if return_features else out

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        features = {}
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        if c.nb_classes > 0:
            x = ops.gemm(ops.cast(x, self.act_dtype), P["head_w"], bias=P["head_b"], out_dtype=torch.float32)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "swin", SwinTransformer, SwinTransformerConfig)
