"""CaiT (class-attention image transformers) forward path as a chain of sm_90a kernels.

Registered on import (``import tfimm.architectures.cait``, module name ``cait``); ``import tfimm`` alone does not
import it.

What the reference computes (tfimm/architectures/cait.py):
  embed   Conv2D(embed_dim, patch_size / patch_size, VALID) + pos_embed (1, N, D), no class-token row (resized
          bicubically on the grid with interpolate_input)                                          (cait.py:391-405)
  SA      nb_blocks LayerScale blocks on the N patch tokens: x += gamma_1 proj(TH(norm1(x))), x += gamma_2 mlp(norm2(x));
          TH is talking-heads attention: S_h = dh^-0.5 q_h k_h^T, L = proj_l over the head axis, softmax over keys,
          P' = proj_w over the head axis, O_f = P'_f V_f                                           (cait.py:207-314)
  cls     the class token prepended, then two class-attention blocks that change row 0 only: u = norm1(x) over all
          rows, q from u[:, 0], k / v from u, one softmax per head; x_cls += gamma_1 proj(.), then
          x_cls += gamma_2 mlp(norm2(x_cls))                                                       (cait.py:97-204)
  head    norm over all rows = features_all, row 0 = features, head                                (cait.py:411-433)

How it runs here (fp32 residual stream in every precision):
  embed   im2col "valid" (uint8 pixels: the preprocessing fused in) -> GEMM + bias -> cait_ops.add_pos
  SA      layernorm -> qkv GEMM -> cait_ops.talking_heads (proj_l with dh^-0.5 log2 e folded into its kernel and log2 e
          into its bias) -> proj GEMM with gamma_1, + the stream in place -> layernorm -> MLP with gamma_2 (ops.mlp_fused
          where ops.mlp_fused_supported in bf16, else fc1 + GELU GEMM and fc2 GEMM) + the stream in place
  cls     ops.assemble_tokens prepends the class token into a new (B * (N + 1), D) stream; per class block: layernorm of
          all rows -> q GEMM on the row-strided class rows and one [k | v] GEMM on all rows -> cait_ops.class_attention
          -> proj GEMM with gamma_1 into the class rows -> layernorm and the MLP with gamma_2 on the class rows
  head    layernorm of the class rows (of all rows when features are returned) -> head GEMM
Talking heads: bf16 -> the mma.sync kernel (head dim 48, H in {4, 6, 8, 16}); fp32 and tf32 -> the fp32 SIMT kernel.
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import List, Tuple

import torch

from ..backend import cait_ops, ops
from ..layers.resize import tf_bicubic_resize
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD
from ._zoo import register_zoo

__all__ = ["CaiT", "CaiTConfig", "param_specs"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}


@dataclass
class CaiTConfig(ModelConfig):
    """Hyper-parameters (same fields and defaults as the reference's ``CaiTConfig``, cait.py:34-94)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_size: int = 16
    embed_dim: int = 768
    nb_blocks: int = 12
    nb_heads: int = 12
    mlp_ratio: float = 4.0
    qkv_bias: bool = True
    drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    attn_drop_rate: float = 0.0
    norm_layer: str = "layer_norm_eps_1e-6"
    act_layer: str = "gelu"
    init_scale: float = 1e-4
    interpolate_input: bool = False
    crop_pct: float = 1.0
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD
    first_conv: str = "patch_embed/proj"
    classifier: str = "head"

    @property
    def grid_size(self) -> Tuple[int, int]:
        return self.input_size[0] // self.patch_size, self.input_size[1] // self.patch_size

    @property
    def nb_patches(self) -> int:
        return self.grid_size[0] * self.grid_size[1]

    @property
    def transform_weights(self):
        return {"pos_embed": CaiT.transform_pos_embed}


def param_specs(c: CaiTConfig) -> "OrderedDict[str, ParamSpec]":
    """The reference's variables (names, shapes, initial values) in its order: the model's own cls_token and pos_embed
    (zeros), then the sub-layers in the order the model's __init__ assigns them, each layer's own variables before
    its sub-layers' -- so a block's gamma_1 / gamma_2 (Constant(init_scale)) come first, and the attention's qkv and
    proj precede proj_l and proj_w.  Keras' default initialisers otherwise (glorot_uniform kernels, zero biases,
    LayerNorm 1 / 0)."""
    s = OrderedDict()
    D = c.embed_dim
    hid = int(D * c.mlp_ratio)

    def dense(prefix, shape, bias=True):
        s[f"{prefix}/kernel"] = ParamSpec(shape, "glorot_uniform")
        if bias:
            s[f"{prefix}/bias"] = ParamSpec((shape[-1],), "zeros")

    def norm(prefix):
        s[f"{prefix}/gamma"] = ParamSpec((D,), "ones")
        s[f"{prefix}/beta"] = ParamSpec((D,), "zeros")

    def layer_scale(prefix):
        s[f"{prefix}/gamma_1"] = ParamSpec((D,), f"const:{c.init_scale!r}")
        s[f"{prefix}/gamma_2"] = ParamSpec((D,), f"const:{c.init_scale!r}")

    s["cls_token"] = ParamSpec((1, 1, D), "zeros")
    s["pos_embed"] = ParamSpec((1, c.nb_patches, D), "zeros")
    dense("patch_embed/proj", (c.patch_size, c.patch_size, c.in_channels, D))
    for j in range(c.nb_blocks):
        p = f"blocks/{j}"
        layer_scale(p)
        norm(f"{p}/norm1")
        dense(f"{p}/attn/qkv", (D, 3 * D), bias=c.qkv_bias)
        dense(f"{p}/attn/proj", (D, D))
        dense(f"{p}/attn/proj_l", (c.nb_heads, c.nb_heads))
        dense(f"{p}/attn/proj_w", (c.nb_heads, c.nb_heads))
        norm(f"{p}/norm2")
        dense(f"{p}/mlp/fc1", (D, hid))
        dense(f"{p}/mlp/fc2", (hid, D))
    for j in range(2):
        p = f"blocks_token_only/{j}"
        layer_scale(p)
        norm(f"{p}/norm1")
        dense(f"{p}/attn/q", (D, D), bias=c.qkv_bias)
        dense(f"{p}/attn/k", (D, D), bias=c.qkv_bias)
        dense(f"{p}/attn/v", (D, D), bias=c.qkv_bias)
        dense(f"{p}/attn/proj", (D, D))
        norm(f"{p}/norm2")
        dense(f"{p}/mlp/fc1", (D, hid))
        dense(f"{p}/mlp/fc2", (hid, D))
    norm("norm")
    if c.nb_classes > 0:
        dense("head", (D, c.nb_classes))
    return s


class CaiT(Model):
    cfg_class = CaiTConfig
    accepts_uint8 = True

    def __init__(self, cfg: CaiTConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = CaiTConfig(**cfg)
        if cfg.norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        if cfg.embed_dim % cfg.nb_heads:
            raise ValueError(f"embed_dim {cfg.embed_dim} is not a multiple of nb_heads {cfg.nb_heads}")
        dh = cfg.embed_dim // cfg.nb_heads
        precision = kwargs.get("precision", "bf16")
        if precision == "bf16" and not cait_ops.bf16_supported(cfg.nb_heads, dh):
            raise ValueError(f"no bf16 talking-heads kernel for nb_heads {cfg.nb_heads} at head_dim {dh} (have "
                             f"nb_heads in {cait_ops.BF16_HEADS} at head_dim {cait_ops.BF16_HEAD_DIM})")
        if precision != "bf16" and not cait_ops.f32_supported(cfg.nb_heads, dh):
            raise ValueError(f"no fp32 talking-heads kernel for nb_heads {cfg.nb_heads} at head_dim {dh} (have "
                             f"nb_heads in {cait_ops.F32_HEADS}, head_dim a multiple of 4 up to 64)")
        if dh not in cait_ops.CLS_HEAD_DIMS:
            raise ValueError(f"class attention needs head_dim in {cait_ops.CLS_HEAD_DIMS} (got {dh})")
        if int(cfg.embed_dim * cfg.mlp_ratio) % 8:
            raise ValueError(f"the kernels need the MLP width to be a multiple of 8 (mlp_ratio {cfg.mlp_ratio})")
        self.nb_features = cfg.embed_dim
        super().__init__(cfg, *args, **kwargs)

    def _param_specs(self):
        return param_specs(self.cfg)

    def transform_pos_embed(self, src_weights, target_cfg: CaiTConfig):
        """pos_embed resized bicubically on its grid to ``target_cfg``'s (cait.py:383-389, nb_tokens = 0)."""
        return self._resized_pos(self.params["pos_embed"], self.cfg.grid_size, target_cfg.grid_size)

    @staticmethod
    def _resized_pos(pos_embed, src, grid):
        """(1, N, D) pos_embed on grid ``src`` -> (1, gh * gw, D) on ``grid``."""
        if tuple(grid) == tuple(src):
            return pos_embed
        pos = tf_bicubic_resize(pos_embed.reshape(1, *src, -1), tuple(grid))
        return pos.reshape(1, grid[0] * grid[1], -1)

    @property
    def feature_names(self) -> List[str]:
        return (["patch_embedding"] + [f"block_{j}" for j in range(self.cfg.nb_blocks)] + ["features_cls_token"]
                + [f"block_cls_token_{j}" for j in range(2)] + ["features_all", "features", "logits"])

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        dh = c.embed_dim // c.nb_heads
        P = {"eps": _LN_EPS[c.norm_layer], "blocks": [], "cls_blocks": [], "pos": {}}
        P["pe_w"], P["pe_b"] = self._dense_weight("patch_embed/proj/kernel"), self._vec("patch_embed/proj/bias")
        P["cls"] = self.params["cls_token"].float().reshape(-1).contiguous()

        def opt_vec(key):
            return self._vec(key) if key in self.params else None

        def mlp(p):
            return dict(n2=(self._vec(f"{p}/norm2/gamma"), self._vec(f"{p}/norm2/beta")),
                        fc1_w=self._dense_weight(f"{p}/mlp/fc1/kernel"), fc1_b=self._vec(f"{p}/mlp/fc1/bias"),
                        fc2_w=self._dense_weight(f"{p}/mlp/fc2/kernel"), fc2_b=self._vec(f"{p}/mlp/fc2/bias"),
                        g1=self._vec(f"{p}/gamma_1"), g2=self._vec(f"{p}/gamma_2"),
                        n1=(self._vec(f"{p}/norm1/gamma"), self._vec(f"{p}/norm1/beta")),
                        proj_w=self._dense_weight(f"{p}/attn/proj/kernel"), proj_b=self._vec(f"{p}/attn/proj/bias"))

        for j in range(c.nb_blocks):
            p = f"blocks/{j}"
            blk = mlp(p)
            wl, bl = cait_ops.fold_premix(self.params[f"{p}/attn/proj_l/kernel"].float(),
                                          self.params[f"{p}/attn/proj_l/bias"].float(), dh)
            blk.update(qkv_w=self._dense_weight(f"{p}/attn/qkv/kernel"), qkv_b=opt_vec(f"{p}/attn/qkv/bias"),
                       wl=wl, bl=bl,
                       ww=self.params[f"{p}/attn/proj_w/kernel"].float().contiguous(),
                       bw=self._vec(f"{p}/attn/proj_w/bias"))
            P["blocks"].append(blk)
        for j in range(2):
            p = f"blocks_token_only/{j}"
            blk = mlp(p)
            kv_w = torch.cat((self.params[f"{p}/attn/k/kernel"], self.params[f"{p}/attn/v/kernel"]), dim=1)
            blk.update(q_w=self._dense_weight(f"{p}/attn/q/kernel"), q_b=opt_vec(f"{p}/attn/q/bias"),
                       kv_w=self._gemm_operand(kv_w.float().t().contiguous()))
            if c.qkv_bias:
                blk["kv_b"] = torch.cat((self._vec(f"{p}/attn/k/bias"), self._vec(f"{p}/attn/v/bias"))).contiguous()
            else:
                blk["kv_b"] = None
            P["cls_blocks"].append(blk)
        P["norm"] = (self._vec("norm/gamma"), self._vec("norm/beta"))
        if c.nb_classes > 0:
            P["head_w"], P["head_b"] = self._dense_weight("head/kernel"), self._vec("head/bias")
        return P

    def _pos_table(self, P, grid):
        """(gh * gw, D) fp32 pos_embed on ``grid``, and the zero (1 + gh * gw, D) table of the class-token prepend
        (built once per grid size)."""
        if grid not in P["pos"]:
            pos = self._resized_pos(self.params["pos_embed"].float(), self.cfg.grid_size, grid)[0].contiguous()
            zeros = torch.zeros((pos.shape[0] + 1, pos.shape[1]), dtype=torch.float32, device=pos.device)
            P["pos"][grid] = (pos, zeros)
        return P["pos"][grid]

    # ------------------------------------------------------------------ forward
    def _tokens(self, x, P):
        """Image batch -> (stream (B * N, D) fp32 with the position embedding, grid)."""
        c = self.cfg
        B, H, W, _ = x.shape
        if not c.interpolate_input and (H, W) != tuple(c.input_size):
            raise ValueError(f"Input size {(H, W)} does not match the model's {tuple(c.input_size)}; "
                             "create the model with interpolate_input=True to allow this.")
        if H < c.patch_size or W < c.patch_size:
            raise ValueError(f"Input size {(H, W)} is smaller than the patch size {c.patch_size}")
        pre = self._pixel_stats(x.device) if x.dtype == torch.uint8 else None
        cols, gh, gw = ops.im2col(x, c.patch_size, c.patch_size, "valid", self.act_dtype, pre=pre)
        tok = ops.gemm(cols, P["pe_w"], bias=P["pe_b"], out_dtype=torch.float32)
        if tok.stride(0) != tok.shape[1]:
            tok = tok.contiguous()
        cait_ops.add_pos(tok, self._pos_table(P, (gh, gw))[0], B, gh * gw)
        return tok, (gh, gw)

    def _mlp(self, blk, xs):
        """xs += gamma_2 mlp(norm2(xs)), in place; xs may be row-strided (the class rows)."""
        c = self.cfg
        adt = self.act_dtype
        h = ops.layernorm(xs, *blk["n2"], self._plan["eps"], adt)
        if adt == torch.bfloat16 and ops.mlp_fused_supported(c.embed_dim, blk["fc1_w"].shape[0]):
            # one kernel: the (M, 4D) hidden activations stay on the SM (csrc/mlp_sm90.cu)
            ops.mlp_fused(h, blk["fc1_w"], blk["fc1_b"], blk["fc2_w"], blk["fc2_b"], c.act_layer, gamma=blk["g2"],
                          residual=xs, out=xs)
        else:
            hid = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
            ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], gamma=blk["g2"], residual=xs, out=xs)

    def _block(self, blk, xs, B, N):
        c = self.cfg
        Hh, dh = c.nb_heads, c.embed_dim // c.nb_heads
        h = ops.layernorm(xs, *blk["n1"], self._plan["eps"], self.act_dtype)
        qkv = ops.gemm(h, blk["qkv_w"], bias=blk["qkv_b"])
        a = cait_ops.talking_heads(qkv, blk["wl"], blk["bl"], blk["ww"], blk["bw"], B, N, Hh, dh)
        ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], gamma=blk["g1"], residual=xs, out=xs)
        self._mlp(blk, xs)

    def _cls_block(self, blk, xs, B, T):
        """One class-attention block on the (B * T, D) stream: only the class rows change."""
        c = self.cfg
        D, Hh = c.embed_dim, c.nb_heads
        dh = D // Hh
        u = ops.layernorm(xs, *blk["n1"], self._plan["eps"], self.act_dtype)
        q = ops.gemm(u.view(B, T, D)[:, 0], blk["q_w"], bias=blk["q_b"])
        kv = ops.gemm(u, blk["kv_w"], bias=blk["kv_b"])
        a = cait_ops.class_attention(q, kv, B, T, Hh, dh, dh ** -0.5)
        x_cls = xs.view(B, T, D)[:, 0]
        ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], gamma=blk["g1"], residual=x_cls, out=x_cls)
        self._mlp(blk, x_cls)

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        features = OrderedDict()
        xs, grid = self._tokens(x, P)
        B, N, D = x.shape[0], grid[0] * grid[1], c.embed_dim
        if return_features:
            features["patch_embedding"] = xs.view(B, N, D).clone()
        for j, blk in enumerate(P["blocks"]):
            self._block(blk, xs, B, N)
            if return_features:
                features[f"block_{j}"] = xs.view(B, N, D).clone()
        T = N + 1
        xs = ops.assemble_tokens(xs, P["cls"], None, self._pos_table(P, grid)[1], B, N, torch.float32)
        if return_features:
            features["features_cls_token"] = xs.view(B, T, D).clone()
        for j, blk in enumerate(P["cls_blocks"]):
            self._cls_block(blk, xs, B, T)
            if return_features:
                features[f"block_cls_token_{j}"] = xs.view(B, T, D).clone()
        if return_features:
            full = ops.layernorm(xs, *P["norm"], P["eps"], torch.float32).view(B, T, D)
            features["features_all"] = full
            out = full[:, 0]
            features["features"] = out
            return out, features
        return ops.layernorm(xs.view(B, T, D)[:, 0], *P["norm"], P["eps"], torch.float32)

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


register_zoo(__name__, "cait", CaiT, CaiTConfig)
