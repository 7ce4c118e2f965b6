"""ViT / DeiT forward path as a chain of sm_90a kernels.

What the reference computes (tfimm/architectures/vit.py): PatchEmbeddings conv (k = s = patch)
-> prepend cls (and dist) token -> + pos_embed -> nb_blocks x [x + attn(LN(x)); x + mlp(LN(x))]
-> LN -> token 0 (tokens 0..1 if distilled, tanh(Dense) pre-logits if representation_size)
-> head Dense (two heads stacked on axis 1 if distilled)        [vit.py:219-235, 422-478]

How it runs here (per image batch, all on the current CUDA stream):
  patchify (im2col gather, fp32/bf16/u8 in -> bf16)            1 kernel
  patch GEMM + bias (wgmma)                                  1 kernel
  assemble tokens (+cls, +pos) into the fp32 residual stream   1 kernel
  per block: LN -> qkv GEMM -> fused attention -> proj GEMM(+residual, in place)
             LN -> fc1 GEMM(+GELU) -> fc2 GEMM(+residual, in place)          7 kernels
  final LN over the class-token rows only, head GEMM                         2-4 kernels
The residual stream stays in fp32 (bf16 would add ~2^-9 relative noise 24 times); every GEMM
operand is bf16 with fp32 accumulation.  ``precision="fp32"`` runs the same graph with fp32 SIMT
kernels and matches the oracle to ~1e-6.
"""
from collections import OrderedDict
from dataclasses import dataclass
from typing import Optional, Tuple, Union

import torch

from ..backend import ops
from ..layers.resize import interpolate_pos_embeddings
from ..models import Model, ModelConfig, ParamSpec
from ..utils import IMAGENET_INCEPTION_MEAN, IMAGENET_INCEPTION_STD
from ._zoo import register_zoo

__all__ = ["ViT", "ViTConfig"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}


@dataclass
class ViTConfig(ModelConfig):
    """Hyper-parameters of a ViT / DeiT (same fields and defaults as the reference's
    ``ViTConfig``, tfimm/architectures/vit.py:36-119)."""

    nb_classes: int = 1000
    in_channels: int = 3
    input_size: Tuple[int, int] = (224, 224)
    patch_layer: str = "patch_embeddings"
    patch_nb_blocks: tuple = ()
    patch_size: int = 16
    embed_dim: int = 768
    nb_blocks: int = 12
    nb_heads: int = 12
    mlp_ratio: float = 4.0
    qkv_bias: bool = True
    representation_size: Optional[int] = None
    distilled: bool = False
    drop_rate: float = 0.0
    attn_drop_rate: float = 0.0
    drop_path_rate: float = 0.0
    norm_layer: str = "layer_norm_eps_1e-6"
    act_layer: str = "gelu"
    interpolate_input: bool = False
    crop_pct: float = 0.875
    interpolation: str = "bicubic"
    mean: Tuple[float, float, float] = IMAGENET_INCEPTION_MEAN
    std: Tuple[float, float, float] = IMAGENET_INCEPTION_STD
    first_conv: str = "patch_embed/proj"
    classifier: Union[str, Tuple[str, str]] = "head"

    @property
    def nb_tokens(self) -> int:
        return 2 if self.distilled else 1

    @property
    def grid_size(self) -> Tuple[int, int]:
        return (self.input_size[0] // self.patch_size, self.input_size[1] // self.patch_size)

    @property
    def nb_patches(self) -> int:
        return self.grid_size[0] * self.grid_size[1]

    @property
    def transform_weights(self):
        return {"pos_embed": ViT.transform_pos_embed}


class ViT(Model):
    cfg_class = ViTConfig
    accepts_uint8 = True
    # Graph-level optimisation of the bf16 fast path (see forward_features); output-preserving, on by default.
    prune_last_block = True

    def __init__(self, cfg: ViTConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = ViTConfig(**cfg)
        if cfg.patch_layer != "patch_embeddings":
            raise ValueError(f"Unknown patch layer: {cfg.patch_layer}.")
        if cfg.representation_size and cfg.distilled:
            raise ValueError("Cannot combine distillation token and a representation layer.")
        if cfg.norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.norm_layer}")
        ops.act_code(cfg.act_layer)  # ValueError for unknown activations
        self.nb_features = cfg.representation_size or cfg.embed_dim
        super().__init__(cfg, *args, **kwargs)

    # ------------------------------------------------------------------ parameters
    def _param_specs(self):
        c = self.cfg
        D, hid = c.embed_dim, int(c.embed_dim * c.mlp_ratio)
        s = OrderedDict()

        def dense(prefix, n_in, n_out, bias=True):
            s[f"{prefix}/kernel"] = ParamSpec((n_in, n_out), "glorot_uniform")
            if bias:
                s[f"{prefix}/bias"] = ParamSpec((n_out,), "zeros")

        def norm(prefix, n):
            s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
            s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

        s["patch_embed/proj/kernel"] = ParamSpec((c.patch_size, c.patch_size, c.in_channels, D), "glorot_uniform")
        s["patch_embed/proj/bias"] = ParamSpec((D,), "zeros")
        s["cls_token"] = ParamSpec((1, 1, D), "zeros")
        if c.distilled:
            s["dist_token"] = ParamSpec((1, 1, D), "zeros")
        s["pos_embed"] = ParamSpec((1, c.nb_patches + c.nb_tokens, D), "zeros")
        for j in range(c.nb_blocks):
            p = f"blocks/{j}"
            norm(f"{p}/norm1", D)
            dense(f"{p}/attn/qkv", D, 3 * D, bias=c.qkv_bias)
            dense(f"{p}/attn/proj", D, D)
            norm(f"{p}/norm2", D)
            dense(f"{p}/mlp/fc1", D, hid)
            dense(f"{p}/mlp/fc2", hid, D)
        norm("norm", D)
        if c.representation_size:
            dense("pre_logits/fc", D, c.representation_size)
        if c.nb_classes > 0:
            dense("head", self.nb_features, c.nb_classes)
            if c.distilled:
                dense("head_dist", self.nb_features, c.nb_classes)
        return s

    def transform_pos_embed(self, src_weights, target_cfg: ViTConfig):
        return interpolate_pos_embeddings(
            self.params["pos_embed"], self.cfg.grid_size, target_cfg.grid_size, self.cfg.nb_tokens
        )

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        P = {"eps": _LN_EPS[c.norm_layer], "blocks": []}
        P["pe_w"] = self._dense_weight("patch_embed/proj/kernel")
        P["pe_b"] = self._vec("patch_embed/proj/bias")
        P["cls"] = self._vec("cls_token")
        P["dist"] = self._vec("dist_token") if c.distilled else None
        P["pos"] = self.params["pos_embed"][0].float().contiguous()
        for j in range(c.nb_blocks):
            p = f"blocks/{j}"
            P["blocks"].append(dict(
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
        P["norm"] = (self._vec("norm/gamma"), self._vec("norm/beta"))
        if c.representation_size:
            P["pre_w"] = self._dense_weight("pre_logits/fc/kernel")
            P["pre_b"] = self._vec("pre_logits/fc/bias")
        if c.nb_classes > 0:
            P["head_w"] = self._dense_weight("head/kernel")
            P["head_b"] = self._vec("head/bias")
            if c.distilled:
                P["headd_w"] = self._dense_weight("head_dist/kernel")
                P["headd_b"] = self._vec("head_dist/bias")
        return P

    # ------------------------------------------------------------------ forward
    def _tokens(self, x, P):
        """Image batch -> residual stream (B*T, D) fp32 with cls/dist tokens and pos_embed added."""
        c = self.cfg
        B, H, W, _ = x.shape
        if not c.interpolate_input and (H, W) != tuple(c.input_size):
            raise ValueError(f"Input size {(H, W)} does not match the model's {tuple(c.input_size)}; "
                             "create the model with interpolate_input=True to allow this.")
        gh, gw = H // c.patch_size, W // c.patch_size
        patches = self._patchify(x, c.patch_size)
        tok = ops.gemm(patches, P["pe_w"], bias=P["pe_b"])
        pos = P["pos"]
        if (gh, gw) != c.grid_size:
            pos = interpolate_pos_embeddings(self.params["pos_embed"], c.grid_size, (gh, gw), c.nb_tokens)
            pos = pos[0].float().contiguous()
        xs = ops.assemble_tokens(tok, P["cls"], P["dist"], pos, B, gh * gw, torch.float32)
        return xs, B, gh * gw + c.nb_tokens

    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        features = OrderedDict()
        xs, B, T = self._tokens(x, P)
        D, Hh = c.embed_dim, c.nb_heads
        dh = D // Hh
        scale = dh ** -0.5
        eps, adt = P["eps"], self.act_dtype
        if return_features:
            features["patch_embedding"] = xs.view(B, T, D).clone()
        prune_last = not return_features and self.precision == "bf16" and dh == 64 and T <= 512 and self.prune_last_block
        for j, blk in enumerate(P["blocks"]):
            h = ops.layernorm(xs, *blk["n1"], eps, adt)
            qkv = ops.gemm(h, blk["qkv_w"], bias=blk["qkv_b"])
            if return_features:
                probs = torch.empty((B, Hh, T, T), device=xs.device, dtype=torch.float32)
                ops.attention(ops.cast(qkv, torch.float32), B, T, Hh, dh, scale, probs=probs)
                features[f"block_{j}/attn"] = probs
            if prune_last and j == len(P["blocks"]) - 1:
                # Last block: only the class (and distillation) token rows reach the head (vit.py:452-464), so
                # attention, proj, norm2 and the MLP run on those B * nq rows only; keys / values above came from
                # every token.  Same arithmetic per row, 6-7 % of a ViT-B step.  ``model.prune_last_block = False`` disables.
                nq = 2 if c.distilled else 1
                a = ops.attention_cls(qkv, B, T, Hh, dh, scale, nq)
                x3 = xs.view(B, T, D)
                for i in range(nq):
                    xi = x3[:, i]                                   # (B, D) view of the fp32 stream, row stride T*D
                    ops.gemm(a.view(B, nq, D)[:, i], blk["proj_w"], bias=blk["proj_b"], residual=xi, out=xi)
                    hi = ops.layernorm(xi, *blk["n2"], eps, adt)
                    hid = ops.gemm(hi, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
                    ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], residual=xi, out=xi)
                continue
            if qkv.dtype == torch.bfloat16 and not ops.attention_bf16_supported(T, dh):
                # head_dim != 64 (vit_huge: 80) or K/V too long for shared memory: fp32 SIMT attention on the
                # same bf16 qkv values (as Swin does for window-12 models); correctness first, not a fast path
                a = ops.cast(ops.attention(ops.cast(qkv, torch.float32), B, T, Hh, dh, scale), torch.bfloat16)
            else:
                a = ops.attention(qkv, B, T, Hh, dh, scale)
            ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], residual=xs, out=xs)
            h = ops.layernorm(xs, *blk["n2"], eps, adt)
            hid = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=c.act_layer)
            ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], residual=xs, out=xs)
            if return_features:
                features[f"block_{j}"] = xs.view(B, T, D).clone()
        x3 = xs.view(B, T, D)
        if return_features:
            full = ops.layernorm(xs, *P["norm"], eps, torch.float32).view(B, T, D)
            features["features_all"] = full
            if c.distilled:
                out = full[:, :2]
            elif c.representation_size:
                out = ops.gemm(ops.cast(full[:, 0].contiguous(), adt), P["pre_w"], bias=P["pre_b"], act="tanh",
                               out_dtype=torch.float32)
            else:
                out = full[:, 0]
            features["features"] = out
            return out, features
        # Fast path: the final LayerNorm is per token, so only the rows that feed the head are normalised.
        if c.distilled:
            out = torch.stack(
                [ops.layernorm(x3[:, i], *P["norm"], eps, torch.float32) for i in range(2)], dim=1)
        else:
            out = ops.layernorm(x3[:, 0], *P["norm"], eps, torch.float32)
            if c.representation_size:
                out = ops.gemm(ops.cast(out, adt), P["pre_w"], bias=P["pre_b"], act="tanh", out_dtype=torch.float32)
        return out

    def _head(self, feats, w, b):
        return ops.gemm(ops.cast(feats.contiguous(), self.act_dtype), w, bias=b, out_dtype=torch.float32)

    def call(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        features = {}
        x = self.forward_features(x, training, return_features)
        if return_features:
            x, features = x
        if c.nb_classes > 0:
            if not c.distilled:
                x = self._head(x, P["head_w"], P["head_b"])
            else:
                y = self._head(x[:, 0], P["head_w"], P["head_b"])
                y_dist = self._head(x[:, 1], P["headd_w"], P["headd_b"])
                x = torch.stack((y, y_dist), dim=1)
        features["logits"] = x
        return (x, features) if return_features else x


register_zoo(__name__, "vit", ViT, ViTConfig)
