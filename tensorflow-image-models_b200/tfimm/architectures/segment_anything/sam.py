"""Segment Anything: the model object with every reference variable, and the image encoder as a chain of sm_90a kernels.

What the reference computes (tfimm/architectures/segment_anything/image_encoder.py:363-515): PatchEmbeddings conv
(k = s = 16) -> + pos_embed (bilinearly resized to the input's grid when ``fixed_input_size=False``) -> nb_blocks x
[x + proj(relpos_attn(LN(x))); x + lin2(gelu(lin1(LN(x))))], where most blocks attend inside 14 x 14 windows of the
grid padded to a multiple of 14 and the blocks of ``encoder_global_attn_indices`` over the whole grid, both with
decomposed relative-position terms -> neck: 1x1 conv (no bias) -> LN(1e-6) -> 3x3 "same" conv (no bias) -> LN(1e-6).

How it runs here (per image batch, on the current CUDA stream):
  patchify (fp32/bf16/u8 in)                                             1 kernel
  patch GEMM + bias + pos_embed (residual epilogue, fp32 stream)         1 kernel per image
  per block: LN -> qkv GEMM -> relpos attention -> proj GEMM(+residual, in place)
             LN -> lin1 GEMM(+GELU) -> lin2 GEMM(+residual, in place)                      7 kernels
  neck: cast -> 1x1 GEMM -> LN -> 3x3 implicit-GEMM conv (bf16; im2col + GEMM in fp32) -> LN
The window partition is index math inside the attention kernel (``csrc/relpos_attention.cu``): the qkv GEMM runs on
the real tokens only, and the padding positions' keys / values (the qkv bias, as in the reference) are synthesised.

The prompt encoder and the mask decoder hold their variables (checkpoints load with ``strict=True``) but do not run:
``SegmentAnythingModel.__call__`` raises ``NotImplementedError``; ``model.image_encoder(images)`` computes the image
embeddings.
"""
from collections import OrderedDict
from collections.abc import MutableMapping
from dataclasses import dataclass
from functools import partial
from typing import Optional, Tuple

import torch

from ...backend import ops, sam_ops
from ...layers.resize import tf_bilinear_resize
from ...models import Model, ModelConfig, ParamSpec, register_model
from ...utils import IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD

__all__ = ["SegmentAnythingModel", "SegmentAnythingModelConfig", "ImageEncoder"]

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}
_ENC = "image_encoder/"


@dataclass
class SegmentAnythingModelConfig(ModelConfig):
    """Hyper-parameters of a SAM model (same fields and defaults as the reference's ``SegmentAnythingModelConfig``,
    tfimm/architectures/segment_anything/sam.py:61-173)."""

    in_channels: int = 3
    input_size: Tuple[int, int] = (1024, 1024)
    fixed_input_size: bool = True
    embed_dim: int = 256
    nb_multimask_outputs: int = 3
    mask_threshold: float = 0.0

    encoder_patch_size: int = 16
    encoder_embed_dim: int = 768
    encoder_nb_blocks: int = 12
    encoder_nb_heads: int = 12
    encoder_mlp_ratio: float = 4.0

    encoder_drop_rate: float = 0.0
    encoder_attn_drop_rate: float = 0.0
    encoder_drop_path_rate: float = 0.0

    encoder_norm_layer: str = "layer_norm_eps_1e-6"
    encoder_act_layer: str = "gelu"
    encoder_qkv_bias: bool = True
    encoder_global_attn_indices: Tuple = (2, 5, 8, 11)
    encoder_window_size: int = 14

    prompt_mask_hidden_dim: int = 16

    decoder_nb_blocks: int = 2
    decoder_nb_heads: int = 8
    decoder_mlp_channels: int = 2048
    decoder_iou_head_depth: int = 3
    decoder_iou_hidden_dim: int = 256

    mean: Tuple[float, float, float] = IMAGENET_DEFAULT_MEAN
    std: Tuple[float, float, float] = IMAGENET_DEFAULT_STD

    first_conv: str = "image_encoder/patch_embed/proj"

    @property
    def transform_weights(self):
        """Weights that need resampling when ``create_model`` changes ``input_size`` (reference sam.py:158-173): the
        absolute position embedding, and the relative-position tables of the global blocks (the window blocks' tables
        depend on the window size only)."""
        transforms = {"image_encoder/pos_embed": transform_pos_embed}
        for j in self.encoder_global_attn_indices:
            prefix = f"image_encoder/blocks/{j}/attn/rel_pos"
            transforms[prefix + "_h"] = partial(transform_rel_pos, axis=0)
            transforms[prefix + "_w"] = partial(transform_rel_pos, axis=1)
        return transforms


def _resize_rel_pos(rel_pos: torch.Tensor, length: int) -> torch.Tensor:
    """(L, C) -> (length, C): tf.image.resize of the (1, L, C) image to (1, length), bilinear."""
    return tf_bilinear_resize(rel_pos.float()[None, None], (1, length))[0, 0]


def transform_rel_pos(model, rel_pos, target_cfg: SegmentAnythingModelConfig, axis: int):
    """Reference sam.py:176-190."""
    grid_dim = target_cfg.input_size[axis] // target_cfg.encoder_patch_size
    return _resize_rel_pos(rel_pos, 2 * grid_dim - 1)


def transform_pos_embed(model, pos_embed, target_cfg: SegmentAnythingModelConfig):
    """Reference sam.py:193-203."""
    grid = (target_cfg.input_size[0] // target_cfg.encoder_patch_size,
            target_cfg.input_size[1] // target_cfg.encoder_patch_size)
    return tf_bilinear_resize(pos_embed.float(), grid)


def param_specs(cfg: SegmentAnythingModelConfig) -> "OrderedDict[str, ParamSpec]":
    """Every variable of the reference model (image_encoder.py, prompt_encoder.py, mask_decoder.py, transformer.py),
    names without the "<model>/" prefix and ":0"."""
    s = OrderedDict()

    def dense(prefix, n_in, n_out, bias=True):
        s[f"{prefix}/kernel"] = ParamSpec((n_in, n_out), "glorot_uniform")
        if bias:
            s[f"{prefix}/bias"] = ParamSpec((n_out,), "zeros")

    def conv(prefix, k, n_in, n_out, bias=True, transpose=False):
        s[f"{prefix}/kernel"] = ParamSpec((k, k, n_out, n_in) if transpose else (k, k, n_in, n_out), "glorot_uniform")
        if bias:
            s[f"{prefix}/bias"] = ParamSpec((n_out,), "zeros")

    def norm(prefix, n):
        s[f"{prefix}/gamma"] = ParamSpec((n,), "ones")
        s[f"{prefix}/beta"] = ParamSpec((n,), "zeros")

    # image encoder (image_encoder.py:171-229, 266-338, 363-492; common.py:6-36)
    D, p, E = cfg.encoder_embed_dim, cfg.encoder_patch_size, cfg.embed_dim
    dh, hid = D // cfg.encoder_nb_heads, int(D * cfg.encoder_mlp_ratio)
    gh, gw = cfg.input_size[0] // p, cfg.input_size[1] // p
    s["image_encoder/pos_embed"] = ParamSpec((1, gh, gw, D), "zeros")
    conv("image_encoder/patch_embed/proj", p, cfg.in_channels, D)
    for j in range(cfg.encoder_nb_blocks):
        b = f"image_encoder/blocks/{j}"
        ws = 0 if j in cfg.encoder_global_attn_indices else cfg.encoder_window_size
        norm(f"{b}/norm1", D)
        dense(f"{b}/attn/qkv", D, 3 * D, bias=cfg.encoder_qkv_bias)
        dense(f"{b}/attn/proj", D, D)
        s[f"{b}/attn/rel_pos_h"] = ParamSpec((2 * (ws or gh) - 1, dh), "zeros")
        s[f"{b}/attn/rel_pos_w"] = ParamSpec((2 * (ws or gw) - 1, dh), "zeros")
        norm(f"{b}/norm2", D)
        dense(f"{b}/mlp/lin1", D, hid)
        dense(f"{b}/mlp/lin2", hid, D)
    conv("image_encoder/neck/0", 1, D, E, bias=False)
    norm("image_encoder/neck/1", E)
    conv("image_encoder/neck/2", 3, E, E, bias=False)
    norm("image_encoder/neck/3", E)

    # prompt encoder (prompt_encoder.py:30-75, 187-215, 264-270)
    s["prompt_encoder/pe_layer/positional_encoding_gaussian_matrix"] = ParamSpec((2, E // 2), "normal:1.0", False)
    for j in range(4):
        s[f"prompt_encoder/point_embeddings/{j}/weight"] = ParamSpec((1, E), "normal:0.05")
    s["prompt_encoder/not_a_point_embed/weight"] = ParamSpec((1, E), "normal:0.05")
    mh = cfg.prompt_mask_hidden_dim
    conv("prompt_encoder/mask_downscaling/0", 2, 1, mh // 4)
    norm("prompt_encoder/mask_downscaling/1", mh // 4)
    conv("prompt_encoder/mask_downscaling/3", 2, mh // 4, mh)
    norm("prompt_encoder/mask_downscaling/4", mh)
    conv("prompt_encoder/mask_downscaling/6", 1, mh, E)
    s["prompt_encoder/no_mask_embed/weight"] = ParamSpec((1, E), "normal:0.05")

    # mask decoder (mask_decoder.py:45-76, 170-241; transformer.py:8-260)
    nmt = cfg.nb_multimask_outputs + 1
    s["mask_decoder/iou_token/weight"] = ParamSpec((1, E), "normal:0.05")
    s["mask_decoder/mask_tokens/weight"] = ParamSpec((nmt, E), "normal:0.05")

    def attn(prefix, rate):
        for n in ("q_proj", "k_proj", "v_proj"):
            dense(f"{prefix}/{n}", E, E // rate)
        dense(f"{prefix}/out_proj", E // rate, E)

    t = "mask_decoder/transformer"
    for j in range(cfg.decoder_nb_blocks):
        b = f"{t}/layers/{j}"
        attn(f"{b}/self_attn", 1)
        norm(f"{b}/norm1", E)
        attn(f"{b}/cross_attn_token_to_image", 2)
        norm(f"{b}/norm2", E)
        dense(f"{b}/mlp/lin1", E, cfg.decoder_mlp_channels)
        dense(f"{b}/mlp/lin2", cfg.decoder_mlp_channels, E)
        norm(f"{b}/norm3", E)
        attn(f"{b}/cross_attn_image_to_token", 2)
        norm(f"{b}/norm4", E)
    attn(f"{t}/final_attn_token_to_image", 2)
    norm(f"{t}/norm_final_attn", E)
    conv("mask_decoder/output_upscaling/0", 2, E, E // 4, transpose=True)
    norm("mask_decoder/output_upscaling/1", E // 4)
    conv("mask_decoder/output_upscaling/3", 2, E // 4, E // 8, transpose=True)
    for j in range(nmt):
        for k, (n_in, n_out) in enumerate(((E, E), (E, E), (E, E // 8))):
            dense(f"mask_decoder/output_hypernetworks_mlps/{j}/layers/{k}", n_in, n_out)
    dims = [E] + [cfg.decoder_iou_hidden_dim] * (cfg.decoder_iou_head_depth - 1) + [nmt]
    for k in range(cfg.decoder_iou_head_depth):
        dense(f"mask_decoder/iou_prediction_head/layers/{k}", dims[k], dims[k + 1])
    return s


class _EncoderParams(MutableMapping):
    """The parent model's ``image_encoder/*`` tensors under their names inside the encoder: reads and writes go to the
    parent's dict, so both objects always see the same tensors."""

    def __init__(self, parent_params):
        self._p = parent_params

    def __getitem__(self, key):
        return self._p[_ENC + key]

    def __setitem__(self, key, value):
        self._p[_ENC + key] = value

    def __delitem__(self, key):
        raise TypeError("the image encoder's variables cannot be removed")

    def __iter__(self):
        return (k[len(_ENC):] for k in self._p if k.startswith(_ENC))

    def __len__(self):
        return sum(1 for _ in self)


class ImageEncoder(Model):
    """SAM's image encoder (reference ``ImageEncoder``, a ``tf.keras.Model`` too): NHWC images (N, H, W, C) -> image
    embeddings (N, H/16, W/16, embed_dim) fp32.  Its variables are the parent model's ``image_encoder/*`` tensors."""

    cfg_class = SegmentAnythingModelConfig
    accepts_uint8 = True

    def __init__(self, parent: "SegmentAnythingModel"):
        # No Model.__init__ (it would create a second set of variables): the bookkeeping attributes it sets are set
        # here instead.  tests/test_sam_cpu.py::test_image_encoder_has_the_model_attributes fails when Model.__init__
        # gains one that is missing here.
        self._parent = parent
        self.cfg = parent.cfg
        self.name = "image_encoder"
        self.precision = parent.precision
        self.params = _EncoderParams(parent.params)
        self._specs = None
        self._plan = None
        self._plan_version = 0
        self._seed = parent._seed

    @property
    def device(self):
        return self._parent.device

    def to(self, device):
        self._parent.to(device)
        return self

    def _param_specs(self):
        return OrderedDict((k[len(_ENC):], v) for k, v in self._parent.param_specs().items() if k.startswith(_ENC))

    def _invalidate(self):
        self._plan = None
        self._plan_version += 1

    def load_weights_dict(self, weights, strict: bool = True):
        super().load_weights_dict(weights, strict)
        self._parent._plan_version += 1

    # ------------------------------------------------------------------ engine plan
    def _compile(self):
        c = self.cfg
        D, Hh = c.encoder_embed_dim, c.encoder_nb_heads
        if D % 8 or (D // Hh) % 2:
            raise ValueError(f"the image encoder's kernels need embed_dim % 8 == 0 and an even head_dim (got {D}, {Hh} "
                             "heads)")
        P = {"eps": _LN_EPS[c.encoder_norm_layer], "blocks": [], "geo": {}}
        P["pe_w"] = self._dense_weight("patch_embed/proj/kernel")
        P["pe_b"] = self._vec("patch_embed/proj/bias")
        for j in range(c.encoder_nb_blocks):
            p = f"blocks/{j}"
            qkv_b = self._vec(f"{p}/attn/qkv/bias") if c.encoder_qkv_bias else None
            P["blocks"].append(dict(
                window=0 if j in c.encoder_global_attn_indices else c.encoder_window_size,
                n1=(self._vec(f"{p}/norm1/gamma"), self._vec(f"{p}/norm1/beta")),
                qkv_w=self._dense_weight(f"{p}/attn/qkv/kernel"),
                qkv_b=qkv_b,
                # keys / values of the window padding: the qkv bias as the GEMM would store it
                pad=qkv_b.to(self.act_dtype).contiguous() if qkv_b is not None else None,
                proj_w=self._dense_weight(f"{p}/attn/proj/kernel"),
                proj_b=self._vec(f"{p}/attn/proj/bias"),
                n2=(self._vec(f"{p}/norm2/gamma"), self._vec(f"{p}/norm2/beta")),
                fc1_w=self._dense_weight(f"{p}/mlp/lin1/kernel"),
                fc1_b=self._vec(f"{p}/mlp/lin1/bias"),
                fc2_w=self._dense_weight(f"{p}/mlp/lin2/kernel"),
                fc2_b=self._vec(f"{p}/mlp/lin2/bias"),
            ))
        P["neck0_w"] = self._dense_weight("neck/0/kernel")
        P["neck1"] = (self._vec("neck/1/gamma"), self._vec("neck/1/beta"))
        P["neck2_w"] = self._dense_weight("neck/2/kernel")
        P["neck3"] = (self._vec("neck/3/gamma"), self._vec("neck/3/beta"))
        return P

    def _geometry(self, P, gh, gw):
        """Position embedding and relative-position tables for a gh x gw token grid: computed once per grid size (cold
        path, cached with the plan).  ``fixed_input_size=False`` resizes them as the reference does on every call
        (image_encoder.py:497-504, 76-118); the window blocks' tables keep their size (their extent is the window)."""
        if (gh, gw) in P["geo"]:
            return P["geo"][(gh, gw)]
        c = self.cfg
        pos = self.params["pos_embed"].float()
        if not c.fixed_input_size:
            pos = tf_bilinear_resize(pos, (gh, gw))
        rel = []
        for j, blk in enumerate(P["blocks"]):
            rh = self.params[f"blocks/{j}/attn/rel_pos_h"].float()
            rw = self.params[f"blocks/{j}/attn/rel_pos_w"].float()
            sh, sw = (blk["window"], blk["window"]) if blk["window"] else (gh, gw)
            if not c.fixed_input_size:
                rh, rw = _resize_rel_pos(rh, 2 * sh - 1), _resize_rel_pos(rw, 2 * sw - 1)
            if rh.shape[0] != 2 * sh - 1 or rw.shape[0] != 2 * sw - 1:
                raise ValueError(f"block {j}: relative-position tables {tuple(rh.shape)} / {tuple(rw.shape)} do not fit "
                                 f"a {sh} x {sw} attention extent")
            rel.append((rh.contiguous(), rw.contiguous()))
        geo = P["geo"][(gh, gw)] = (pos.reshape(gh * gw, -1).contiguous(), rel)
        return geo

    # ------------------------------------------------------------------ forward
    def forward_features(self, x, training=False, return_features=False):
        c = self.cfg
        P = self._ensure_plan()
        x = self._input(x)
        B, H, W, _ = x.shape
        p = c.encoder_patch_size
        if c.fixed_input_size and (H, W) != tuple(c.input_size):
            raise ValueError(f"Input size {(H, W)} does not match the model's {tuple(c.input_size)}; create the model "
                             "with fixed_input_size=False to allow this.")
        gh, gw = H // p, W // p
        T, D, Hh = gh * gw, c.encoder_embed_dim, c.encoder_nb_heads
        dh = D // Hh
        scale = dh ** -0.5
        eps, adt = P["eps"], self.act_dtype
        pos, rel = self._geometry(P, gh, gw)
        features = OrderedDict()

        patches = self._patchify(x, p)
        xs = torch.empty((B * T, D), device=patches.device, dtype=torch.float32)   # fp32 residual stream
        for b in range(B):
            ops.gemm(patches[b * T:(b + 1) * T], P["pe_w"], bias=P["pe_b"], residual=pos, out=xs[b * T:(b + 1) * T])
        if return_features:
            features["patch_embedding"] = xs.view(B, gh, gw, D).clone()
        for j, blk in enumerate(P["blocks"]):
            h = ops.layernorm(xs, *blk["n1"], eps, adt)
            qkv = ops.gemm(h, blk["qkv_w"], bias=blk["qkv_b"])
            rh, rw = rel[j]
            sh, sw = (blk["window"], blk["window"]) if blk["window"] else (gh, gw)
            if qkv.dtype == torch.bfloat16 and not sam_ops.relpos_attention_bf16_supported(dh, sh, sw):
                # head dims other than 64 / 80, and global grids too large for the tensor-core kernel's shared memory
                # (fixed_input_size=False above ~1200 px): the fp32 kernel on the same bf16 values
                pad = ops.cast(blk["pad"], torch.float32) if blk["pad"] is not None else None
                a = sam_ops.relpos_attention(ops.cast(qkv, torch.float32), B, gh, gw, Hh, dh, scale, rh, rw,
                                             blk["window"], pad)
                a = ops.cast(a, torch.bfloat16)
            else:
                a = sam_ops.relpos_attention(qkv, B, gh, gw, Hh, dh, scale, rh, rw, blk["window"], blk["pad"])
            ops.gemm(a, blk["proj_w"], bias=blk["proj_b"], residual=xs, out=xs)
            h = ops.layernorm(xs, *blk["n2"], eps, adt)
            hid = ops.gemm(h, blk["fc1_w"], bias=blk["fc1_b"], act=c.encoder_act_layer)
            ops.gemm(hid, blk["fc2_w"], bias=blk["fc2_b"], residual=xs, out=xs)
            if return_features:
                features[f"block_{j}"] = xs.view(B, gh, gw, D).clone()

        E = c.embed_dim
        y = ops.gemm(ops.cast(xs, adt), P["neck0_w"], out_dtype=torch.float32)
        y = ops.layernorm(y, *P["neck1"], 1e-6, adt).view(B, gh, gw, E)
        if adt == torch.bfloat16 and E % 64 == 0:
            y = ops.conv_gemm(y, P["neck2_w"], ks=3, stride=1, pad=1, out_dtype=torch.float32)
        else:
            cols, _, _ = ops.im2col(y, 3, 1, 1, adt)
            y = ops.gemm(cols, P["neck2_w"], out_dtype=torch.float32)
        y = ops.layernorm(y.reshape(B * T, E), *P["neck3"], 1e-6, torch.float32).view(B, gh, gw, E)
        features["neck"] = y
        return (y, features) if return_features else y

    def call(self, x, training=False, return_features=False):
        return self.forward_features(x, training, return_features)


class SegmentAnythingModel(Model):
    """Reference ``SegmentAnythingModel`` (sam.py:206-419).  Holds every variable of the model; the image encoder
    runs (``model.image_encoder``), mask prediction does not yet."""

    cfg_class = SegmentAnythingModelConfig

    def __init__(self, cfg: SegmentAnythingModelConfig, *args, **kwargs):
        if isinstance(cfg, dict):
            cfg = SegmentAnythingModelConfig(**cfg)
        if kwargs.get("precision", "bf16") == "tf32":
            raise ValueError("Segment Anything models run in precision 'bf16' or 'fp32'; tf32 is not implemented for "
                             "them.")
        if cfg.encoder_norm_layer not in _LN_EPS:
            raise ValueError(f"Unknown normalization layer: {cfg.encoder_norm_layer}")
        ops.act_code(cfg.encoder_act_layer)  # ValueError for unknown activations
        super().__init__(cfg, *args, **kwargs)
        self.image_encoder = ImageEncoder(self)

    def _param_specs(self):
        return param_specs(self.cfg)

    def load_weights_dict(self, weights, strict: bool = True):
        super().load_weights_dict(weights, strict)
        if hasattr(self, "image_encoder"):
            self.image_encoder._invalidate()

    def to(self, device):
        super().to(device)
        self.image_encoder._invalidate()
        return self

    def grid_size(self, input_size: Optional[Tuple[int, int]] = None) -> Tuple[int, int]:
        """Spatial size (H'', W'') of the image embeddings for an input size (default: the config's)."""
        input_size = input_size or self.cfg.input_size
        return input_size[0] // self.cfg.encoder_patch_size, input_size[1] // self.cfg.encoder_patch_size

    def mask_size(self, input_size: Optional[Tuple[int, int]] = None) -> Tuple[int, int]:
        """Spatial size (H', W') = 4 x grid size of the low-resolution masks."""
        gh, gw = self.grid_size(input_size)
        return 4 * gh, 4 * gw

    @property
    def mask_threshold(self):
        """Threshold for turning mask logits into boolean masks."""
        return self.cfg.mask_threshold

    @property
    def dummy_inputs(self):
        c = self.cfg
        z = partial(torch.zeros, device=self.device)
        return {"images": z((1, *c.input_size, c.in_channels)), "points": z((1, 1, 2)), "labels": z((1, 1)),
                "boxes": z((1, 1, 4)), "masks": z((1, 1, *self.mask_size(c.input_size)))}

    def forward_features(self, x, training=False, return_features=False):
        return self.image_encoder(x, return_features=return_features)

    def call(self, inputs, training=False, return_features=False):
        raise NotImplementedError(
            "Mask prediction (prompt encoder and mask decoder) is not implemented for Segment Anything models yet; "
            "`model.image_encoder(images)` computes the image embeddings.")


def _variant(name, url, dim, blocks, heads, global_idx):
    cfg = SegmentAnythingModelConfig(name=name, url=url, encoder_embed_dim=dim, encoder_nb_blocks=blocks,
                                     encoder_nb_heads=heads, encoder_global_attn_indices=global_idx)
    return SegmentAnythingModel, cfg


@register_model
def sam_vit_b():
    """SAM ViT-Base"""
    return _variant("sam_vit_b", "[pytorch]https://dl.fbaipublicfiles.com/segment_anything/sam_vit_b_01ec64.pth",
                    768, 12, 12, (2, 5, 8, 11))


@register_model
def sam_vit_l():
    """SAM ViT-Large"""
    return _variant("sam_vit_l", "[pytorch]https://dl.fbaipublicfiles.com/segment_anything/sam_vit_l_0b3195.pth",
                    1024, 24, 16, (5, 11, 17, 23))


@register_model
def sam_vit_h():
    """SAM ViT-Huge"""
    return _variant("sam_vit_h", "[pytorch]https://dl.fbaipublicfiles.com/segment_anything/sam_vit_h_4b8939.pth",
                    1280, 32, 16, (7, 15, 23, 31))
