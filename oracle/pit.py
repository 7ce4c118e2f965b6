"""Oracle restatement of the reference PiT forward (tfimm/architectures/pit.py, reusing vit.ViTBlock), in float64 on
the CPU."""
from collections import OrderedDict
from types import SimpleNamespace

import torch

from . import tf_ops as tf
from . import vit as ovit


def grid_size(cfg, input_size=None):
    h, w = input_size or cfg.input_size
    return (h - cfg.patch_size) // cfg.stride + 1, (w - cfg.patch_size) // cfg.stride + 1


def param_shapes(cfg):
    """Variable names (without the "<model>/" prefix and ":0") and shapes, in creation order: pos_embed and cls_token
    by the model's build() (pit.py:266-281), then the layers in call order (pit.py:331-395)."""
    nb = 2 if cfg.distilled else 1
    gh, gw = grid_size(cfg)
    s = OrderedDict()
    s["pos_embed"] = (1, cfg.embed_dim[0], gh, gw)
    s["cls_token"] = (1, nb, cfg.embed_dim[0])
    s["patch_embed/conv/kernel"] = (cfg.patch_size, cfg.patch_size, cfg.in_channels, cfg.embed_dim[0])
    s["patch_embed/conv/bias"] = (cfg.embed_dim[0],)
    for j, (D, depth) in enumerate(zip(cfg.embed_dim, cfg.nb_blocks)):
        hid = int(D * cfg.mlp_ratio)
        for k in range(depth):
            p = f"transformers/{j}/blocks/{k}"
            s[f"{p}/norm1/gamma"] = (D,)
            s[f"{p}/norm1/beta"] = (D,)
            s[f"{p}/attn/qkv/kernel"] = (D, 3 * D)
            s[f"{p}/attn/qkv/bias"] = (3 * D,)
            s[f"{p}/attn/proj/kernel"] = (D, D)
            s[f"{p}/attn/proj/bias"] = (D,)
            s[f"{p}/norm2/gamma"] = (D,)
            s[f"{p}/norm2/beta"] = (D,)
            s[f"{p}/mlp/fc1/kernel"] = (D, hid)
            s[f"{p}/mlp/fc1/bias"] = (hid,)
            s[f"{p}/mlp/fc2/kernel"] = (hid, D)
            s[f"{p}/mlp/fc2/bias"] = (D,)
        if j < len(cfg.nb_blocks) - 1:
            p = f"transformers/{j + 1}/pool"
            s[f"{p}/conv/kernel"] = (3, 3, 1, cfg.embed_dim[j + 1])
            s[f"{p}/conv/bias"] = (cfg.embed_dim[j + 1],)
            s[f"{p}/fc/kernel"] = (D, cfg.embed_dim[j + 1])
            s[f"{p}/fc/bias"] = (cfg.embed_dim[j + 1],)
    s["norm/gamma"] = (cfg.embed_dim[-1],)
    s["norm/beta"] = (cfg.embed_dim[-1],)
    if cfg.nb_classes > 0:
        s["head/kernel"] = (cfg.embed_dim[-1], cfg.nb_classes)
        s["head/bias"] = (cfg.nb_classes,)
        if cfg.distilled:
            s["head_dist/kernel"] = (cfg.embed_dim[-1], cfg.nb_classes)
            s["head_dist/bias"] = (cfg.nb_classes,)
    return s


def conv_head_pooling(x, w, prefix, nb_tokens, grid):
    """ConvHeadPooling.call (pit.py:172-188): the grid rows zero-padded by 1 and convolved 3 x 3 / 2 with groups = C
    (output channel o reads input channel o // 2), the token rows through Dense; tokens first."""
    B, _, C = x.shape
    tokens, g = x[:, :nb_tokens], x[:, nb_tokens:].reshape(B, *grid, C)
    g = tf.conv2d(g, w[f"{prefix}/conv/kernel"], w[f"{prefix}/conv/bias"], stride=2, padding=1, groups=C)
    tokens = tf.dense(tokens, w[f"{prefix}/fc/kernel"], w[f"{prefix}/fc/bias"])
    return torch.cat((tokens, g.reshape(B, -1, g.shape[-1])), dim=1), tuple(g.shape[1:3])


def forward_features(cfg, w, x, return_features=False):
    """PoolingVisionTransformer.forward_features, pit.py:310-364."""
    features = OrderedDict()
    nb = 2 if cfg.distilled else 1
    B = x.shape[0]
    x = tf.conv2d(x, w["patch_embed/conv/kernel"], w["patch_embed/conv/bias"], stride=cfg.stride)
    pos = w["pos_embed"].permute(0, 2, 3, 1)
    grid = tuple(x.shape[1:3])
    if getattr(cfg, "interpolate_input", False) and grid != tuple(pos.shape[1:3]):
        # interpolate_pos_embeddings_grid: tf.image.resize on the grid, which returns float32 whatever its input
        pos = tf.resize_bicubic(pos, grid).float().to(pos.dtype)
    x = x + pos
    x = torch.cat((w["cls_token"].expand(B, -1, -1), x.reshape(B, -1, x.shape[-1])), dim=1)
    features["patch_embedding"] = x
    for j, depth in enumerate(cfg.nb_blocks):
        bcfg = SimpleNamespace(nb_heads=cfg.nb_heads[j], qkv_bias=True, norm_layer=cfg.norm_layer,
                               act_layer=cfg.act_layer)
        for k in range(depth):
            x, _ = ovit.block(x, w, f"transformers/{j}/blocks/{k}", bcfg)
            features[f"stage_{j}/block_{k}"] = x
        if j < len(cfg.nb_blocks) - 1:
            x, grid = conv_head_pooling(x, w, f"transformers/{j + 1}/pool", nb, grid)
            features[f"stage_{j}/pool"] = x
    features["features_all"] = x
    x = tf.norm(x[:, :nb], w, "norm", cfg.norm_layer)
    x = x if cfg.distilled else x[:, 0]
    features["features"] = x
    return (x, features) if return_features else x


def forward(cfg, w, x, return_features=False):
    """PoolingVisionTransformer.call, pit.py:366-395.  w: {name: tensor} in reference layouts; x: (B, H, W, C)
    preprocessed images."""
    w = {k: torch.as_tensor(v).double() for k, v in w.items()}
    x = torch.as_tensor(x).double()
    features = {}
    x = forward_features(cfg, w, x, return_features)
    if return_features:
        x, features = x
    if cfg.nb_classes > 0:
        if not cfg.distilled:
            x = tf.dense(x, w["head/kernel"], w["head/bias"])
        else:
            x = torch.stack((tf.dense(x[:, 0], w["head/kernel"], w["head/bias"]),
                             tf.dense(x[:, 1], w["head_dist/kernel"], w["head_dist/bias"])), dim=1)
    features["logits"] = x
    return (x, features) if return_features else x
