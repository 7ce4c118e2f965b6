"""Oracle restatement of the reference PVT v2 forward (tfimm/architectures/pvt_v2.py), in float64 on the CPU."""
from collections import OrderedDict

import torch

from . import tf_ops as tf
from .pvt import sr_attention


def patch_geometry(j):
    """(kernel, stride, zero padding) of stage j's PatchEmbeddings (pvt_v2.py:319-326; padding patch_size // 2,
    layers/transformers.py:121-130)."""
    k, s = (7, 4) if j == 0 else (3, 2)
    return k, s, k // 2


def grid_sizes(cfg, input_size=None):
    h, w = input_size or cfg.input_size
    out = []
    for j in range(len(cfg.nb_blocks)):
        k, s, p = patch_geometry(j)
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        out.append((h, w))
    return out


def param_shapes(cfg):
    """Variable names (without the "<model>/" prefix and ":0") and shapes, in the order of the reference's
    ``weights``: patch_embed*, then blocks, then norms (the lists in __init__ order, pvt_v2.py:314-346), then head."""
    s = OrderedDict()
    cin = cfg.in_channels
    for j, D in enumerate(cfg.embed_dim):
        k = patch_geometry(j)[0]
        s[f"patch_embed{j + 1}/proj/kernel"] = (k, k, cin, D)
        s[f"patch_embed{j + 1}/proj/bias"] = (D,)
        s[f"patch_embed{j + 1}/norm/gamma"] = (D,)
        s[f"patch_embed{j + 1}/norm/beta"] = (D,)
        cin = D
    for j, (D, depth) in enumerate(zip(cfg.embed_dim, cfg.nb_blocks)):
        sr, hid = cfg.sr_ratio[j], int(D * cfg.mlp_ratio[j])
        for k in range(depth):
            b = f"block{j + 1}/{k}"
            s[f"{b}/norm1/gamma"] = (D,)
            s[f"{b}/norm1/beta"] = (D,)
            s[f"{b}/attn/q/kernel"] = (D, D)
            if cfg.qkv_bias:
                s[f"{b}/attn/q/bias"] = (D,)
            s[f"{b}/attn/kv/kernel"] = (D, 2 * D)
            if cfg.qkv_bias:
                s[f"{b}/attn/kv/bias"] = (2 * D,)
            s[f"{b}/attn/proj/kernel"] = (D, D)
            s[f"{b}/attn/proj/bias"] = (D,)
            if sr > 1:
                s[f"{b}/attn/sr/kernel"] = (sr, sr, D, D)
                s[f"{b}/attn/sr/bias"] = (D,)
                s[f"{b}/attn/norm/gamma"] = (D,)
                s[f"{b}/attn/norm/beta"] = (D,)
            s[f"{b}/norm2/gamma"] = (D,)
            s[f"{b}/norm2/beta"] = (D,)
            s[f"{b}/mlp/fc1/kernel"] = (D, hid)
            s[f"{b}/mlp/fc1/bias"] = (hid,)
            s[f"{b}/mlp/dwconv/dwconv/depthwise_kernel"] = (3, 3, hid, 1)
            s[f"{b}/mlp/dwconv/dwconv/bias"] = (hid,)
            s[f"{b}/mlp/fc2/kernel"] = (hid, D)
            s[f"{b}/mlp/fc2/bias"] = (D,)
    for j, D in enumerate(cfg.embed_dim):
        s[f"norm{j + 1}/gamma"] = (D,)
        s[f"norm{j + 1}/beta"] = (D,)
    if cfg.nb_classes > 0:
        s["head/kernel"] = (cfg.embed_dim[-1], cfg.nb_classes)
        s["head/bias"] = (cfg.nb_classes,)
    return s


def conv_mlp(x, w, prefix, act, grid):
    """MLP.call with DWConv, pvt_v2.py:77-139 (linear_sr False: the "relu" slot is the identity)."""
    B, N, _ = x.shape
    y = tf.dense(x, w[f"{prefix}/fc1/kernel"], w[f"{prefix}/fc1/bias"])
    y = tf.depthwise_conv2d(y.reshape(B, *grid, -1), w[f"{prefix}/dwconv/dwconv/depthwise_kernel"],
                            w[f"{prefix}/dwconv/dwconv/bias"], padding="same").reshape(B, N, -1)
    return tf.dense(tf.act(y, act), w[f"{prefix}/fc2/kernel"], w[f"{prefix}/fc2/bias"])


def block(x, w, prefix, cfg, j, grid):
    """Block.call, pvt_v2.py:283-297 (DropPath is the identity at inference)."""
    y = tf.norm(x, w, f"{prefix}/norm1", cfg.norm_layer)
    x = x + sr_attention(y, w, f"{prefix}/attn", cfg.nb_heads[j], cfg.sr_ratio[j], grid)
    y = tf.norm(x, w, f"{prefix}/norm2", cfg.norm_layer)
    return x + conv_mlp(y, w, f"{prefix}/mlp", cfg.act_layer, grid)


def forward_features(cfg, w, x, return_features=False):
    """PyramidVisionTransformerV2.forward_features, pvt_v2.py:381-405; PatchEmbeddings.call, layers/transformers.py."""
    features = OrderedDict()
    B = x.shape[0]
    k = 0
    for j in range(len(cfg.nb_blocks)):
        pe = f"patch_embed{j + 1}"
        _, s, p = patch_geometry(j)
        x = tf.conv2d(x, w[f"{pe}/proj/kernel"], w[f"{pe}/proj/bias"], stride=s, padding=p)
        grid = tuple(x.shape[1:3])
        x = tf.layer_norm(x.reshape(B, grid[0] * grid[1], -1), w[f"{pe}/norm/gamma"], w[f"{pe}/norm/beta"], 1e-5)
        features[f"patch_embedding_{j}"] = x
        for i in range(cfg.nb_blocks[j]):
            x = block(x, w, f"block{j + 1}/{i}", cfg, j, grid)
            features[f"block_{k}"] = x
            k += 1
        x = tf.norm(x, w, f"norm{j + 1}", cfg.norm_layer).reshape(B, *grid, -1)
        features[f"stage_{j}"] = x
    x = x.reshape(B, -1, cfg.embed_dim[-1])
    features["features_all"] = x
    x = x.mean(dim=1)
    features["features"] = x
    return (x, features) if return_features else x


def forward(cfg, w, x, return_features=False):
    """PyramidVisionTransformerV2.call, pvt_v2.py:407-414.  w: {name: tensor} in reference layouts; x: (B, H, W, C)
    preprocessed images."""
    w = {k: torch.as_tensor(v).double() for k, v in w.items()}
    x = torch.as_tensor(x).double()
    features = {}
    x = forward_features(cfg, w, x, return_features)
    if return_features:
        x, features = x
    if cfg.nb_classes > 0:
        x = tf.dense(x, w["head/kernel"], w["head/bias"])
    features["logits"] = x
    return (x, features) if return_features else x
