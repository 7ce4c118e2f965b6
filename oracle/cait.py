"""Oracle restatement of the reference CaiT forward (tfimm/architectures/cait.py), in float64 on the CPU."""
from collections import OrderedDict

import torch

from . import tf_ops as tf


def grid_size(cfg, input_size=None):
    h, w = input_size or cfg.input_size
    return h // cfg.patch_size, w // cfg.patch_size


def interpolate_pos_embeddings(pos_embed, src_grid, tgt_grid):
    """layers/transformers.py:13-47 with nb_tokens = 0: tf.image.resize on the grid, which returns float32 whatever its
    input, cast back."""
    if tuple(src_grid) == tuple(tgt_grid):
        return pos_embed
    grid = pos_embed.reshape(1, *src_grid, -1)
    grid = tf.resize_bicubic(grid, tgt_grid).float().to(pos_embed.dtype)
    return grid.reshape(1, tgt_grid[0] * tgt_grid[1], -1)


def mlp(x, w, prefix, act):
    return tf.dense(tf.act(tf.dense(x, w[f"{prefix}/fc1/kernel"], w[f"{prefix}/fc1/bias"]), act),
                    w[f"{prefix}/fc2/kernel"], w[f"{prefix}/fc2/bias"])


def _bias(w, key):
    return w.get(key)


def talking_head_attention(x, w, prefix, nb_heads):
    """TalkingHeadAttention.call, cait.py:232-258."""
    B, N, D = x.shape
    dh = D // nb_heads
    qkv = tf.dense(x, w[f"{prefix}/qkv/kernel"], _bias(w, f"{prefix}/qkv/bias"))
    q, k, v = qkv.reshape(B, N, 3, nb_heads, dh).permute(2, 0, 3, 1, 4)
    q = dh ** -0.5 * q
    attn = (q @ k.transpose(-1, -2)).permute(0, 2, 3, 1)                      # (B, N, N, H)
    attn = tf.dense(attn, w[f"{prefix}/proj_l/kernel"], w[f"{prefix}/proj_l/bias"]).permute(0, 3, 1, 2)
    attn = torch.softmax(attn, dim=-1).permute(0, 2, 3, 1)
    attn = tf.dense(attn, w[f"{prefix}/proj_w/kernel"], w[f"{prefix}/proj_w/bias"]).permute(0, 3, 1, 2)
    x = (attn @ v).permute(0, 2, 1, 3).reshape(B, N, D)
    return tf.dense(x, w[f"{prefix}/proj/kernel"], w[f"{prefix}/proj/bias"])


def class_attention(x, w, prefix, nb_heads):
    """ClassAttention.call, cait.py:118-146."""
    B, N, D = x.shape
    dh = D // nb_heads
    q = tf.dense(x[:, 0], w[f"{prefix}/q/kernel"], _bias(w, f"{prefix}/q/bias")).reshape(B, 1, nb_heads, dh)
    q = q.permute(0, 2, 1, 3) * dh ** -0.5
    k = tf.dense(x, w[f"{prefix}/k/kernel"], _bias(w, f"{prefix}/k/bias")).reshape(B, N, nb_heads, dh).permute(0, 2, 1, 3)
    v = tf.dense(x, w[f"{prefix}/v/kernel"], _bias(w, f"{prefix}/v/bias")).reshape(B, N, nb_heads, dh).permute(0, 2, 1, 3)
    attn = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
    x = (attn @ v).permute(0, 2, 1, 3).reshape(B, 1, D)
    return tf.dense(x, w[f"{prefix}/proj/kernel"], w[f"{prefix}/proj/bias"])


def layer_scale_block(x, w, prefix, cfg):
    """LayerScaleBlock.call, cait.py:300-314."""
    x = x + w[f"{prefix}/gamma_1"] * talking_head_attention(tf.norm(x, w, f"{prefix}/norm1", cfg.norm_layer), w,
                                                           f"{prefix}/attn", cfg.nb_heads)
    return x + w[f"{prefix}/gamma_2"] * mlp(tf.norm(x, w, f"{prefix}/norm2", cfg.norm_layer), w, f"{prefix}/mlp",
                                            cfg.act_layer)


def class_attention_block(x, w, prefix, cfg):
    """LayerScaleBlockClassAttention.call, cait.py:188-204: only row 0 changes."""
    x_cls = x[:, :1]
    u = tf.norm(x, w, f"{prefix}/norm1", cfg.norm_layer)
    x_cls = x_cls + w[f"{prefix}/gamma_1"] * class_attention(u, w, f"{prefix}/attn", cfg.nb_heads)
    x_cls = x_cls + w[f"{prefix}/gamma_2"] * mlp(tf.norm(x_cls, w, f"{prefix}/norm2", cfg.norm_layer), w,
                                                 f"{prefix}/mlp", cfg.act_layer)
    return torch.cat((x_cls, x[:, 1:]), dim=1)


def forward_features(cfg, w, x, return_features=False):
    """CaiT.forward_features, cait.py:391-424."""
    features = OrderedDict()
    B = x.shape[0]
    x = tf.conv2d(x, w["patch_embed/proj/kernel"], w["patch_embed/proj/bias"], stride=cfg.patch_size)
    grid = tuple(x.shape[1:3])
    x = x.reshape(B, -1, x.shape[-1])
    pos = w["pos_embed"]
    if getattr(cfg, "interpolate_input", False):
        pos = interpolate_pos_embeddings(pos, grid_size(cfg), grid)
    x = x + pos
    features["patch_embedding"] = x
    for j in range(cfg.nb_blocks):
        x = layer_scale_block(x, w, f"blocks/{j}", cfg)
        features[f"block_{j}"] = x
    x = torch.cat((w["cls_token"].expand(B, -1, -1), x), dim=1)
    features["features_cls_token"] = x
    for j in range(2):
        x = class_attention_block(x, w, f"blocks_token_only/{j}", cfg)
        features[f"block_cls_token_{j}"] = x
    x = tf.norm(x, w, "norm", cfg.norm_layer)
    features["features_all"] = x
    x = x[:, 0]
    features["features"] = x
    return (x, features) if return_features else x


def forward(cfg, w, x, return_features=False):
    """CaiT.call, cait.py:426-433.  w: {name: tensor} in reference layouts; x: (B, H, W, C) preprocessed images."""
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
