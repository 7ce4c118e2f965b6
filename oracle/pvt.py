"""Oracle restatement of the reference PVT forward (tfimm/architectures/pvt.py), in float64 on the CPU."""
from collections import OrderedDict

import torch

from . import tf_ops as tf


def grid_sizes(cfg, input_size=None):
    """Each stage's grid: the VALID patch embeddings floor (PyramidVisionTransformerConfig.grid_size, pvt.py:85-94)."""
    h, w = input_size or cfg.input_size
    out = []
    for p in cfg.patch_size:
        h, w = h // p, w // p
        out.append((h, w))
    return out


def nb_tokens(cfg):
    return [0] * (len(cfg.nb_blocks) - 1) + [1]


def param_shapes(cfg):
    """Variable names (without the "<model>/" prefix and ":0") and shapes, in the order of the reference's
    ``weights``: pos_embed1 .. and cls_token, added by the model's build() (pvt.py:267-321), then the layers as Keras
    tracks them -- the patch embeddings, the blocks (the attention's q, kv, proj, sr, norm in __init__ order,
    pvt.py:136-151), the norm, the head."""
    s = OrderedDict()
    grids, ntok = grid_sizes(cfg), nb_tokens(cfg)
    for j, D in enumerate(cfg.embed_dim):
        s[f"pos_embed{j + 1}"] = (1, grids[j][0] * grids[j][1] + ntok[j], D)
    s["cls_token"] = (1, 1, cfg.embed_dim[-1])
    cin = cfg.in_channels
    for j, D in enumerate(cfg.embed_dim):
        p = cfg.patch_size[j]
        s[f"patch_embed{j + 1}/proj/kernel"] = (p, p, cin, D)
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
            s[f"{b}/mlp/fc2/kernel"] = (hid, D)
            s[f"{b}/mlp/fc2/bias"] = (D,)
    s["norm/gamma"] = (cfg.embed_dim[-1],)
    s["norm/beta"] = (cfg.embed_dim[-1],)
    if cfg.nb_classes > 0:
        s["head/kernel"] = (cfg.embed_dim[-1], cfg.nb_classes)
        s["head/bias"] = (cfg.nb_classes,)
    return s


def sr_attention(x, w, prefix, nb_heads, sr, grid):
    """SpatialReductionAttention.call, pvt.py:153-188."""
    B, N, D = x.shape
    dh = D // nb_heads
    q = tf.dense(x, w[f"{prefix}/q/kernel"], w.get(f"{prefix}/q/bias"))
    q = q.reshape(B, N, nb_heads, dh).permute(0, 2, 1, 3)
    if sr > 1:
        x = tf.conv2d(x.reshape(B, *grid, D), w[f"{prefix}/sr/kernel"], w[f"{prefix}/sr/bias"], stride=sr)
        x = tf.layer_norm(x.reshape(B, -1, D), w[f"{prefix}/norm/gamma"], w[f"{prefix}/norm/beta"], 1e-5)
    kv = tf.dense(x, w[f"{prefix}/kv/kernel"], w.get(f"{prefix}/kv/bias"))
    k, v = kv.reshape(B, -1, 2, nb_heads, dh).permute(2, 0, 3, 1, 4)
    attn = tf.softmax(dh ** -0.5 * (q @ k.transpose(-1, -2)))
    y = (attn @ v).permute(0, 2, 1, 3).reshape(B, N, D)
    return tf.dense(y, w[f"{prefix}/proj/kernel"], w[f"{prefix}/proj/bias"])


def block(x, w, prefix, cfg, j, grid):
    """Block.call, pvt.py:233-247 (DropPath is the identity at inference)."""
    y = tf.norm(x, w, f"{prefix}/norm1", cfg.norm_layer)
    x = x + sr_attention(y, w, f"{prefix}/attn", cfg.nb_heads[j], cfg.sr_ratio[j], grid)
    y = tf.norm(x, w, f"{prefix}/norm2", cfg.norm_layer)
    y = tf.act(tf.dense(y, w[f"{prefix}/mlp/fc1/kernel"], w[f"{prefix}/mlp/fc1/bias"]), cfg.act_layer)
    return x + tf.dense(y, w[f"{prefix}/mlp/fc2/kernel"], w[f"{prefix}/mlp/fc2/bias"])


def interpolate_pos_embeddings(pos_embed, src_grid, tgt_grid, ntok):
    """layers/transformers.py:13-47; tf.image.resize returns float32, cast back to the table's dtype."""
    if tuple(src_grid) == tuple(tgt_grid):
        return pos_embed
    grid = pos_embed[:, ntok:].reshape(1, *src_grid, -1)
    grid = tf.resize_bicubic(grid, tgt_grid).float().to(pos_embed.dtype).reshape(1, tgt_grid[0] * tgt_grid[1], -1)
    return torch.cat((pos_embed[:, :ntok], grid), dim=1)


def forward_features(cfg, w, x, return_features=False):
    """PyramidVisionTransformer.forward_features, pvt.py:360-400; PatchEmbeddings.call, layers/transformers.py."""
    features = OrderedDict()
    B = x.shape[0]
    src_grids, ntok = grid_sizes(cfg), nb_tokens(cfg)
    last = len(cfg.nb_blocks) - 1
    k = 0
    for j in range(len(cfg.nb_blocks)):
        pe = f"patch_embed{j + 1}"
        x = tf.conv2d(x, w[f"{pe}/proj/kernel"], w[f"{pe}/proj/bias"], stride=cfg.patch_size[j])
        grid = tuple(x.shape[1:3])
        x = tf.layer_norm(x.reshape(B, grid[0] * grid[1], -1), w[f"{pe}/norm/gamma"], w[f"{pe}/norm/beta"], 1e-5)
        features[f"patch_embedding_{j}"] = x
        if j == last:
            x = torch.cat((w["cls_token"].expand(B, -1, -1), x), dim=1)
        pos = w[f"pos_embed{j + 1}"]
        if getattr(cfg, "interpolate_input", False):
            pos = interpolate_pos_embeddings(pos, src_grids[j], grid, ntok[j])
        x = x + pos
        features[f"pos_embedding_{j}"] = x
        for _ in range(cfg.nb_blocks[j]):
            x = block(x, w, f"block{j + 1}/{k - sum(cfg.nb_blocks[:j])}", cfg, j, grid)
            features[f"block_{k}"] = x
            k += 1
        if j != last:
            x = x.reshape(B, *grid, -1)
        features[f"stage_{j}"] = x
    x = tf.norm(x, w, "norm", cfg.norm_layer)
    features["features_all"] = x
    x = x[:, 0]
    features["features"] = x
    return (x, features) if return_features else x


def forward(cfg, w, x, return_features=False):
    """PyramidVisionTransformer.call, pvt.py:402-409.  w: {name: tensor} in reference layouts; x: (B, H, W, C)
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
