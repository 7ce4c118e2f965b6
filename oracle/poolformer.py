"""Oracle restatement of the reference PoolFormer forward (tfimm/architectures/poolformer.py), in float64 on the CPU.

Op for op what the reference computes, with no use of the identity the token-mixer kernel relies on: GN(x) is formed,
zero-padded for the "same" average pool (padded cells excluded from the count), and GN(x) is subtracted again."""
from collections import OrderedDict

import torch
import torch.nn.functional as F

EPS = 1e-5  # GroupNormalization's default (layers/norm.py)


def param_shapes(cfg):
    """Variable names (without the "<model>/" prefix and ":0") and shapes, in creation order (poolformer.py:119-276):
    the block's layer scales come first, created by its build() before its sublayers."""
    s = OrderedDict()
    s["patch_embed/proj/kernel"] = (7, 7, cfg.in_channels, cfg.embed_dim[0])
    s["patch_embed/proj/bias"] = (cfg.embed_dim[0],)
    for j, (dim, depth) in enumerate(zip(cfg.embed_dim, cfg.nb_blocks)):
        hid = int(dim * cfg.mlp_ratio[j])
        for k in range(depth):
            p = f"network/{2 * j}/{k}"
            s[f"{p}/layer_scale_1"] = (dim,)
            s[f"{p}/layer_scale_2"] = (dim,)
            for n in ("norm1", "norm2"):
                s[f"{p}/{n}/gamma"] = (dim,)
                s[f"{p}/{n}/beta"] = (dim,)
            s[f"{p}/mlp/fc1/kernel"] = (1, 1, dim, hid)
            s[f"{p}/mlp/fc1/bias"] = (hid,)
            s[f"{p}/mlp/fc2/kernel"] = (1, 1, hid, dim)
            s[f"{p}/mlp/fc2/bias"] = (dim,)
        if j < len(cfg.nb_blocks) - 1:
            s[f"network/{2 * j + 1}/proj/kernel"] = (3, 3, dim, cfg.embed_dim[j + 1])
            s[f"network/{2 * j + 1}/proj/bias"] = (cfg.embed_dim[j + 1],)
    s["norm/gamma"] = (cfg.embed_dim[-1],)
    s["norm/beta"] = (cfg.embed_dim[-1],)
    if cfg.nb_classes > 0:
        s["head/kernel"] = (cfg.embed_dim[-1], cfg.nb_classes)
        s["head/bias"] = (cfg.nb_classes,)
    return s


def group_norm1(x, gamma, beta, eps=EPS):
    """GroupNormalization(nb_groups=1) of NHWC x: moments over (H, W, C) per image, biased variance."""
    mean = x.mean(dim=(1, 2, 3), keepdim=True)
    var = ((x - mean) ** 2).mean(dim=(1, 2, 3), keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * gamma + beta


def avg_pool3_same(x):
    """AveragePooling2D(3, strides=1, padding="same") of NHWC x: padded cells are excluded from the count."""
    y = F.avg_pool2d(x.permute(0, 3, 1, 2), 3, stride=1, padding=1, count_include_pad=False)
    return y.permute(0, 2, 3, 1)


def token_mixer(x, gamma, beta, ls1, eps=EPS):
    """x + ls1 * (pool(GN(x)) - GN(x)) (poolformer.py:189-194)."""
    n = group_norm1(x, gamma, beta, eps)
    return x + ls1 * (avg_pool3_same(n) - n)


def _conv(x, kernel, bias, stride, pad):
    """ZeroPadding2D(pad) then a VALID Conv2D with a TF (kh, kw, in, out) kernel, NHWC."""
    y = F.conv2d(x.permute(0, 3, 1, 2), kernel.permute(3, 2, 0, 1), bias, stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1)


def forward(cfg, w, x, return_features=False):
    """cfg: PoolFormerConfig; w: {name: tensor} in reference layouts; x: (B, H, W, C) preprocessed images."""
    w = {k: torch.as_tensor(v).double() for k, v in w.items()}
    x = torch.as_tensor(x).double()
    feats = OrderedDict()
    x = _conv(x, w["patch_embed/proj/kernel"], w["patch_embed/proj/bias"], 4, 2)
    feats["patch_embedding"] = x
    for j, depth in enumerate(cfg.nb_blocks):
        for k in range(depth):
            p = f"network/{2 * j}/{k}"
            x = token_mixer(x, w[f"{p}/norm1/gamma"], w[f"{p}/norm1/beta"], w[f"{p}/layer_scale_1"])
            h = group_norm1(x, w[f"{p}/norm2/gamma"], w[f"{p}/norm2/beta"])
            h = h @ w[f"{p}/mlp/fc1/kernel"][0, 0] + w[f"{p}/mlp/fc1/bias"]
            h = F.gelu(h)
            h = h @ w[f"{p}/mlp/fc2/kernel"][0, 0] + w[f"{p}/mlp/fc2/bias"]
            x = x + w[f"{p}/layer_scale_2"] * h
            feats[f"stage_{j}/block_{k}"] = x
        if j < len(cfg.nb_blocks) - 1:
            x = _conv(x, w[f"network/{2 * j + 1}/proj/kernel"], w[f"network/{2 * j + 1}/proj/bias"], 2, 1)
            feats[f"stage_{j}/downsample"] = x
    x = group_norm1(x, w["norm/gamma"], w["norm/beta"])
    feats["features_all"] = x
    x = x.mean(dim=(1, 2))
    feats["features"] = x
    if cfg.nb_classes > 0:
        x = x @ w["head/kernel"] + w["head/bias"]
    feats["logits"] = x
    return (x, feats) if return_features else x
