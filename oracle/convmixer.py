"""Oracle restatement of the reference ConvMixer forward (tfimm/architectures/convmixer.py), in float64 on the CPU.

Op for op what the reference computes: every BatchNorm is applied where the reference applies it, after its
activation, with no folding; the depthwise convolution zero-pads x itself ("same")."""
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

EPS = 1e-5  # the reference's "batch_norm" factory (layers/factory.py)


def param_shapes(cfg):
    """Variable names (without the "<model>/" prefix and ":0") and shapes, in creation order: the trainable variables,
    then each BN's moving statistics."""
    s = OrderedDict()
    C, k = cfg.embed_dim, cfg.kernel_size
    bns = ["stem/2"]
    s["stem/0/kernel"] = (*cfg.patch_size, cfg.in_channels, C)
    s["stem/0/bias"] = (C,)
    s["stem/2/gamma"] = (C,)
    s["stem/2/beta"] = (C,)
    for j in range(cfg.depth):
        p = f"blocks/{j}"
        s[f"{p}/0/fn/0/depthwise_kernel"] = (k, k, C, 1)
        s[f"{p}/0/fn/0/bias"] = (C,)
        s[f"{p}/0/fn/2/gamma"] = (C,)
        s[f"{p}/0/fn/2/beta"] = (C,)
        s[f"{p}/1/kernel"] = (1, 1, C, C)
        s[f"{p}/1/bias"] = (C,)
        s[f"{p}/3/gamma"] = (C,)
        s[f"{p}/3/beta"] = (C,)
        bns += [f"{p}/0/fn/2", f"{p}/3"]
    if cfg.nb_classes > 0:
        s["head/kernel"] = (C, cfg.nb_classes)
        s["head/bias"] = (cfg.nb_classes,)
    for b in bns:
        s[f"{b}/moving_mean"] = (C,)
        s[f"{b}/moving_variance"] = (C,)
    return s


def act(x, name):
    if name == "relu":
        return torch.relu(x)
    if name == "gelu":  # Keras default: the exact erf form
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    raise ValueError(name)


def batch_norm(x, w, prefix, eps=EPS):
    """Inference BatchNormalization with the moving statistics, NHWC."""
    return ((x - w[f"{prefix}/moving_mean"]) / torch.sqrt(w[f"{prefix}/moving_variance"] + eps) * w[f"{prefix}/gamma"]
            + w[f"{prefix}/beta"])


def depthwise_same(x, kernel, bias):
    """DepthwiseConv2D(k, padding="same", stride 1) with a (k, k, C, 1) kernel and bias: x zero-padded by (k - 1) / 2 on
    every side (k odd), NHWC."""
    k, C = kernel.shape[0], kernel.shape[2]
    pad = (k - 1) // 2
    xin = F.pad(x.permute(0, 3, 1, 2), (pad, pad, pad, pad))
    wt = kernel[..., 0].permute(2, 0, 1)[:, None]          # (C, 1, k, k)
    return F.conv2d(xin, wt, bias, groups=C).permute(0, 2, 3, 1)


def forward(cfg, w, x, return_features=False):
    """cfg: ConvMixerConfig; w: {name: tensor} in reference layouts; x: (B, H, W, C) preprocessed images."""
    w = {k: torch.as_tensor(v).double() for k, v in w.items()}
    x = torch.as_tensor(x).double()
    feats = OrderedDict()
    p = cfg.patch_size
    x = F.conv2d(x.permute(0, 3, 1, 2), w["stem/0/kernel"].permute(3, 2, 0, 1), w["stem/0/bias"], stride=p)
    x = batch_norm(act(x.permute(0, 2, 3, 1), cfg.act_layer), w, "stem/2")
    feats["stem"] = x
    for j in range(cfg.depth):
        b = f"blocks/{j}"
        r = x
        x = depthwise_same(x, w[f"{b}/0/fn/0/depthwise_kernel"], w[f"{b}/0/fn/0/bias"])
        x = batch_norm(act(x, cfg.act_layer), w, f"{b}/0/fn/2") + r
        x = x @ w[f"{b}/1/kernel"][0, 0] + w[f"{b}/1/bias"]
        x = batch_norm(act(x, cfg.act_layer), w, f"{b}/3")
        feats[f"block_{j}"] = x
    feats["features_all"] = x
    x = x.mean(dim=(1, 2))
    feats["features"] = x
    if cfg.nb_classes > 0:
        x = x @ w["head/kernel"] + w["head/bias"]
    feats["logits"] = x
    return (x, feats) if return_features else x
