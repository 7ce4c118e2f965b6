"""Oracle restatement of the reference MLP-Mixer / gMixer / ResMLP / gMLP forward (tfimm/architectures/mlp_mixer.py),
in float64 on the CPU."""
from collections import OrderedDict

import torch

_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}


def hidden_dims(cfg):
    """(token MLP hidden, channel MLP hidden): mlp_mixer.py:95 (MixerBlock), 154 (ResBlock), 209 (SpatialGatingBlock)."""
    D = cfg.embed_dim
    if cfg.block_layer == "mixer_block":
        return int(cfg.mlp_ratio[0] * D), int(cfg.mlp_ratio[1] * D)
    return 0, int(D * cfg.mlp_ratio[1])


def param_shapes(cfg):
    """Variable names (without the "<model>/" prefix and ":0") and shapes, in creation order.
    mlp_mixer.py:83-304; layers/transformers.py:316-414 (GluMLP, SpatialGatingUnit, GatedMLP); layers/norm.py:7-34."""
    D = cfg.embed_dim
    N = (cfg.input_size[0] // cfg.patch_size) * (cfg.input_size[1] // cfg.patch_size)
    Ht, Hc = hidden_dims(cfg)
    s = OrderedDict()

    def norm(p, n, kind=cfg.norm_layer):
        names = ("alpha", "beta") if kind == "affine" else ("gamma", "beta")
        for k in names:
            s[f"{p}/{k}"] = (n,)

    def dense(p, i, o):
        s[f"{p}/kernel"] = (i, o)
        s[f"{p}/bias"] = (o,)

    def mlp(p, hidden, dim):
        dense(f"{p}/fc1", dim, hidden)
        if cfg.mlp_layer == "gated_mlp":
            norm(f"{p}/gate/norm", hidden // 2, "layer_norm")
            dense(f"{p}/gate/proj", N, N)
        dense(f"{p}/fc2", hidden // 2 if cfg.mlp_layer in ("glu_mlp", "gated_mlp") else hidden, dim)

    s["stem/proj/kernel"] = (cfg.patch_size, cfg.patch_size, cfg.in_channels, D)
    s["stem/proj/bias"] = (D,)
    if cfg.stem_norm:
        norm("stem/norm", D)
    for j in range(cfg.nb_blocks):
        p = f"blocks/{j}"
        if cfg.block_layer == "mixer_block":
            norm(f"{p}/norm1", D)
            mlp(f"{p}/mlp_tokens", Ht, N)
            norm(f"{p}/norm2", D)
            mlp(f"{p}/mlp_channels", Hc, D)
        elif cfg.block_layer == "res_block":
            s[f"{p}/ls1"] = (D,)
            s[f"{p}/ls2"] = (D,)
            norm(f"{p}/norm1", D)
            dense(f"{p}/linear_tokens", N, N)
            norm(f"{p}/norm2", D)
            mlp(f"{p}/mlp_channels", Hc, D)
        else:
            norm(f"{p}/norm", D)
            mlp(f"{p}/mlp_channels", Hc, D)
    norm("norm", D)
    if cfg.nb_classes > 0:
        dense("head", D, cfg.nb_classes)
    return s


def _act(x, name):
    if name == "gelu":
        return 0.5 * x * (1.0 + torch.erf(x / 2 ** 0.5))
    if name in ("swish", "silu"):
        return x * torch.sigmoid(x)
    raise ValueError(name)


def _norm(x, w, p, kind):
    if kind == "affine":
        return w[f"{p}/alpha"] * x + w[f"{p}/beta"]
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + _EPS[kind]) * w[f"{p}/gamma"] + w[f"{p}/beta"]


def _dense(x, w, p):
    return x @ w[f"{p}/kernel"] + w[f"{p}/bias"]


def _mlp(x, w, p, cfg):
    """MLP / GluMLP / GatedMLP (layers/transformers.py:208-214, 345-352, 407-414) on the last axis of x."""
    x = _dense(x, w, f"{p}/fc1")
    if cfg.mlp_layer == "glu_mlp":
        v, g = x.chunk(2, dim=-1)
        x = v * _act(g, cfg.act_layer)
    else:
        x = _act(x, cfg.act_layer)
    if cfg.mlp_layer == "gated_mlp":   # SpatialGatingUnit.call, transformers.py:376-383
        u, v = x.chunk(2, dim=-1)
        v = _norm(v, w, f"{p}/gate/norm", "layer_norm")
        v = _dense(v.transpose(1, 2), w, f"{p}/gate/proj").transpose(1, 2)
        x = u * v
    return _dense(x, w, f"{p}/fc2")


def forward(cfg, weights, images, return_features=False):
    """images: (B, H, W, C) -> logits (float64), optionally with the reference's features dict."""
    w = {k: torch.as_tensor(v).double() for k, v in weights.items()}
    x = torch.as_tensor(images).double()
    B, H, W, C = x.shape
    p = cfg.patch_size
    gh, gw = H // p, W // p
    # PatchEmbeddings: Conv2D(k = s = p) then flatten (layers/transformers.py:131-140)
    x = x[:, : gh * p, : gw * p].reshape(B, gh, p, gw, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, gh * gw, p * p * C)
    x = x @ w["stem/proj/kernel"].reshape(p * p * C, -1) + w["stem/proj/bias"]
    if cfg.stem_norm:
        x = _norm(x, w, "stem/norm", cfg.norm_layer)
    feats = OrderedDict(stem=x)
    for j in range(cfg.nb_blocks):
        q = f"blocks/{j}"
        if cfg.block_layer == "mixer_block":
            y = _norm(x, w, f"{q}/norm1", cfg.norm_layer).transpose(1, 2)
            x = x + _mlp(y, w, f"{q}/mlp_tokens", cfg).transpose(1, 2)
            x = x + _mlp(_norm(x, w, f"{q}/norm2", cfg.norm_layer), w, f"{q}/mlp_channels", cfg)
        elif cfg.block_layer == "res_block":
            y = _norm(x, w, f"{q}/norm1", cfg.norm_layer).transpose(1, 2)
            x = x + w[f"{q}/ls1"] * _dense(y, w, f"{q}/linear_tokens").transpose(1, 2)
            x = x + w[f"{q}/ls2"] * _mlp(_norm(x, w, f"{q}/norm2", cfg.norm_layer), w, f"{q}/mlp_channels", cfg)
        else:
            x = x + _mlp(_norm(x, w, f"{q}/norm", cfg.norm_layer), w, f"{q}/mlp_channels", cfg)
        feats[f"block_{j}"] = x
    x = _norm(x, w, "norm", cfg.norm_layer)
    feats["features_all"] = x
    x = x.mean(1)
    feats["features"] = x
    if cfg.nb_classes > 0:
        x = _dense(x, w, "head")
    feats["logits"] = x
    return (x, feats) if return_features else x
