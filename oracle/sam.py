"""Oracle restatement of the reference Segment Anything image encoder
(tfimm/architectures/segment_anything/image_encoder.py), in whatever dtype the weights come in (float64 for the tests).
It follows the reference literally: the window partition pads the normalised activations with zeros and projects the
padded rows, the (N, N) score matrix is materialised, and the relative-position tables are gathered per query / key.
"""
from collections import OrderedDict

import torch

from . import tf_ops as tf

_LN_EPS = {"layer_norm": 1e-5, "layer_norm_eps_1e-6": 1e-6}


def param_shapes(cfg):
    """Every variable of the reference SAM model (image encoder, prompt encoder, mask decoder): names without the
    "<model>/" prefix and ":0", and shapes, from image_encoder.py:171-229,363-492, common.py:6-36,
    prompt_encoder.py:30-75,187-215,264-270, mask_decoder.py:45-76,170-241 and transformer.py:8-260."""
    s = OrderedDict()
    D, p, E = cfg.encoder_embed_dim, cfg.encoder_patch_size, cfg.embed_dim
    dh, hid = D // cfg.encoder_nb_heads, int(D * cfg.encoder_mlp_ratio)
    gh, gw = cfg.input_size[0] // p, cfg.input_size[1] // p

    def dense(prefix, n_in, n_out, bias=True):
        s[f"{prefix}/kernel"] = (n_in, n_out)
        if bias:
            s[f"{prefix}/bias"] = (n_out,)

    def norm(prefix, n):
        s[f"{prefix}/gamma"] = (n,)
        s[f"{prefix}/beta"] = (n,)

    s["image_encoder/pos_embed"] = (1, gh, gw, D)
    s["image_encoder/patch_embed/proj/kernel"] = (p, p, cfg.in_channels, D)
    s["image_encoder/patch_embed/proj/bias"] = (D,)
    for j in range(cfg.encoder_nb_blocks):
        b = f"image_encoder/blocks/{j}"
        window = j not in cfg.encoder_global_attn_indices
        norm(f"{b}/norm1", D)
        dense(f"{b}/attn/qkv", D, 3 * D, cfg.encoder_qkv_bias)
        dense(f"{b}/attn/proj", D, D)
        # RelPosAttention.build sees the (windowed) input: (2 * extent - 1, head_dim)
        s[f"{b}/attn/rel_pos_h"] = (2 * (cfg.encoder_window_size if window else gh) - 1, dh)
        s[f"{b}/attn/rel_pos_w"] = (2 * (cfg.encoder_window_size if window else gw) - 1, dh)
        norm(f"{b}/norm2", D)
        dense(f"{b}/mlp/lin1", D, hid)
        dense(f"{b}/mlp/lin2", hid, D)
    s["image_encoder/neck/0/kernel"] = (1, 1, D, E)
    norm("image_encoder/neck/1", E)
    s["image_encoder/neck/2/kernel"] = (3, 3, E, E)
    norm("image_encoder/neck/3", E)

    mh = cfg.prompt_mask_hidden_dim
    s["prompt_encoder/pe_layer/positional_encoding_gaussian_matrix"] = (2, E // 2)
    for j in range(4):
        s[f"prompt_encoder/point_embeddings/{j}/weight"] = (1, E)
    s["prompt_encoder/not_a_point_embed/weight"] = (1, E)
    s["prompt_encoder/mask_downscaling/0/kernel"] = (2, 2, 1, mh // 4)
    s["prompt_encoder/mask_downscaling/0/bias"] = (mh // 4,)
    norm("prompt_encoder/mask_downscaling/1", mh // 4)
    s["prompt_encoder/mask_downscaling/3/kernel"] = (2, 2, mh // 4, mh)
    s["prompt_encoder/mask_downscaling/3/bias"] = (mh,)
    norm("prompt_encoder/mask_downscaling/4", mh)
    s["prompt_encoder/mask_downscaling/6/kernel"] = (1, 1, mh, E)
    s["prompt_encoder/mask_downscaling/6/bias"] = (E,)
    s["prompt_encoder/no_mask_embed/weight"] = (1, E)

    K = cfg.nb_multimask_outputs + 1
    s["mask_decoder/iou_token/weight"] = (1, E)
    s["mask_decoder/mask_tokens/weight"] = (K, E)
    t = "mask_decoder/transformer"

    def attention(prefix, rate):
        for n in ("q_proj", "k_proj", "v_proj"):
            dense(f"{prefix}/{n}", E, E // rate)
        dense(f"{prefix}/out_proj", E // rate, E)

    for j in range(cfg.decoder_nb_blocks):
        b = f"{t}/layers/{j}"
        attention(f"{b}/self_attn", 1)
        norm(f"{b}/norm1", E)
        attention(f"{b}/cross_attn_token_to_image", 2)
        norm(f"{b}/norm2", E)
        dense(f"{b}/mlp/lin1", E, cfg.decoder_mlp_channels)
        dense(f"{b}/mlp/lin2", cfg.decoder_mlp_channels, E)
        norm(f"{b}/norm3", E)
        attention(f"{b}/cross_attn_image_to_token", 2)
        norm(f"{b}/norm4", E)
    attention(f"{t}/final_attn_token_to_image", 2)
    norm(f"{t}/norm_final_attn", E)
    # Conv2DTranspose kernels are (kh, kw, out, in)
    s["mask_decoder/output_upscaling/0/kernel"] = (2, 2, E // 4, E)
    s["mask_decoder/output_upscaling/0/bias"] = (E // 4,)
    norm("mask_decoder/output_upscaling/1", E // 4)
    s["mask_decoder/output_upscaling/3/kernel"] = (2, 2, E // 8, E // 4)
    s["mask_decoder/output_upscaling/3/bias"] = (E // 8,)
    for j in range(K):
        dense(f"mask_decoder/output_hypernetworks_mlps/{j}/layers/0", E, E)
        dense(f"mask_decoder/output_hypernetworks_mlps/{j}/layers/1", E, E)
        dense(f"mask_decoder/output_hypernetworks_mlps/{j}/layers/2", E, E // 8)
    n_in = E
    for k in range(cfg.decoder_iou_head_depth):
        n_out = K if k == cfg.decoder_iou_head_depth - 1 else cfg.decoder_iou_hidden_dim
        dense(f"mask_decoder/iou_prediction_head/layers/{k}", n_in, n_out)
        n_in = n_out
    return s


def _linear_weights(n_in, n_out, dtype, device):
    """(n_out, n_in) matrix of TF2's bilinear resize along one axis: half-pixel centres, source clamped to the image."""
    src = ((torch.arange(n_out, dtype=torch.float64) + 0.5) * (n_in / n_out) - 0.5).clamp(min=0.0)
    lo = src.floor().long().clamp(max=n_in - 1)
    hi = (lo + 1).clamp(max=n_in - 1)
    frac = src - lo.double()
    m = torch.zeros(n_out, n_in, dtype=torch.float64)
    m[torch.arange(n_out), lo] += 1.0 - frac
    m[torch.arange(n_out), hi] += frac
    return m.to(dtype=dtype, device=device)


def resize_bilinear(images, size):
    """tf.image.resize(images, size, method="bilinear") on NHWC."""
    _, h, w, _ = images.shape
    mh = _linear_weights(h, size[0], images.dtype, images.device)
    mw = _linear_weights(w, size[1], images.dtype, images.device)
    return torch.einsum("pw,bowc->bopc", mw, torch.einsum("oh,bhwc->bowc", mh, images))


def get_rel_pos(q_size, k_size, rel_pos, interpolate_pos):
    """image_encoder.py:76-118 (q_size == k_size here): R[qi, ki] = rel_pos[qi - ki + k_size - 1]."""
    max_rel_dist = 2 * max(q_size, k_size) - 1
    if interpolate_pos:
        rel_pos = resize_bilinear(rel_pos[None, None], (1, max_rel_dist))[0, 0]
    q = torch.arange(q_size)[:, None] * max(k_size / q_size, 1.0)
    k = torch.arange(k_size)[None, :] * max(q_size / k_size, 1.0)
    idx = ((q - k) + (k_size - 1) * max(q_size / k_size, 1.0)).long()
    return rel_pos[idx]


def add_decomposed_rel_pos(attn, q, rel_pos_h, rel_pos_w, q_size, k_size, interpolate_pos):
    """image_encoder.py:121-168."""
    qh, qw = q_size
    kh, kw = k_size
    n, _, c = q.shape
    r_q = q.reshape(n, qh, qw, c)
    rh = get_rel_pos(qh, kh, rel_pos_h, interpolate_pos)
    rw = get_rel_pos(qw, kw, rel_pos_w, interpolate_pos)
    rel_h = torch.einsum("nhwc,hkc->nhwk", r_q, rh)[..., None]
    rel_w = torch.einsum("nhwc,wkc->nhwk", r_q, rw)[..., None, :]
    attn = attn.reshape(n, qh, qw, kh, kw) + rel_h + rel_w
    return attn.reshape(n, qh * qw, kh * kw)


def window_partition(x, ws):
    """image_encoder.py:11-43."""
    n, h, w, c = x.shape
    pad_h, pad_w = (ws - h % ws) % ws, (ws - w % ws) % ws
    if pad_h or pad_w:
        x = torch.nn.functional.pad(x, (0, 0, 0, pad_w, 0, pad_h))
    hp, wp = h + pad_h, w + pad_w
    x = x.reshape(n, hp // ws, ws, wp // ws, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws, ws, c)
    return x, (hp, wp)


def window_unpartition(windows, ws, pad_hw, hw):
    """image_encoder.py:46-73."""
    hp, wp = pad_hw
    h, w = hw
    n = windows.shape[0] // ((hp // ws) * (wp // ws))
    x = windows.reshape(n, hp // ws, wp // ws, ws, ws, -1).permute(0, 1, 3, 2, 4, 5).reshape(n, hp, wp, -1)
    return x[:, :h, :w]


def rel_pos_attention(x, w, prefix, cfg):
    """RelPosAttention.call, image_encoder.py:231-263."""
    n, h, wd, c = x.shape
    H = cfg.encoder_nb_heads
    qkv = tf.dense(x, w[f"{prefix}/qkv/kernel"], w.get(f"{prefix}/qkv/bias") if cfg.encoder_qkv_bias else None)
    qkv = qkv.reshape(n, h * wd, 3, H, -1).permute(2, 0, 3, 1, 4).reshape(3, n * H, h * wd, -1)
    q, k, v = qkv[0], qkv[1], qkv[2]
    attn = (q @ k.transpose(-1, -2)) * (c // H) ** -0.5
    attn = add_decomposed_rel_pos(attn, q, w[f"{prefix}/rel_pos_h"], w[f"{prefix}/rel_pos_w"], (h, wd), (h, wd),
                                  not cfg.fixed_input_size)
    y = (tf.softmax(attn) @ v).reshape(n, H, h, wd, -1).permute(0, 2, 3, 1, 4).reshape(n, h, wd, -1)
    return tf.dense(y, w[f"{prefix}/proj/kernel"], w[f"{prefix}/proj/bias"])


def block(x, w, prefix, cfg, window_size):
    """ImageEncoderBlock.call, image_encoder.py:340-360 (DropPath / Dropout are the identity at inference)."""
    eps = _LN_EPS[cfg.encoder_norm_layer]
    shortcut = x
    y = tf.layer_norm(x, w[f"{prefix}/norm1/gamma"], w[f"{prefix}/norm1/beta"], eps)
    if window_size > 0:
        hw = y.shape[1:3]
        y, pad_hw = window_partition(y, window_size)
    y = rel_pos_attention(y, w, f"{prefix}/attn", cfg)
    if window_size > 0:
        y = window_unpartition(y, window_size, pad_hw, hw)
    x = y + shortcut
    y = tf.layer_norm(x, w[f"{prefix}/norm2/gamma"], w[f"{prefix}/norm2/beta"], eps)
    y = tf.dense(y, w[f"{prefix}/mlp/lin1/kernel"], w[f"{prefix}/mlp/lin1/bias"])   # MLPBlock, common.py:38-44
    y = tf.dense(tf.act(y, cfg.encoder_act_layer), w[f"{prefix}/mlp/lin2/kernel"], w[f"{prefix}/mlp/lin2/bias"])
    return x + y


def image_encoder(cfg, w, x, return_features=False):
    """ImageEncoder.call, image_encoder.py:494-515."""
    e = "image_encoder"
    features = OrderedDict()
    x = tf.conv2d(x, w[f"{e}/patch_embed/proj/kernel"], w[f"{e}/patch_embed/proj/bias"], stride=cfg.encoder_patch_size)
    pos = w[f"{e}/pos_embed"]
    if not cfg.fixed_input_size:
        pos = resize_bilinear(pos, x.shape[1:3])
    x = x + pos
    features["patch_embedding"] = x
    for j in range(cfg.encoder_nb_blocks):
        ws = 0 if j in cfg.encoder_global_attn_indices else cfg.encoder_window_size
        x = block(x, w, f"{e}/blocks/{j}", cfg, ws)
        features[f"block_{j}"] = x
    x = tf.conv2d(x, w[f"{e}/neck/0/kernel"])
    x = tf.layer_norm(x, w[f"{e}/neck/1/gamma"], w[f"{e}/neck/1/beta"], 1e-6)
    x = tf.conv2d(x, w[f"{e}/neck/2/kernel"], padding="same")
    x = tf.layer_norm(x, w[f"{e}/neck/3/gamma"], w[f"{e}/neck/3/beta"], 1e-6)
    features["neck"] = x
    return (x, features) if return_features else x
