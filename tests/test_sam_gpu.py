"""Segment Anything on the H100: the relative-position attention kernels against their float64 statement
(tests/sam_oracle.py) over global and windowed geometry, shadowed op-by-op forwards, whole-encoder accuracy against the
float64 oracle, CUDA-graph replay and raw uint8 pixels."""
import importlib
import sys
from copy import deepcopy

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def sam():
    """Registers the SAM models for this module and restores the registry afterwards (tests/test_api_cpu.py pins the
    exact list of models)."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.segment_anything.sam"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


def _nerr(out, ref):
    out, ref = out.double(), ref.double().to(out.device)
    return (out - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)


def _inputs(B, gh, gw, H, dh, window, dtype, seed=0, bias_scale=0.5):
    """qkv of LayerNorm-ed activations through a random projection (entries ~N(0, 1)), tables of the magnitude of
    trained SAM tables (~N(0, 0.5^2)), qkv bias ~N(0, bias_scale^2)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sh, sw = (window, window) if window else (gh, gw)
    qkv = torch.randn(B * gh * gw, 3 * H * dh, device="cuda", generator=g).to(dtype)
    rh = 0.5 * torch.randn(2 * sh - 1, dh, device="cuda", generator=g)
    rw = 0.5 * torch.randn(2 * sw - 1, dh, device="cuda", generator=g)
    pad = (bias_scale * torch.randn(3 * H * dh, device="cuda", generator=g)).to(dtype)
    return qkv, rh, rw, pad


GEOMETRY = [   # B, gh, gw, H, dh, window
    (1, 64, 64, 12, 64, 0),      # sam_vit_b global block
    (1, 64, 64, 16, 80, 0),      # sam_vit_h global block
    (2, 24, 40, 12, 64, 0),      # a smaller, non-square grid
    (1, 64, 64, 12, 64, 14),     # 64 -> 70: 5 x 5 windows of 196 tokens, padded on the right / bottom
    (4, 10, 10, 16, 80, 4),      # 10 -> 12: 3 x 3 windows, batch 4
    (3, 28, 28, 12, 64, 14),     # windows without padding
    (2, 64, 64, 16, 80, 14),
]


@pytest.mark.parametrize("B,gh,gw,H,dh,window", GEOMETRY)
def test_relpos_attention_bf16(B, gh, gw, H, dh, window):
    """Within the derived bound of tests/sam_oracle.py::relpos_bound (+ one bf16 ulp) of the float64 statement."""
    from oracle import shadow
    from sam_oracle import relpos_attention, relpos_bound
    from tfimm.backend import sam_ops

    qkv, rh, rw, pad = _inputs(B, gh, gw, H, dh, window, torch.bfloat16)
    scale = dh ** -0.5
    out = sam_ops.relpos_attention(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    torch.cuda.synchronize()
    ref = relpos_attention(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    bound = relpos_bound(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    ok, worst, _ = shadow.check("relpos_attention", out, ref, shadow._bounded(bound))
    print(f"relpos bf16 B={B} grid={gh}x{gw} H={H} dh={dh} window={window}: worst {worst:.3f} x bound")
    assert ok, worst


@pytest.mark.parametrize("B,gh,gw,H,dh,window", [(1, 32, 32, 12, 64, 0), (2, 10, 10, 16, 80, 4),
                                                  (1, 20, 20, 2, 6, 7)])
def test_relpos_attention_f32(B, gh, gw, H, dh, window):
    from sam_oracle import relpos_attention
    from tfimm.backend import sam_ops

    qkv, rh, rw, pad = _inputs(B, gh, gw, H, dh, window, torch.float32)
    scale = dh ** -0.5
    out = sam_ops.relpos_attention(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    ref = relpos_attention(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    assert _nerr(out, ref) < 1e-5


def test_padding_keys_are_keys_not_masked():
    """Window padding with large k / v biases: the kernel stays within its bound of the statement, while the same
    attention with the padding keys masked out is far outside that bound, so a kernel that masks them fails."""
    from oracle import shadow
    from sam_oracle import relpos_attention, relpos_bound
    from tfimm.backend import sam_ops

    B, gh, gw, H, dh, window = 2, 10, 10, 12, 64, 4
    qkv, rh, rw, pad = _inputs(B, gh, gw, H, dh, window, torch.bfloat16, seed=5, bias_scale=3.0)
    scale = dh ** -0.5
    out = sam_ops.relpos_attention(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    ref = relpos_attention(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    bound = relpos_bound(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
    assert shadow.check("relpos_attention", out, ref, shadow._bounded(bound))[0]
    # padding keys masked: the attention of each window over its real tokens only
    x = qkv.double().view(B, gh, gw, 3, H, dh)
    masked = torch.empty(B, gh, gw, H, dh, dtype=torch.float64, device="cuda")
    for wy in range(0, gh, window):
        for wx in range(0, gw, window):
            t = x[:, wy:wy + window, wx:wx + window]
            hh, ww = t.shape[1:3]
            q, k, v = t.reshape(B, hh * ww, 3, H, dh).permute(2, 0, 3, 1, 4)
            ty, tx = torch.arange(hh, device="cuda"), torch.arange(ww, device="cuda")
            Rh = rh.double()[ty[:, None] - ty[None, :] + window - 1]
            Rw = rw.double()[tx[:, None] - tx[None, :] + window - 1]
            qr = q.reshape(B, H, hh, ww, dh)
            rel = (torch.einsum("bhyxd,ykd->bhyxk", qr, Rh)[..., :, None]
                   + torch.einsum("bhyxd,xkd->bhyxk", qr, Rw)[..., None, :]).reshape(B, H, hh * ww, hh * ww)
            o = torch.softmax(scale * q @ k.transpose(-1, -2) + rel, -1) @ v
            masked[:, wy:wy + hh, wx:wx + ww] = o.permute(0, 2, 1, 3).reshape(B, hh, ww, H, dh)
    ok, worst, _ = shadow.check("relpos_attention", masked.reshape(B * gh * gw, H * dh).to(torch.bfloat16), ref,
                                shadow._bounded(bound, flips=False))
    assert not ok and worst > 10, worst


SMALL = {
    "pad": dict(input_size=(160, 160), encoder_embed_dim=128, encoder_nb_heads=2, encoder_nb_blocks=3,
                encoder_global_attn_indices=(1,), encoder_window_size=4, embed_dim=128, fixed_input_size=False),
    "dh80": dict(input_size=(128, 128), encoder_embed_dim=160, encoder_nb_heads=2, encoder_nb_blocks=2,
                 encoder_global_attn_indices=(1,), encoder_window_size=3, embed_dim=64),
    # head_dim 32: bf16 models run the fp32 kernel on the bf16 qkv values
    "dh32": dict(input_size=(128, 128), encoder_embed_dim=64, encoder_nb_heads=2, encoder_nb_blocks=2,
                 encoder_global_attn_indices=(1,), encoder_window_size=3, embed_dim=64),
}


def _model(name, precision, overrides=None, seed=7):
    import tfimm
    from oracle import params
    from oracle import sam as osam

    model = tfimm.create_model(name, precision=precision, device="cuda", **(overrides or {}))
    w = params.random_params(osam.param_shapes(model.cfg), seed=seed)
    model.load_weights_dict(w)
    return model, w


def _oracle(model, w, x):
    from oracle import sam as osam

    wd = {k: v.to("cuda", torch.float64) for k, v in w.items() if k.startswith("image_encoder/")}
    with torch.no_grad():
        return osam.image_encoder(model.cfg, wd, x.to("cuda", torch.float64))


@pytest.mark.parametrize("case", list(SMALL))
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_shadowed_forward_small(case, precision):
    from oracle import params
    from sam_oracle import shadowed_sam_ops

    model, _ = _model("sam_vit_b", precision, SMALL[case])
    x = params.test_images(2, *model.cfg.input_size).cuda()
    with shadowed_sam_ops() as census:
        model.image_encoder(x)
    census.assert_ok()
    assert "relpos_attention" in census.ops()


@pytest.mark.parametrize("dh,edge", [(64, 76), (80, 68)])
def test_relpos_attention_bf16_shared_memory_edge(dh, edge):
    """The largest global grid the tensor-core kernel takes runs within its bound; one more row and column is refused
    with an error (the host then uses the fp32 kernel, see the next test), and sam_ops predicts both."""
    from oracle import shadow
    from sam_oracle import relpos_attention, relpos_bound
    from tfimm.backend import sam_ops
    from tfimm.backend.lib import KernelLibraryError

    B, H, scale = 1, 2, dh ** -0.5
    assert sam_ops.relpos_attention_bf16_supported(dh, edge, edge)
    assert not sam_ops.relpos_attention_bf16_supported(dh, edge + 1, edge + 1)
    qkv, rh, rw, pad = _inputs(B, edge, edge, H, dh, 0, torch.bfloat16)
    out = sam_ops.relpos_attention(qkv, B, edge, edge, H, dh, scale, rh, rw, 0, pad)
    ref = relpos_attention(qkv, B, edge, edge, H, dh, scale, rh, rw, 0, pad)
    bound = relpos_bound(qkv, B, edge, edge, H, dh, scale, rh, rw, 0, pad)
    assert shadow.check("relpos_attention", out, ref, shadow._bounded(bound))[0]
    qkv, rh, rw, pad = _inputs(B, edge + 1, edge + 1, H, dh, 0, torch.bfloat16)
    with pytest.raises(KernelLibraryError, match="shared memory"):
        sam_ops.relpos_attention(qkv, B, edge + 1, edge + 1, H, dh, scale, rh, rw, 0, pad)


def test_large_global_grid_runs_the_fp32_kernel():
    """fixed_input_size=False at 1280 x 1280 (an 80 x 80 grid): the global block is beyond the tensor-core kernel's
    shared memory and runs the fp32 kernel on the bf16 values; every launch is checked."""
    from oracle import params
    from sam_oracle import shadowed_sam_ops

    model, w = _model("sam_vit_b", "bf16", dict(SMALL["pad"], encoder_nb_blocks=2))
    x = params.test_images(1, 1280, 1280).cuda()
    with shadowed_sam_ops() as census:
        y = model.image_encoder(x)
    census.assert_ok()
    rel = [r for r in census.rows if r["op"] == "relpos_attention"]
    assert any("qkv=f32(6400" in r["args"] and "window=0" in r["args"] for r in rel)
    assert any("qkv=bf16(6400" in r["args"] and "window=4" in r["args"] for r in rel)
    assert _nerr(y, _oracle(model, w, x.cpu())) < 2e-2


def test_shadowed_forward_sam_vit_b():
    """sam_vit_b at 1024 x 1024, batch 1, every launch checked; the relpos kernel ran in its global and its windowed
    form."""
    from oracle import params
    from sam_oracle import shadowed_sam_ops

    model, _ = _model("sam_vit_b", "bf16")
    x = params.test_images(1, 1024, 1024).cuda()
    with shadowed_sam_ops() as census:
        model.image_encoder(x)
    census.assert_ok()
    rel = [r for r in census.rows if r["op"] == "relpos_attention"]
    assert len(rel) == 12
    assert any("window=0" in r["args"] for r in rel) and any("window=14" in r["args"] for r in rel)
    print("\n".join(census._fmt(r) for r in rel))


@pytest.mark.parametrize("name", ["sam_vit_b", "sam_vit_h"])
def test_bf16_encoder_against_the_fp64_oracle(name):
    from oracle import params

    model, w = _model(name, "bf16")
    x = params.test_images(1, 1024, 1024)
    y = model.image_encoder(x.cuda())
    assert y.shape == (1, 64, 64, 256) and y.dtype == torch.float32
    err = _nerr(y, _oracle(model, w, x))
    print(f"{name} bf16 image embeddings vs fp64 oracle: normalised max error {err:.3e}")
    assert err < 1.5e-2   # measured 8.5e-3 (sam_vit_b) and 8.1e-3 (sam_vit_h) on an H100


@pytest.mark.parametrize("case", ["sam_vit_b"] + list(SMALL))
def test_fp32_encoder_against_the_fp64_oracle(case):
    from oracle import params

    model, w = _model("sam_vit_b", "fp32", SMALL.get(case))
    sizes = [model.cfg.input_size] + ([(128, 192)] if not model.cfg.fixed_input_size else [])
    for size in sizes:
        x = params.test_images(1, *size)
        err = _nerr(model.image_encoder(x.cuda()), _oracle(model, w, x))
        print(f"{case} fp32 {size}: normalised max error {err:.3e}")
        assert err < 1e-5


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_cuda_graph_replay_equals_eager(precision):
    from oracle import params

    model, _ = _model("sam_vit_b", precision, SMALL["pad"])
    x = params.test_images(2, *model.cfg.input_size).cuda()
    eager = model.image_encoder(x).clone()
    fwd = model.image_encoder.cuda_graph(2)
    assert torch.equal(fwd(x), eager)


@pytest.mark.parametrize("precision,tol", [("bf16", 2e-2), ("fp32", 1e-5)])
def test_uint8_pixels_equal_preprocessed_floats(precision, tol):
    import tfimm

    model, _ = _model("sam_vit_b", precision, SMALL["pad"])
    px = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (2, 160, 160, 3), dtype=np.uint8))
    pre = tfimm.create_preprocessing("sam_vit_b")
    a = model.image_encoder(px.cuda())
    b = model.image_encoder(pre(px.cuda()))
    assert _nerr(a, b) < tol
