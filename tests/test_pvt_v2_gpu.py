"""PVT v2 family on the H100: the fused ConvFFN and head-dim-32 spatial-reduction attention against their float64
statements (tests/pvt_v2_oracle.py) within their derived bounds, bitwise equality with pit_attention_bf16<32> where
N' = N, guard regions and determinism, and the six models in every precision.

``-s`` prints each census (worst error / bound, flip %) and the model-level error figures.
"""
import sys
from contextlib import nullcontext
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
if str(HERE) not in sys.path:
    sys.path.insert(0, str(HERE))

import pvt_v2_oracle as pvo  # noqa: E402
from tf32_oracle import tf32_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

NAMES = ["pvt_v2_b0", "pvt_v2_b1", "pvt_v2_b2", "pvt_v2_b3", "pvt_v2_b4", "pvt_v2_b5"]
DH = 32
# (B, gh, gw, C, hidden): the family's stage-0 / 1 shapes at 224 px (b0: C 32 / 64, b1-b4: 64 / 128 at mlp_ratio 8,
# b5: mlp_ratio 4), then partial and edge tiles of the 8 x 16 output tile
CONV_SHAPES = [(2, 56, 56, 32, 256), (2, 28, 28, 64, 512), (2, 56, 56, 64, 512), (2, 28, 28, 128, 1024),
               (2, 56, 56, 64, 256), (2, 28, 28, 128, 512),
               (3, 1, 1, 64, 128), (2, 1, 7, 32, 64), (2, 7, 1, 128, 64), (4, 5, 6, 64, 192), (2, 13, 17, 32, 256),
               (1, 55, 57, 128, 128), (256, 7, 7, 64, 128)]
# (B, N, N', H): b0's stages at 224 px, then N' across the 64-key block and ring edges, N across the query tiles
SR_SHAPES = [(4, 3136, 49, 1), (8, 784, 49, 2), (32, 196, 49, 5), (64, 49, 49, 8), (256, 196, 49, 5),
             (2, 197, 1, 2), (2, 130, 63, 5), (2, 65, 65, 8), (2, 300, 100, 2), (1, 257, 785, 8), (5, 1, 49, 2),
             (256, 3136, 49, 1)]


def _report(census, title):
    print(f"\n=== {title}\n" + census.table())
    census.assert_ok()


def conv_inputs(B, gh, gw, C, hidden, seed, hscale=1.0):
    g = torch.Generator().manual_seed(seed)
    M = B * gh * gw
    h = (torch.randn((M, C), generator=g) * hscale).to(torch.bfloat16)
    w1 = (torch.randn((hidden, C), generator=g) * C ** -0.5).to(torch.bfloat16)
    b1 = torch.randn(hidden, generator=g) * 0.5
    wdw = torch.randn((9, hidden), generator=g) / 3.0
    bdw = torch.randn(hidden, generator=g) * 0.5
    w2 = (torch.randn((C, hidden), generator=g) * hidden ** -0.5).to(torch.bfloat16)
    b2 = torch.randn(C, generator=g) * 0.5
    res = torch.randn((M, C), generator=g) * 2.0
    return [t.cuda() for t in (h, w1, b1, wdw, bdw, w2, b2, res)]


# ------------------------------------------------------------------------------------------- against the statement
@pytest.mark.parametrize("B,gh,gw,C,hidden", CONV_SHAPES)
def test_conv_mlp_within_its_bound(B, gh, gw, C, hidden):
    from tfimm.backend import pvt_v2_ops

    with pvo.shadowed_pvt_v2_ops() as census:
        for i, hscale in enumerate((1.0, 1e2)):
            h, w1, b1, wdw, bdw, w2, b2, res = conv_inputs(B, gh, gw, C, hidden, seed=gh * gw + C + i, hscale=hscale)
            pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu")
            # in place, as the model runs it
            pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu", out=res)
    _report(census, f"pvt_v2_conv_mlp_bf16 B={B} {gh}x{gw} C={C} hidden={hidden}")
    assert census.ops() == {"pvt_v2_conv_mlp_bf16"} and len(census.rows) == 4


@pytest.mark.parametrize("B,gh,gw,C,hidden", CONV_SHAPES[:6])
def test_conv_mlp_against_the_unfused_chain(B, gh, gw, C, hidden):
    """The unfused chain (fc1 GEMM, dwconv_bias_act, fc2 GEMM) is within the same bound; the share of outputs equal bit
    for bit to the fused kernel's is reported, not asserted (the GEMMs accumulate in another order)."""
    from tfimm.backend import ops, pvt_v2_ops

    h, w1, b1, wdw, bdw, w2, b2, res = conv_inputs(B, gh, gw, C, hidden, seed=C + hidden)
    fused = pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu")
    hid = ops.gemm(h, w1, bias=b1)
    hid = ops.dwconv_bias_act(hid.view(B, gh, gw, hidden), wdw, bdw, 3, 1, "symmetric", act="gelu")
    chain = ops.gemm(hid.view(-1, hidden), w2, bias=b2, residual=res)
    bound = pvo.conv_mlp_bound(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu")
    ref = pvo.conv_mlp_statement(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu")[3].to(torch.float32).double()
    for out in (fused, chain):
        assert ((out.double() - ref).abs() <= bound).all()
    same = (fused == chain).double().mean().item()
    print(f"\nBITWISE {B}x{gh}x{gw} C={C} hidden={hidden}: {100 * same:.2f} % of fused outputs equal the chain's")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("B,N,Nk,H", SR_SHAPES)
def test_sr_attention_dh32_within_its_bound(B, N, Nk, H, dtype):
    from tfimm.backend import pvt_v2_ops

    name = "pvt_v2_sr_attention_bf16" if dtype == torch.bfloat16 else "pvt_v2_sr_attention_f32"
    g = torch.Generator().manual_seed(N + Nk)
    q = torch.randn((B * N, H * DH), generator=g).to(dtype).cuda()
    kv = torch.randn((B * Nk, 2 * H * DH), generator=g).to(dtype).cuda()
    with pvo.shadowed_pvt_v2_ops() as census:
        getattr(pvt_v2_ops, name)(q, kv, B, N, Nk, H, DH, DH ** -0.5)
    _report(census, f"{name} B={B} N={N} N'={Nk} H={H}")
    assert census.ops() == {name}


@pytest.mark.parametrize("N", [1, 17, 49, 64, 65, 197, 785])
def test_dh32_equals_pit_attention_when_keys_are_the_queries(N):
    from tfimm.backend import pit_ops, pvt_v2_ops

    B, H = 3, 5
    g = torch.Generator().manual_seed(N)
    qkv = (torch.randn((B * N, 3 * H * DH), generator=g) * 2.0).to(torch.bfloat16).cuda()
    x = qkv.view(B * N, 3, H * DH)
    q, kv = x[:, 0].contiguous(), x[:, 1:].reshape(B * N, 2 * H * DH).contiguous()
    a = pvt_v2_ops.pvt_v2_sr_attention_bf16(q, kv, B, N, N, H, DH, DH ** -0.5)
    b = pit_ops.pit_attention_bf16(qkv, B, N, H, DH, DH ** -0.5)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------------------------- guard regions, determinism
G = 4096


def test_outputs_stay_inside_their_buffers():
    from tfimm.backend import lib, pvt_v2_ops

    handle = lib.load()
    for B, gh, gw, C, hidden in ((2, 13, 17, 64, 128), (1, 1, 7, 32, 64), (2, 9, 33, 128, 64)):
        h, w1, b1, wdw, bdw, w2, b2, res = conv_inputs(B, gh, gw, C, hidden, seed=9)
        buf = torch.full((G + res.numel() + G,), -12345.0, device="cuda")
        out = buf[G:G + res.numel()]
        assert handle.tfimm_b200_pvt_v2_conv_mlp_bf16(h.data_ptr(), w1.data_ptr(), b1.data_ptr(), wdw.data_ptr(),
                                                      bdw.data_ptr(), w2.data_ptr(), b2.data_ptr(), res.data_ptr(),
                                                      out.data_ptr(), B, gh, gw, C, hidden, 1, None) == 0
        torch.cuda.synchronize()
        assert (buf[:G] == -12345.0).all() and (buf[-G:] == -12345.0).all()
        assert not (out == -12345.0).any() and not out.isnan().any()
        assert torch.equal(out.view(-1, C), pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, res, B, gh,
                                                                           gw, "gelu"))
    for dtype, fn in ((torch.bfloat16, handle.tfimm_b200_pvt_v2_sr_attention_bf16),
                      (torch.float32, handle.tfimm_b200_pvt_v2_sr_attention_f32)):
        B, N, Nk, H = 3, 131, 49, 2
        q = torch.randn((B * N, H * DH)).to(dtype).cuda()
        kv = torch.randn((B * Nk, 2 * H * DH)).to(dtype).cuda()
        buf = torch.full((G + B * N * H * DH + G,), -12345.0, dtype=dtype, device="cuda")
        out = buf[G:G + B * N * H * DH]
        assert fn(q.data_ptr(), kv.data_ptr(), out.data_ptr(), B, N, Nk, H, DH, DH ** -0.5, None) == 0
        torch.cuda.synchronize()
        assert (buf[:G] == -12345.0).all() and (buf[-G:] == -12345.0).all()
        assert not (out == -12345.0).any() and not out.isnan().any()


def test_conv_mlp_refuses_other_shapes():
    from tfimm.backend import lib, pvt_v2_ops

    h, w1, b1, wdw, bdw, w2, b2, res = conv_inputs(1, 4, 4, 64, 128, seed=1)
    with pytest.raises(ValueError):
        pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1[:96], b1[:96], wdw[:, :96], bdw[:96], w2[:, :96].contiguous(), b2, res,
                                        1, 4, 4, "gelu")
    handle = lib.load()
    assert handle.tfimm_b200_pvt_v2_conv_mlp_bf16(h.data_ptr(), w1.data_ptr(), b1.data_ptr(), wdw.data_ptr(),
                                                  bdw.data_ptr(), w2.data_ptr(), b2.data_ptr(), res.data_ptr(),
                                                  res.data_ptr(), 1, 4, 4, 96, 128, 1, None) != 0


def test_determinism_and_batch_independence():
    from tfimm.backend import pvt_v2_ops

    B, gh, gw, C, hidden = 64, 28, 28, 64, 512
    h, w1, b1, wdw, bdw, w2, b2, res = conv_inputs(B, gh, gw, C, hidden, seed=3)
    a = pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu")
    assert torch.equal(a, pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu"))
    M = gh * gw
    for i in (0, B // 2, B - 1):
        one = pvt_v2_ops.pvt_v2_conv_mlp_bf16(h[i * M:(i + 1) * M], w1, b1, wdw, bdw, w2, b2, res[i * M:(i + 1) * M],
                                              1, gh, gw, "gelu")
        assert torch.equal(one, a[i * M:(i + 1) * M])
    B, N, Nk, H = 256, 3136, 49, 1
    q = torch.randn((B * N, H * DH)).to(torch.bfloat16).cuda()
    kv = torch.randn((B * Nk, 2 * H * DH)).to(torch.bfloat16).cuda()
    x = pvt_v2_ops.pvt_v2_sr_attention_bf16(q, kv, B, N, Nk, H, DH, DH ** -0.5)
    assert torch.equal(x, pvt_v2_ops.pvt_v2_sr_attention_bf16(q, kv, B, N, Nk, H, DH, DH ** -0.5))
    one = pvt_v2_ops.pvt_v2_sr_attention_bf16(q[-N:], kv[-Nk:], 1, N, Nk, H, DH, DH ** -0.5)
    assert torch.equal(one, x[-N:])


# ------------------------------------------------------------------------------------------------------ models
@pytest.fixture
def pvt_v2():
    with pvo.pvt_v2_registered() as mod:
        yield mod


def _model(name, precision, seed=11, **kw):
    import dataclasses

    import tfimm
    from oracle import params
    from oracle import pvt_v2 as op
    from tfimm.architectures.pvt_v2 import PyramidVisionTransformerV2

    cfg = dataclasses.replace(tfimm.models.registry.model_config(name), **kw)
    m = PyramidVisionTransformerV2(cfg, precision=precision, device="cuda")
    w = params.random_params(op.param_shapes(cfg), seed=seed)
    m.load_weights_dict(w)
    return m, w


def _nerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("precision", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("name", NAMES)
def test_shadowed_forward_registered(pvt_v2, name, precision):
    """Each registration in each precision at batch 2 (b3-b5 cut to two blocks per stage), every launch inside its
    bound; in bf16 the fused ConvFFN runs at the stages of 32 and 64 channels."""
    from oracle import params
    from tfimm.backend import ops, pvt_v2_ops

    kw = dict(nb_blocks=(2, 2, 2, 2)) if name in ("pvt_v2_b3", "pvt_v2_b4", "pvt_v2_b5") else {}
    m, _ = _model(name, precision, **kw)
    x = params.test_images(2, *m.cfg.input_size).cuda()
    ops.trace = []
    try:
        with (tf32_oracle() if precision == "tf32" else nullcontext()), pvo.shadowed_pvt_v2_ops() as census:
            m(x)
        names = [t[0] for t in ops.trace]
    finally:
        ops.trace = None
    census.assert_ok()
    attn = "pvt_v2_sr_attention" if m.cfg.embed_dim[0] == 32 else "pvt_sr_attention"
    if precision == "bf16":
        fused = sum(n for n, D in zip(m.cfg.nb_blocks, m.cfg.embed_dim) if D in pvt_v2_ops.CONV_MLP_FUSED_CHANNELS)
        assert names.count("pvt_v2_conv_mlp_bf16") == fused > 0, names
        assert f"{attn}_bf16" in names
    else:
        assert "pvt_v2_conv_mlp_bf16" not in names and "dwconv_bias_act" in names
        assert f"{attn}_f32" in names


@pytest.mark.parametrize("name", ["pvt_v2_b0", "pvt_v2_b2"])
def test_fp32_logits_match_oracle(pvt_v2, name):
    from oracle import params
    from oracle import pvt_v2 as op

    m, w = _model(name, "fp32")
    x = params.test_images(2, *m.cfg.input_size)
    y = m(x.cuda()).cpu()
    ref = op.forward(m.cfg, w, x)
    err = _nerr(y, ref)
    print(f"FP32 {name}: normalised max error {err:.2e}")
    assert err < 2e-6, err   # measured 4.3e-7 (b0) and 7.7e-7 (b2)


def _rms(a, b):
    return ((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("name", ["pvt_v2_b0", "pvt_v2_b2"])
def test_bf16_error_budget(pvt_v2, name):
    """The engine is no farther from the float64 oracle than the ideal bf16 graph (the engine's storage points in
    float64 arithmetic)."""
    from oracle import params
    from oracle import pvt_v2 as op

    m, w = _model(name, "bf16")
    x = params.test_images(4, *m.cfg.input_size)
    xc = x.cuda()
    y = m(xc).double().cpu()
    with pvo.emulated_pvt_v2_ops():
        y_ideal = m(xc).double().cpu()
    ref = op.forward(m.cfg, w, x)
    r_eng, r_ideal = _rms(y, ref), _rms(y_ideal, ref)
    print(f"BUDGET {name}: rms engine-vs-oracle {r_eng:.2e} | ideal-vs-oracle {r_ideal:.2e}")
    assert r_eng < 1.25 * r_ideal + 1e-4, (r_eng, r_ideal)


@pytest.mark.parametrize("name", ["pvt_v2_b0", "pvt_v2_b2"])
def test_cuda_graph_uint8_and_features(pvt_v2, name):
    m, _ = _model(name, "bf16")
    cfg = m.cfg
    x = torch.rand((8, *cfg.input_size, 3), device="cuda")
    eager = m(x)
    run = m.cuda_graph(8)
    assert torch.equal(run(x), eager)
    u8 = torch.randint(0, 256, (4, *cfg.input_size, 3), dtype=torch.uint8, device="cuda")
    mean = torch.tensor(cfg.mean, device="cuda")
    std = torch.tensor(cfg.std, device="cuda")
    err = _nerr(m(u8), m((u8.float() / 255.0 - mean) / std))
    print(f"UINT8 {name}: normalised max error vs float input {err:.2e}")
    assert err < 1e-2, err
    m32, _ = _model(name, "fp32")
    assert _nerr(m32(u8), m32((u8.float() / 255.0 - mean) / std)) < 1e-5
    y, feats = m(x[:2], return_features=True)
    assert list(feats) == m.feature_names
    assert torch.equal(feats["logits"], y)
    shapes = {k: tuple(v.shape) for k, v in feats.items()}
    D = cfg.embed_dim
    assert shapes["patch_embedding_0"] == (2, 56 * 56, D[0]) and shapes["block_0"] == (2, 56 * 56, D[0])
    assert shapes["stage_0"] == (2, 56, 56, D[0]) and shapes["stage_3"] == (2, 7, 7, D[3])
    assert shapes["features_all"] == (2, 49, D[3]) and shapes["features"] == (2, D[3])


def test_other_input_sizes_and_headless(pvt_v2):
    """A 200 x 264 input (grids 50 x 66, 25 x 33, 13 x 17, 7 x 9: the padded convolutions round up, no sr ratio
    divides) and nb_classes = 0, in fp32 against the oracle."""
    from oracle import params
    from oracle import pvt_v2 as op

    for kw in ({}, dict(nb_classes=0)):
        m, w = _model("pvt_v2_b1", "fp32", seed=4, **kw)
        x = params.test_images(2, 200, 264)
        y = m(x.cuda()).cpu()
        ref = op.forward(m.cfg, w, x)
        err = _nerr(y, ref)
        print(f"SIZE 200x264 {kw}: normalised max error {err:.2e}")
        assert y.shape == ref.shape and err < 2e-6, (kw, err)   # measured 6.2e-7 and 3.5e-7
        mb, _ = _model("pvt_v2_b1", "bf16", seed=4, **kw)
        assert _nerr(mb(x.cuda()).cpu(), ref) < 5e-2
