"""PVT family on the H100: the spatial-reduction attention kernels and pvt_embed_norm against their float64 statements
(tests/pvt_oracle.py) within their derived bounds, bitwise equality with pit_attention_bf16 where N' = N, guard regions
and determinism, and the four models in every precision.

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

import pvt_oracle as po  # noqa: E402
from tf32_oracle import tf32_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

NAMES = ["pvt_tiny", "pvt_small", "pvt_medium", "pvt_large"]
DH = 64
# (B, N, N', H): the zoo's stages at 224 px (pvt_* share them), then N' across the 64-key block and ring edges (up to
# 192 keys K / V stay resident, past it they stream), then N across the 64-query tile edges, with heads 1, 2, 5, 8
SHAPES = [(4, 3136, 49, 1), (8, 784, 49, 2), (32, 196, 49, 5), (64, 50, 50, 8), (256, 196, 49, 5),
          (2, 197, 1, 2), (2, 130, 63, 5), (3, 64, 64, 1), (2, 65, 65, 8), (2, 300, 100, 2), (1, 197, 196, 5),
          (1, 257, 785, 8), (5, 1, 49, 2), (3, 17, 100, 1), (2, 65, 785, 5), (1, 3136, 196, 1)]
# Launches whose CTAs walk several query tiles with K / V resident, as the models run at batch 256.  Tiles per CTA on
# a 132-SM H100 (csrc/pvt.cu, pvt_tiles_per_cta), per CTA of an (image, head):
#   (256, 3136, 49, 1)  7 7 7 7 7 7 7   stage 0: each Q buffer refilled three times by one CTA
#   (128, 3136, 49, 1)  3 ... 3 1       an odd count and a one-tile last group
#   (256, 784, 49, 2)   4 4 4 1         stage 1: a short last group ending in a partial tile (784 = 12 x 64 + 16)
#   (256, 784, 100, 2)  4 4 4 1         resident K / V of two 64-key blocks
#   (256, 784, 130, 2)  4 4 4 1         resident K / V of three blocks, the whole ring
MULTI_TILE = [(256, 3136, 49, 1), (128, 3136, 49, 1), (256, 784, 49, 2), (256, 784, 100, 2), (256, 784, 130, 2)]
KINDS = ["randn", "large", "late_max"]


@pytest.fixture
def pvt():
    with po.pvt_registered() as mod:
        yield mod


def sr_inputs(kind, B, N, Nk, H, seed, dtype=torch.bfloat16):
    """q (B N, H dh), kv (B N', 2 H dh) with scores scale q.k (scale = dh^-0.5) of the named shape:
    randn     q, k, v ~ N(0, 1);
    large     q, k entries of variance 10 (scores of std ~10), query 0's score of key N' // 2 exactly 80 before the
              bf16 rounding;
    late_max  every query's maximum on the last key (inside the partial last block when N' % 64 != 0)."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, N, H, DH, generator=g, dtype=torch.float64)
    kv = torch.randn(B, Nk, 2, H, DH, generator=g, dtype=torch.float64)
    if kind == "large":
        q *= 10.0 ** 0.5
        kv[:, :, 0] *= 10.0 ** 0.5
        kv[:, Nk // 2, 0] = q[:, 0] * 80.0 * DH ** 0.5 / q[:, 0].pow(2).sum(-1, keepdim=True)
    elif kind == "late_max":
        q += 2.0
        kv[:, :, 0] -= kv[:, :, 0].mean(-1, keepdim=True)
        kv[:, Nk - 1, 0] = 3.0
    return q.reshape(B * N, H * DH).to(dtype).cuda(), kv.reshape(B * Nk, 2 * H * DH).to(dtype).cuda()


def _report(census, title):
    print(f"\n=== {title}\n" + census.table())
    census.assert_ok()
    assert census.rows and all(r["flips"] < 0.02 for r in census.rows)


# ------------------------------------------------------------------------------------------- against the statement
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("B,N,Nk,H", SHAPES + MULTI_TILE)
def test_sr_attention_within_its_bound(B, N, Nk, H, dtype):
    from tfimm.backend import pvt_ops

    launcher = pvt_ops.pvt_sr_attention_bf16 if dtype == torch.bfloat16 else pvt_ops.pvt_sr_attention_f32
    name = launcher.__name__
    with po.shadowed_pvt_ops() as census:
        for i, kind in enumerate(KINDS):
            q, kv = sr_inputs(kind, B, N, Nk, H, seed=N + Nk + i, dtype=dtype)
            getattr(pvt_ops, name)(q, kv, B, N, Nk, H, DH, DH ** -0.5)
    _report(census, f"{name} B={B} N={N} N'={Nk} H={H}: {KINDS}")
    assert census.ops() == {name} and len(census.rows) == len(KINDS)


@pytest.mark.parametrize("N", [1, 17, 49, 64, 65, 197, 785, 3136])
def test_equals_pit_attention_when_keys_are_the_queries(N):
    """q / kv cut from one packed qkv with N' = N: the same arithmetic as pit_attention_bf16<64>, bit for bit."""
    from tfimm.backend import pit_ops, pvt_ops

    B, H = (2, 1) if N > 1000 else (3, 5)
    g = torch.Generator().manual_seed(N)
    qkv = (torch.randn((B * N, 3 * H * DH), generator=g) * 2.0).to(torch.bfloat16).cuda()
    x = qkv.view(B * N, 3, H * DH)
    q, kv = x[:, 0].contiguous(), x[:, 1:].reshape(B * N, 2 * H * DH).contiguous()
    a = pvt_ops.pvt_sr_attention_bf16(q, kv, B, N, N, H, DH, DH ** -0.5)
    b = pit_ops.pit_attention_bf16(qkv, B, N, H, DH, DH ** -0.5)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def _embed_inputs(B, P, C, ntok, seed):
    g = torch.Generator().manual_seed(seed)
    tok = (1e3 + torch.randn((B * P, C), generator=g) * 3.0).cuda()    # mean 1e3: the variance is a small difference
    gamma = (1.0 + 0.1 * torch.randn(C, generator=g)).cuda()
    beta = (0.1 * torch.randn(C, generator=g)).cuda()
    pos = torch.randn((ntok + P, C), generator=g).cuda()
    cls = torch.randn(C, generator=g).cuda() if ntok else None
    return tok, gamma, beta, pos, cls


@pytest.mark.parametrize("B,P,C,ntok", [(4, 3136, 64, 0), (4, 784, 128, 0), (8, 196, 320, 0), (8, 49, 512, 1),
                                        (8, 49, 512, 0), (3, 7, 1024, 1), (2, 5, 4, 1)])
def test_embed_norm_within_its_bound(B, P, C, ntok):
    from tfimm.backend import pvt_ops

    tok, gamma, beta, pos, cls = _embed_inputs(B, P, C, ntok, seed=P + C)
    with po.shadowed_pvt_ops() as census:
        pvt_ops.pvt_embed_norm(tok, gamma, beta, pos, cls, B, P, 1e-5)
    _report(census, f"pvt_embed_norm B={B} P={P} C={C} ntok={ntok}")


# ------------------------------------------------------------------------------------- guard regions, determinism
G = 4096


def _buffer(n, dtype):
    pattern = torch.tensor(-12345.0, dtype=dtype)
    buf = torch.full((G + n + G,), -12345.0, dtype=dtype, device="cuda")
    return buf, buf[G:G + n], pattern.cuda()


def test_outputs_stay_inside_their_buffers():
    """Through the C entry points, into the middle of a canary buffer: nothing outside the output is written, the
    output holds no canary and no NaN, and it equals the launcher's."""
    from tfimm.backend import lib, pvt_ops

    h = lib.load()
    for dtype, fn in ((torch.bfloat16, h.tfimm_b200_pvt_sr_attention_bf16),
                      (torch.float32, h.tfimm_b200_pvt_sr_attention_f32)):
        for B, N, Nk, H in ((3, 131, 49, 2), (2, 65, 257, 1)):
            q, kv = sr_inputs("randn", B, N, Nk, H, seed=7, dtype=dtype)
            buf, out, pattern = _buffer(B * N * H * DH, dtype)
            assert fn(q.data_ptr(), kv.data_ptr(), out.data_ptr(), B, N, Nk, H, DH, DH ** -0.5, None) == 0
            torch.cuda.synchronize()
            assert (buf[:G] == pattern).all() and (buf[-G:] == pattern).all()
            assert not (out == pattern).any() and not out.isnan().any()
            ref = pvt_ops._sr_attention(fn.__name__, dtype, q, kv, B, N, Nk, H, DH, DH ** -0.5)
            assert torch.equal(out.view(B * N, -1), ref)
    for B, P, C, ntok in ((3, 49, 512, 1), (2, 29, 320, 0)):
        tok, gamma, beta, pos, cls = _embed_inputs(B, P, C, ntok, seed=3)
        buf, out, pattern = _buffer(B * (P + ntok) * C, torch.float32)
        assert h.tfimm_b200_pvt_embed_norm(tok.data_ptr(), gamma.data_ptr(), beta.data_ptr(), pos.data_ptr(),
                                           None if cls is None else cls.data_ptr(), out.data_ptr(), B, P, ntok, C,
                                           1e-5, None) == 0
        torch.cuda.synchronize()
        assert (buf[:G] == pattern).all() and (buf[-G:] == pattern).all()
        assert torch.equal(out.view(-1, C), pvt_ops.pvt_embed_norm(tok, gamma, beta, pos, cls, B, P, 1e-5))


def test_determinism_and_batch_independence():
    """Two runs are bit-identical, and image i of a batch equals image i run alone.  The batches are chosen so that the
    full launch walks several query tiles per CTA (MULTI_TILE: 7 at stage 0, 4 with a short last group and three
    resident key blocks) while the single image takes one tile per CTA; a streamed case (785 keys) is added."""
    from tfimm.backend import pvt_ops

    for dtype, launcher in ((torch.bfloat16, pvt_ops.pvt_sr_attention_bf16),
                            (torch.float32, pvt_ops.pvt_sr_attention_f32)):
        for B, N, Nk, H in ((256, 3136, 49, 1), (256, 784, 130, 2), (8, 300, 785, 2)):
            q, kv = sr_inputs("randn", B, N, Nk, H, seed=B + Nk, dtype=dtype)
            a = launcher(q, kv, B, N, Nk, H, DH, DH ** -0.5)
            b = launcher(q, kv, B, N, Nk, H, DH, DH ** -0.5)
            assert torch.equal(a, b)
            for i in (0, B // 2, B - 1):
                one = launcher(q.view(B, N, -1)[i].contiguous(), kv.view(B, Nk, -1)[i].contiguous(), 1, N, Nk, H, DH,
                               DH ** -0.5)
                assert torch.equal(one, a.view(B, N, -1)[i]), (B, N, Nk, H, i)
    tok, gamma, beta, pos, cls = _embed_inputs(16, 49, 512, 1, seed=5)
    a = pvt_ops.pvt_embed_norm(tok, gamma, beta, pos, cls, 16, 49, 1e-5)
    assert torch.equal(a, pvt_ops.pvt_embed_norm(tok, gamma, beta, pos, cls, 16, 49, 1e-5))


# ------------------------------------------------------------------------------------------------------ models
def _model(name, precision, seed=11, **kw):
    import dataclasses

    import tfimm
    from oracle import params
    from oracle import pvt as op
    from tfimm.architectures.pvt import PyramidVisionTransformer

    cfg = dataclasses.replace(tfimm.models.registry.model_config(name), **kw)
    m = PyramidVisionTransformer(cfg, precision=precision, device="cuda")
    w = params.random_params(op.param_shapes(cfg), seed=seed)
    m.load_weights_dict(w)
    return m, w


def _nerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("precision", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("name", NAMES)
def test_shadowed_forward_registered(pvt, name, precision):
    """Each registration in each precision at batch 2, every launch inside its bound; the trace shows the tensor-core
    kernel in bf16 and the fp32 kernel otherwise, and pvt_embed_norm in every precision."""
    from oracle import params
    from tfimm.backend import ops

    m, _ = _model(name, precision)
    x = params.test_images(2, *m.cfg.input_size).cuda()
    ops.trace = []
    try:
        with (tf32_oracle() if precision == "tf32" else nullcontext()), po.shadowed_pvt_ops() as census:
            m(x)
        names = {t[0] for t in ops.trace}
    finally:
        ops.trace = None
    census.assert_ok()
    assert "pvt_embed_norm" in names
    if precision == "bf16":
        assert "pvt_sr_attention_bf16" in names and "pvt_sr_attention_f32" not in names, names
    else:
        assert "pvt_sr_attention_f32" in names and "pvt_sr_attention_bf16" not in names, names


@pytest.mark.parametrize("name", ["pvt_tiny", "pvt_small"])
def test_fp32_logits_match_oracle(pvt, name):
    from oracle import params
    from oracle import pvt as op

    m, w = _model(name, "fp32")
    x = params.test_images(2, *m.cfg.input_size)
    y = m(x.cuda()).cpu()
    ref = op.forward(m.cfg, w, x)
    err = _nerr(y, ref)
    print(f"FP32 {name}: normalised max error {err:.2e}")
    assert err < 5e-6, err


def _rms(a, b):
    return ((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("name", ["pvt_tiny", "pvt_medium"])
def test_bf16_error_budget(pvt, name):
    """The kernels diverge from the ideal bf16 graph (emulated, float64 arithmetic, the engine's bf16 storage points)
    by no more than 1.6 x the float64-vs-float32 emulation floor (B1), and the engine is no farther from the float64
    oracle than the ideal graph (B2)."""
    from oracle import params
    from oracle import pvt as op

    m, w = _model(name, "bf16")
    x = params.test_images(4, *m.cfg.input_size)
    xc = x.cuda()
    y = m(xc).double().cpu()
    with po.emulated_pvt_ops():
        y_ideal = m(xc).double().cpu()
    with po.emulated_pvt_ops(arithmetic=torch.float32):
        y_ideal32 = m(xc).double().cpu()
    ref = op.forward(m.cfg, w, x)
    r_eng, r_ideal, r_kern, r_floor = _rms(y, ref), _rms(y_ideal, ref), _rms(y, y_ideal), _rms(y_ideal32, y_ideal)
    print(f"BUDGET {name}: rms engine-vs-oracle {r_eng:.2e} | ideal-vs-oracle {r_ideal:.2e} | engine-vs-ideal "
          f"{r_kern:.2e} | floor {r_floor:.2e}")
    assert r_kern < 1.6 * r_floor + 1e-4, (r_kern, r_floor)      # B1
    assert r_eng < 1.25 * r_ideal + 1e-4, (r_eng, r_ideal)       # B2


@pytest.mark.parametrize("name", ["pvt_tiny", "pvt_small"])
def test_cuda_graph_uint8_and_features(pvt, name):
    from tfimm.backend import ops

    m, _ = _model(name, "bf16")
    cfg = m.cfg
    x = torch.rand((8, *cfg.input_size, 3), device="cuda")
    eager = m(x)
    run = m.cuda_graph(8)
    assert torch.equal(run(x), eager)
    u8 = torch.randint(0, 256, (4, *cfg.input_size, 3), dtype=torch.uint8, device="cuda")
    mean = torch.tensor(cfg.mean, device="cuda")
    std = torch.tensor(cfg.std, device="cuda")
    ref = m((u8.float() / 255.0 - mean) / std)
    err = _nerr(m(u8), ref)
    print(f"UINT8 {name}: normalised max error vs float input {err:.2e}")
    assert err < 1e-2, err   # the first bf16 rounding of the two pixel paths differs
    m32, _ = _model(name, "fp32")
    err32 = _nerr(m32(u8), m32((u8.float() / 255.0 - mean) / std))
    assert err32 < 1e-5, err32
    y, feats = m(x[:2], return_features=True)
    assert list(feats) == m.feature_names
    assert torch.equal(feats["logits"], y)
    shapes = {k: tuple(v.shape) for k, v in feats.items()}
    D = cfg.embed_dim
    assert shapes["patch_embedding_0"] == (2, 56 * 56, D[0]) and shapes["pos_embedding_3"] == (2, 50, D[3])
    assert shapes["stage_0"] == (2, 56, 56, D[0]) and shapes["stage_2"] == (2, 14, 14, D[2])
    assert shapes["stage_3"] == shapes["features_all"] == (2, 50, D[3]) and shapes["features"] == (2, D[3])
    assert ops.launch_count > 0


@pytest.mark.parametrize("size", [(200, 264), (320, 320)])
def test_interpolate_input_and_headless(pvt, size):
    """Inputs through interpolate_input in fp32 against the oracle: 200 x 264, whose grids 50 x 66, 25 x 33, 12 x 16
    and 6 x 8 no sr ratio divides (the remainders are dropped), and 320 x 320 (100 keys at stage 0: two 64-key
    blocks); and nb_classes = 0, whose logits are the normalised class row."""
    from oracle import params
    from oracle import pvt as op

    for kw in (dict(interpolate_input=True), dict(interpolate_input=True, nb_classes=0)):
        m, w = _model("pvt_tiny", "fp32", seed=4, **kw)
        x = params.test_images(2, *size)
        y = m(x.cuda()).cpu()
        ref = op.forward(m.cfg, w, x)
        err = _nerr(y, ref)
        print(f"INTERP {size} {kw}: normalised max error {err:.2e}")
        assert y.shape == ref.shape and err < 5e-6, (kw, err)
        mb, _ = _model("pvt_tiny", "bf16", seed=4, **kw)
        yb = mb(x.cuda()).cpu()
        assert yb.shape == ref.shape and _nerr(yb, ref) < 5e-2
