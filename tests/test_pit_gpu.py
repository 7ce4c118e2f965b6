"""PiT on the H100: the streaming attention and the pooling kernel against float64 (head dims 32, 48, 64 over sequence
lengths from 1 to above 2000, logits of +-80, a row whose maximum is in the last key block; every pooling shape of the
family, odd, even, non-square and 1 x 1 grids, one and two token rows), guard regions around every output, bitwise
determinism, and the eight registrations in every precision, launch by launch under the shadow harness."""
import importlib
import sys
from contextlib import nullcontext
from copy import deepcopy
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = Path(__file__).resolve().parent
if str(HERE) not in sys.path:
    sys.path.insert(0, str(HERE))

import pit_oracle as po  # noqa: E402
from tf32_oracle import tf32_oracle  # noqa: E402

NAMES = ["pit_ti_224", "pit_xs_224", "pit_s_224", "pit_b_224",
         "pit_ti_distilled_224", "pit_xs_distilled_224", "pit_s_distilled_224", "pit_b_distilled_224"]


@pytest.fixture
def pit():
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.pit"
    mod = importlib.reload(sys.modules[name]) if name in sys.modules else importlib.import_module(name)
    try:
        yield mod
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


# ------------------------------------------------------------------------------------------------ attention alone
# the family's stage lengths (plain / distilled), the 64-key block edges, and one interpolated length above 2000
# (pit_ti at 384 x 384: a 47 x 47 grid and two token rows)
LENGTHS = [1, 2, 50, 51, 63, 64, 65, 66, 129, 197, 198, 257, 258, 730, 731, 962, 963, 2211]


def _qkv(B, T, H, dh, seed, std=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn((B * T, 3 * H * dh), generator=g, device="cuda") * std).to(torch.bfloat16)


@pytest.mark.parametrize("T", LENGTHS)
@pytest.mark.parametrize("dh", [32, 48, 64])
def test_attention_against_float64(dh, T):
    """Every output within the derived bound of the bf16 tensor-core attention (shadow._rule_attention)."""
    from tfimm.backend import pit_ops

    B, H = (1, 2) if T > 1000 else (2, 3)
    qkv = _qkv(B, T, H, dh, seed=T + dh)
    with po.shadowed_pit_ops() as census:
        pit_ops.pit_attention_bf16(qkv, B, T, H, dh, dh ** -0.5)
    census.assert_ok()
    assert census.ops() == {"pit_attention_bf16"}


@pytest.mark.parametrize("T", [65, 197, 731])
@pytest.mark.parametrize("dh", [32, 48, 64])
def test_attention_large_logits_and_late_maximum(dh, T):
    """Scores up to about 80, so the running maximum moves by tens between key blocks and the rescale of O and l
    matters; and query 0's maximum placed on the last key (in the partial last block)."""
    from tfimm.backend import pit_ops

    B, H = 2, 2
    qkv = _qkv(B, T, H, dh, seed=7 * dh + T).float().view(B, T, 3, H, dh)
    qkv[:, :, :2] *= 10.0 ** 0.5                    # q and k entries of variance 10: scores of std ~10
    qkv[:, T - 1, 1] = qkv[:, 0, 0] * 8 / dh ** 0.5   # key T - 1 along query 0: a score of ~80, its largest
    qkv = qkv.reshape(B * T, -1).to(torch.bfloat16)
    q, k = qkv.double().view(B, T, 3, H, dh)[:, :, 0], qkv.double().view(B, T, 3, H, dh)[:, :, 1]
    scores = torch.einsum("bihd,bjhd->bhij", q, k) * dh ** -0.5
    assert scores.abs().max().item() > 60
    assert (scores[:, :, 0].argmax(-1) == T - 1).all()
    with po.shadowed_pit_ops() as census:
        pit_ops.pit_attention_bf16(qkv, B, T, H, dh, dh ** -0.5)
    census.assert_ok()


def test_attention_equals_vit_kernel_where_both_apply():
    """At head dim 64 both kernels run the same algorithm (64-key blocks, P rounded per block): the outputs agree to
    within one bf16 ulp of the larger ones."""
    from tfimm.backend import ops, pit_ops

    for T in (65, 197, 258):
        qkv = _qkv(4, T, 8, 64, seed=T)
        a = pit_ops.pit_attention_bf16(qkv, 4, T, 8, 64, 0.125).float()
        b = ops.attention(qkv, 4, T, 8, 64, 0.125).float()
        assert (a - b).abs().max().item() <= 2.0 ** -7 * b.abs().max().item(), T


# ------------------------------------------------------------------------------------------------------ pooling alone
# (B, nb_tokens, H, W, C): every stage shape of the family (pit_ti / xs / s at 27 x 27 and 14 x 14, pit_b at 31 x 31
# and 16 x 16), an odd and an even non-square grid, a 1 x 1 grid
POOL_CASES = [(3, 1, 27, 27, 64), (2, 2, 27, 27, 96), (2, 1, 27, 27, 144), (2, 2, 31, 31, 256),
              (3, 2, 14, 14, 128), (2, 1, 14, 14, 192), (2, 2, 14, 14, 288), (2, 1, 16, 16, 512),
              (3, 2, 9, 13, 32), (2, 1, 12, 6, 48), (4, 1, 1, 1, 64), (3, 2, 1, 1, 16)]


def _pool_inputs(B, nb, H, W, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((B * (nb + H * W), C), generator=g, device="cuda") * 2 + 0.5
    w = torch.randn((9, 2 * C), generator=g, device="cuda") * 0.3
    b = torch.randn((2 * C,), generator=g, device="cuda")
    return x, w, b


@pytest.mark.parametrize("case", POOL_CASES, ids=[f"B{b}-nb{n}-{h}x{w}-C{c}" for b, n, h, w, c in POOL_CASES])
def test_pool_against_float64(case):
    from tfimm.backend import pit_ops

    B, nb, H, W, C = case
    x, w, b = _pool_inputs(*case, seed=C + H)
    with po.shadowed_pit_ops() as census:
        for tok in (False, True):
            pit_ops.pit_pool(x, w, b, B, nb, H, W, tokens_bf16=tok)
    census.assert_ok()
    assert census.ops() == {"pit_pool"}


def test_guard_regions_untouched():
    """Outputs written into the middle of larger buffers: the guard cells on both sides keep their pattern, and the
    token rows of the pooled stream (the token Dense's) are not written."""
    from tfimm.backend import lib, pit_ops

    h = lib.load()
    G = 4096   # guard elements on each side (16-byte multiples)
    pattern = -1232.0   # exact in bf16

    def buffer(n, dtype):
        buf = torch.full((n + 2 * G,), pattern, device="cuda").to(dtype)
        return buf, buf[G:G + n]

    B, T, H, dh = 2, 197, 3, 48
    qkv = _qkv(B, T, H, dh, seed=3)
    buf, out = buffer(B * T * H * dh, torch.bfloat16)
    assert h.tfimm_b200_pit_attention_bf16(qkv.data_ptr(), out.data_ptr(), B, T, H, dh, dh ** -0.5, None) == 0
    torch.cuda.synchronize()
    assert (buf[:G] == pattern).all() and (buf[-G:] == pattern).all()
    ref = pit_ops.pit_attention_bf16(qkv, B, T, H, dh, dh ** -0.5)
    assert torch.equal(out.view(B * T, -1), ref)

    B, nb, Hg, Wg, C = 3, 2, 9, 13, 32
    x, w, b = _pool_inputs(B, nb, Hg, Wg, C, seed=9)
    Ho, Wo = pit_ops.pool_geometry(Hg, Wg)
    obuf, out = buffer(B * (nb + Ho * Wo) * 2 * C, torch.float32)
    tbuf, tok = buffer(B * nb * C, torch.bfloat16)
    assert h.tfimm_b200_pit_pool(x.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), tok.data_ptr(), B, nb, Hg,
                                 Wg, C, None) == 0
    torch.cuda.synchronize()
    for g in (obuf, tbuf):
        assert (g[:G] == pattern).all() and (g[-G:] == pattern).all()
    o3 = out.view(B, nb + Ho * Wo, 2 * C)
    assert (o3[:, :nb] == pattern).all()
    ref, ref_tok = pit_ops.pit_pool(x, w, b, B, nb, Hg, Wg, tokens_bf16=True)
    assert torch.equal(o3[:, nb:], ref.view(B, -1, 2 * C)[:, nb:]) and torch.equal(tok.view(B * nb, C), ref_tok)


def test_determinism():
    from tfimm.backend import pit_ops

    for dh, T in ((32, 731), (48, 198), (64, 963)):
        qkv = _qkv(8, T, 4, dh, seed=dh)
        a = pit_ops.pit_attention_bf16(qkv, 8, T, 4, dh, dh ** -0.5)
        b = pit_ops.pit_attention_bf16(qkv, 8, T, 4, dh, dh ** -0.5)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    x, w, b = _pool_inputs(16, 2, 27, 27, 144, seed=1)
    a = pit_ops.pit_pool(x, w, b, 16, 2, 27, 27, tokens_bf16=True)
    c = pit_ops.pit_pool(x, w, b, 16, 2, 27, 27, tokens_bf16=True)
    nb = 2
    assert torch.equal(a[0].view(16, -1, 288)[:, nb:].view(torch.int32), c[0].view(16, -1, 288)[:, nb:].view(torch.int32))
    assert torch.equal(a[1].view(torch.int16), c[1].view(torch.int16))


# ------------------------------------------------------------------------------------------------------ models
def _model(name, precision, seed=11):
    import tfimm
    from oracle import params
    from oracle import pit as op

    m = tfimm.create_model(name, precision=precision, device="cuda")
    w = params.random_params(op.param_shapes(m.cfg), seed=seed)
    m.load_weights_dict(w)
    return m, w


def _nerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("precision", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("name", NAMES)
def test_shadowed_forward_registered(pit, name, precision):
    """Each registration in each precision at batch 2, every launch inside its bound; the trace shows which attention
    kernels ran: pit_attention_bf16 in bf16 (never the fp32 fallback), the SIMT / TF32 kernels otherwise; pit_pool in
    every precision."""
    from oracle import params
    from tfimm.backend import ops

    m, _ = _model(name, precision)
    x = params.test_images(2, *m.cfg.input_size).cuda()
    ops.trace = []
    try:
        # tf32: the GEMMs' and the head-dim-64 attention's statements and bounds are the TF32 ones, entered first
        with (tf32_oracle() if precision == "tf32" else nullcontext()), po.shadowed_pit_ops() as census:
            m(x)
        names = {t[0] for t in ops.trace}
    finally:
        ops.trace = None
    census.assert_ok()
    assert "pit_pool" in names
    if precision == "bf16":
        assert "pit_attention_bf16" in names and "attention_f32" not in names, names
    else:
        assert "pit_attention_bf16" not in names, names
        dhs = {D // H for D, H in zip(m.cfg.embed_dim, m.cfg.nb_heads)}
        assert ("attention_tf32" in names) == (precision == "tf32" and 64 in dhs), names


@pytest.mark.parametrize("name", ["pit_ti_distilled_224", "pit_s_224", "pit_b_224"])
def test_fp32_logits_match_oracle(pit, name):
    from oracle import params
    from oracle import pit as op

    m, w = _model(name, "fp32")
    x = params.test_images(2, *m.cfg.input_size)
    y = m(x.cuda()).cpu()
    ref = op.forward(m.cfg, w, x)
    err = _nerr(y, ref)
    print(f"FP32 {name}: normalised max error {err:.2e}")
    assert err < 5e-6, err


def _rms(a, b):
    return ((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("name", ["pit_ti_224", "pit_s_distilled_224", "pit_b_224"])
def test_bf16_error_budget(pit, name):
    """The MLP-Mixer method: the kernels diverge from the ideal bf16 graph (emulated, float64 arithmetic, the engine's
    bf16 storage points) by no more than 1.6 x the float64-vs-float32 emulation floor (B1), and add nothing measurable
    to the ideal graph's own distance from the float64 oracle (B2)."""
    from oracle import params
    from oracle import pit as op

    m, w = _model(name, "bf16")
    x = params.test_images(4, *m.cfg.input_size)
    xc = x.cuda()
    y = m(xc).double().cpu()
    with po.emulated_pit_ops():
        y_ideal = m(xc).double().cpu()
    with po.emulated_pit_ops(arithmetic=torch.float32):
        y_ideal32 = m(xc).double().cpu()
    ref = op.forward(m.cfg, w, x)
    r_eng, r_ideal, r_kern, r_floor = _rms(y, ref), _rms(y_ideal, ref), _rms(y, y_ideal), _rms(y_ideal32, y_ideal)
    print(f"BUDGET {name}: rms engine-vs-oracle {r_eng:.2e} | ideal-vs-oracle {r_ideal:.2e} | engine-vs-ideal "
          f"{r_kern:.2e} | floor {r_floor:.2e}")
    assert r_kern < 1.6 * r_floor + 1e-4, (r_kern, r_floor)      # B1
    assert r_eng < 1.25 * r_ideal + 1e-4, (r_eng, r_ideal)       # B2


@pytest.mark.parametrize("name", ["pit_xs_distilled_224", "pit_b_224"])
def test_cuda_graph_uint8_and_features(pit, name):
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
    assert ops.launch_count > 0


def test_interpolate_input_and_headless(pit):
    """A non-square input through interpolate_input (grids 35 x 23 -> 18 x 12 -> 9 x 6), and nb_classes = 0 on a
    distilled model (the logits are the two normalised token rows), in fp32 against the oracle."""
    import dataclasses

    import tfimm
    from oracle import params
    from oracle import pit as op

    for name, kw in (("pit_ti_224", dict(interpolate_input=True)), ("pit_xs_distilled_224", dict(nb_classes=0))):
        cfg = dataclasses.replace(tfimm.models.registry.model_config(name), **kw)
        m = pit.PoolingVisionTransformer(cfg, precision="fp32", device="cuda")
        w = params.random_params(op.param_shapes(cfg), seed=4)
        m.load_weights_dict(w)
        x = params.test_images(2, *((288, 192) if kw.get("interpolate_input") else cfg.input_size))
        y = m(x.cuda()).cpu()
        ref = op.forward(cfg, w, x)
        assert y.shape == ref.shape and _nerr(y, ref) < 5e-6, (name, _nerr(y, ref))
