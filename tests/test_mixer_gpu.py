"""MLP-Mixer family on the H100: the token-mixing GEMM (wgmma with an MN-major operand, and its fp32 form), the channel
GLU, and whole forwards of every block type against the float64 oracle (oracle/mlp_mixer.py)."""
import importlib
import sys
from copy import deepcopy

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def mixer():
    """Registers the MLP-Mixer models for this module and restores the registry afterwards (tests/test_api_cpu.py pins
    the exact list of models)."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    name = "tfimm.architectures.mlp_mixer"
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


def _bf16_ulp(x):
    """One bf16 ulp at |x| (float64 tensor)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _act(x, act):
    if act == "gelu":
        return 0.5 * x * (1.0 + torch.erf(x / 2 ** 0.5))
    if act == "swish":
        return x * torch.sigmoid(x)
    return x


# ---------------------------------------------------------------- token GEMM
@pytest.mark.parametrize("N", [49, 50, 196, 784])
@pytest.mark.parametrize("C", [64, 384, 768, 1024])
@pytest.mark.parametrize("block_n", [64, 128, 256])
def test_token_gemm_permutation_exact(N, C, block_n):
    """Wt a permutation, fp32 out: the result is the permuted X bit for bit -- every element of the MN-major operand
    lands where the descriptor says, for every tile width, K tail and image."""
    from tfimm.backend import mixer_ops

    g = torch.Generator(device="cuda").manual_seed(N * 7 + C)
    B = 3
    perm = torch.randperm(N, generator=g, device="cuda")
    ldw = (N + 7) // 8 * 8
    wt = torch.zeros((N, ldw), device="cuda", dtype=torch.bfloat16)
    wt[torch.arange(N, device="cuda"), perm] = 1
    x = torch.randn((B, N, C), generator=g, device="cuda").to(torch.bfloat16)
    out = mixer_ops.token_gemm(wt[:, :N], x, out_dtype=torch.float32, block_n=block_n)
    torch.cuda.synchronize()
    assert torch.equal(out, x[:, perm].float())


def _token_case(B, M, N, C, glu, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ldw = (N + 7) // 8 * 8
    wt = torch.zeros((M, ldw), device="cuda")
    wt[:, :N] = torch.randn((M, N), generator=g, device="cuda") / N ** 0.5
    x = torch.randn((B, N, C), generator=g, device="cuda")
    bias = 0.3 * torch.randn(M, generator=g, device="cuda")
    gamma = 1 + 0.3 * torch.randn(C, generator=g, device="cuda")
    return wt.to(dtype), x.to(dtype), bias, gamma, g


def _token_ref(wt, N, x, bias, act, glu, gamma, mul, res, m_out):
    acc = torch.einsum("mn,bnc->bmc", wt[:, :N].double(), x.double()) + bias.double()[None, :, None]
    if glu:
        M = acc.shape[1]
        a = acc.view(acc.shape[0], M // 16, 2, 8, -1)
        v = (a[:, :, 0] * _act(a[:, :, 1], act)).reshape(acc.shape[0], M // 2, -1)
    else:
        v = _act(acc, act)
    v = v[:, :m_out]
    if gamma is not None:
        v = v * gamma.double()
    if mul is not None:
        v = v * mul.double()
    if res is not None:
        v = v + res.double()
    return v


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("case", [
    dict(B=3, M=384, N=196, C=768, act="gelu"),                      # Mixer token fc1
    dict(B=2, M=196, N=384, C=768, res=True, out=torch.float32),     # Mixer token fc2, residual in place
    dict(B=5, M=196, N=196, C=384, gamma=True, res=True, out=torch.float32),   # ResMLP linear_tokens
    dict(B=3, M=196, N=196, C=768, mul=True),                        # gMLP spatial gate, strided u
    dict(B=3, M=384, N=196, C=384, act="swish", glu=True),           # gMixer token GLU
    dict(B=2, M=64, N=30, C=40, act="gelu", glu=True),               # 5 x 6 grid, padded GLU halves
    dict(B=4, M=49, N=49, C=136, gamma=True, res=True, out=torch.float32),   # 7 x 7 grid
])
def test_token_gemm_epilogues(case, dtype):
    from tfimm.backend import mixer_ops

    B, M, N, C = case["B"], case["M"], case["N"], case["C"]
    glu = case.get("glu", False)
    if glu:
        M = (M + 15) // 16 * 16
    wt, x, bias, gamma, g = _token_case(B, M, N, C, glu, dtype, seed=M + N + C)
    m_out = M // 2 if glu else M
    odt = case.get("out", dtype) if dtype == torch.bfloat16 else torch.float32
    if case.get("glu") and case["M"] == 64:
        m_out = 27   # rows past m_out are not stored
    # strided X: a column slice of a wider activation
    xw = torch.zeros((B, N, C + 16), device="cuda", dtype=dtype)
    xw[:, :, 8:8 + C] = x
    xv = xw[:, :, 8:8 + C]
    # canary rows after m_out
    big = torch.full((B, m_out + 5, C), 7.0, device="cuda", dtype=odt)
    out = big[:, :m_out]
    res = mul = None
    if case.get("res"):
        out.copy_(torch.randn((B, m_out, C), generator=g, device="cuda"))
        res = out
    if case.get("mul"):
        uw = torch.randn((B, m_out, 2 * C), generator=g, device="cuda").to(odt)
        mul = uw[:, :, :C]
    res0 = res.clone() if res is not None else None
    mixer_ops.token_gemm(wt[:, :N], xv, bias=bias, act=case.get("act"), gamma=gamma if case.get("gamma") else None,
                         residual=res, mul=mul, out=out, m_out=m_out, glu=glu)
    torch.cuda.synchronize()
    ref = _token_ref(wt, N, x, bias, case.get("act"), glu, gamma if case.get("gamma") else None, mul, res0, m_out)
    assert torch.all(big[:, m_out:] == 7.0), "rows >= m_out were written"
    d = (out.double() - ref).abs()
    if odt == torch.bfloat16:
        # fp32 accumulation differs from float64 by ~K 2^-24 |terms|; the stored value must be the correctly rounded
        # one or one bf16 ulp away
        assert torch.all(d <= _bf16_ulp(ref) * 1.01 + 1e-5), d.max().item()
    else:
        assert _nerr(out, ref) < 2e-5, _nerr(out, ref)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_channel_glu(dtype):
    """Channel GLU: exact pairing (value j times act(gate j), nothing shifted), then a random comparison."""
    from tfimm.backend import mixer_ops

    M, K, h = 300, 64, 200
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn((M, K), generator=g, device="cuda")
    # pairing: value feature j reads input column j % K, gate j is a constant distinct per j (through the bias)
    j = torch.arange(h, device="cuda")
    w = torch.zeros((2 * h, K), device="cuda")
    w[j, j % K] = 1.0
    b = torch.zeros(2 * h, device="cuda")
    b[h:] = 1.0 + 0.25 * j
    wi, bi = mixer_ops.glu_interleave(w, b, dtype == torch.float32)
    out = mixer_ops.gemm_glu(a.to(dtype), wi.to(dtype), bi, h, "swish")
    torch.cuda.synchronize()
    exp = a.to(dtype).double()[:, j % K] * _act(b[h:].double(), "swish")
    tol = 1e-5 * exp.abs() if dtype == torch.float32 else _bf16_ulp(exp) * 1.01
    assert torch.all((out.double() - exp).abs() <= tol + 1e-6)
    # random
    w = torch.randn((2 * h, K), generator=g, device="cuda") / K ** 0.5
    b = 0.3 * torch.randn(2 * h, generator=g, device="cuda")
    wi, bi = mixer_ops.glu_interleave(w, b, dtype == torch.float32)
    out = mixer_ops.gemm_glu(a.to(dtype), wi.to(dtype), bi, h, "gelu")
    torch.cuda.synchronize()
    acc = a.to(dtype).double() @ w.to(dtype).double().t() + b.double()
    ref = acc[:, :h] * _act(acc[:, h:], "gelu")
    if dtype == torch.bfloat16:
        assert torch.all((out.double() - ref).abs() <= _bf16_ulp(ref) * 1.01 + 1e-5)
    else:
        assert _nerr(out, ref) < 2e-5


def test_affine():
    from tfimm.backend import mixer_ops

    x = torch.randn((1000, 384), device="cuda")
    a, b = torch.randn(384, device="cuda"), torch.randn(384, device="cuda")
    for dt in (torch.float32, torch.bfloat16):
        out = mixer_ops.affine(x, a, b, dt)
        assert torch.equal(out, torch.addcmul(b, a, x).to(dt))


# ---------------------------------------------------------------- whole models
SMALL = {
    "mixer": dict(input_size=(56, 56), patch_size=8, embed_dim=64, nb_blocks=2, mlp_ratio=(0.5, 4.0), nb_classes=10),
    "mixer_5x6": dict(input_size=(40, 48), patch_size=8, embed_dim=48, nb_blocks=2, mlp_ratio=(1.0, 2.0), nb_classes=10),
    "gmixer": dict(input_size=(56, 56), patch_size=8, embed_dim=64, nb_blocks=2, mlp_ratio=(1.0, 4.0),
                   mlp_layer="glu_mlp", act_layer="swish", nb_classes=10),
    "resmlp": dict(input_size=(56, 56), patch_size=8, embed_dim=64, nb_blocks=2, mlp_ratio=(4.0, 4.0),
                   block_layer="res_block", norm_layer="affine", init_values=0.1, nb_classes=10),
    "gmlp": dict(input_size=(40, 48), patch_size=8, embed_dim=64, nb_blocks=2, mlp_ratio=(6.0, 6.0),
                 block_layer="spatial_gating_block", mlp_layer="gated_mlp", nb_classes=10),
}


def _model(mixer, precision, **kw):
    from oracle import mlp_mixer as om
    from oracle import params

    cfg = mixer.MLPMixerConfig(name="t", **kw)
    m = mixer.MLPMixer(cfg, precision=precision, device="cuda")
    w = params.random_params(om.param_shapes(cfg), seed=5)
    m.load_weights_dict(w)
    return m, cfg, w


@pytest.mark.parametrize("kind", list(SMALL))
def test_small_fp32_matches_oracle(mixer, kind):
    from oracle import mlp_mixer as om
    from oracle import params

    m, cfg, w = _model(mixer, "fp32", **SMALL[kind])
    x = params.test_images(3, *cfg.input_size)
    ref = om.forward(cfg, w, x)
    assert _nerr(m(x.cuda()), ref) < 1e-5


@pytest.mark.parametrize("kind", list(SMALL))
def test_small_bf16_matches_oracle(mixer, kind):
    from oracle import mlp_mixer as om
    from oracle import params
    from tfimm.backend import ops

    m, cfg, w = _model(mixer, "bf16", **SMALL[kind])
    x = params.test_images(3, *cfg.input_size)
    ref = om.forward(cfg, w, x)
    ops.trace = []
    try:
        out = m(x.cuda())
        names = {t[0] for t in ops.trace}
    finally:
        ops.trace = None
    assert "token_gemm_bf16" in names and "token_gemm_f32" not in names, names
    assert _nerr(out, ref) < 2e-2


# bf16 storage noise (2^-9 per rounding) grows with depth under random weights.  gMixer-24's gated products amplify
# it most: the fp32 engine measured 7.4e-5 there (about 9e-7 on the other four), bf16 0.253 (H100 SXM, 400 W limit).
# test_bf16_error_budget shows that this is the bf16 storage of the graph itself: the ideal bf16 graph (exact
# arithmetic, the same storage points) is as far from the oracle, and the kernels stay within the emulation floor.
BF16_BOUND = {"gmixer_24_224": 0.3}


@pytest.mark.parametrize("name", ["mixer_b16_224", "gmixer_24_224", "resmlp_24_224", "resmlp_big_24_224",
                                  "gmlp_s16_224"])
def test_registered_bf16_batch64(mixer, name):
    """Full-size registrations at batch 64 against the float64 oracle (run on the GPU), and which kernels ran."""
    import tfimm
    from oracle import mlp_mixer as om
    from oracle import params
    from tfimm.backend import ops

    m = tfimm.create_model(name, precision="bf16", device="cuda")
    cfg = m.cfg
    w = params.random_params(om.param_shapes(cfg), seed=11)
    m.load_weights_dict(w)
    x = params.test_images(64, *cfg.input_size).cuda()
    ops.trace = []
    try:
        out = m(x)
        names = [t[0] for t in ops.trace]
    finally:
        ops.trace = None
    assert "token_gemm_bf16" in names and "token_gemm_f32" not in names
    with torch.no_grad():
        ref = om.forward(cfg, {k: v.cuda() for k, v in w.items()}, x)
    m32 = tfimm.create_model(name, precision="fp32", device="cuda")
    m32.load_weights_dict(w)
    err32 = _nerr(m32(x[:8]), ref[:8])
    err = _nerr(out, ref)
    print(f"{name}: normalised max error vs float64 oracle: fp32 {err32:.3e}, bf16 {err:.3e}")
    assert err32 < 1e-4, err32
    assert err < BF16_BOUND.get(name, 3e-2), err


def test_cuda_graph_uint8_and_features(mixer):
    from tfimm.backend import ops

    m, cfg, w = _model(mixer, "bf16", **SMALL["gmlp"])
    x = torch.rand((256, *cfg.input_size, 3), device="cuda")
    eager = m(x)
    run = m.cuda_graph(256)
    assert torch.equal(run(x), eager)
    # raw uint8 pixels = the preprocessed float images
    u8 = torch.randint(0, 256, (4, *cfg.input_size, 3), dtype=torch.uint8, device="cuda")
    mean = torch.tensor(cfg.mean, device="cuda")
    std = torch.tensor(cfg.std, device="cuda")
    ref = m((u8.float() / 255.0 - mean) / std)
    assert _nerr(m(u8), ref) < 1e-2   # measured 3.2e-3: the first bf16 rounding of the two pixel paths differs
    _, feats = m(x[:2], return_features=True)
    assert list(feats) == m.feature_names
    assert ops.launch_count > 0


# ---------------------------------------------------------------- op by op
def _mixer_oracle():
    from pathlib import Path

    p = str(Path(__file__).resolve().parent)
    if p not in sys.path:
        sys.path.insert(0, p)
    import mixer_oracle

    return mixer_oracle


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", list(SMALL))
def test_shadowed_forward_small(mixer, kind, precision):
    """Every launch of a small forward checked against its own float64 statement within its derived bound."""
    from oracle import params

    m, cfg, w = _model(mixer, precision, **SMALL[kind])
    x = params.test_images(2, *cfg.input_size).cuda()
    with _mixer_oracle().shadowed_mixer_ops() as census:
        m(x)
    census.assert_ok()
    assert "token_gemm" in census.ops()


@pytest.mark.parametrize("name", ["mixer_b16_224", "gmixer_24_224", "resmlp_24_224", "resmlp_big_24_224",
                                  "gmlp_s16_224"])
def test_shadowed_forward_registered_batch64(mixer, name):
    """Full-size registrations in bf16 at batch 64, every launch checked op by op; the wgmma token kernel ran."""
    import tfimm
    from oracle import mlp_mixer as om
    from oracle import params
    from tfimm.backend import ops

    m = tfimm.create_model(name, precision="bf16", device="cuda")
    m.load_weights_dict(params.random_params(om.param_shapes(m.cfg), seed=11))
    x = params.test_images(64, *m.cfg.input_size).cuda()
    ops.trace = []
    try:
        with _mixer_oracle().shadowed_mixer_ops() as census:
            m(x)
        names = {t[0] for t in ops.trace}
    finally:
        ops.trace = None
    census.assert_ok()
    assert "token_gemm_bf16" in names and "token_gemm_f32" not in names, names
    if m.cfg.mlp_layer == "glu_mlp":
        assert "gemm_glu_bf16" in names


def _rms(a, b):
    return ((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("name", ["mixer_b16_224", "resmlp_24_224", "gmlp_s16_224", "gmixer_24_224"])
def test_bf16_error_budget(mixer, name):
    """B1 / B2 of tests/test_parity_budget_gpu.py: the kernels diverge from the ideal bf16 graph (emulated, float64
    arithmetic, the engine's bf16 storage points) by no more than 1.6 x the float64-vs-float32 emulation floor (B1), and
    add nothing measurable to the ideal graph's own distance from the float64 oracle (B2).  For gMixer-24 this shows its
    large bf16 error is the bf16 storage of the graph itself, not the kernels."""
    import tfimm
    from oracle import mlp_mixer as om
    from oracle import params

    mo = _mixer_oracle()
    m = tfimm.create_model(name, precision="bf16", device="cuda")
    w = params.random_params(om.param_shapes(m.cfg), seed=11)
    m.load_weights_dict(w)
    x = params.test_images(4, *m.cfg.input_size).cuda()
    y = m(x).double()
    with mo.emulated_mixer_ops():
        y_ideal = m(x).double()
    with mo.emulated_mixer_ops(arithmetic=torch.float32):
        y_ideal32 = m(x).double()
    with torch.no_grad():
        ref = om.forward(m.cfg, {k: v.cuda() for k, v in w.items()}, x)
    r_eng, r_ideal, r_kern, r_floor = _rms(y, ref), _rms(y_ideal, ref), _rms(y, y_ideal), _rms(y_ideal32, y_ideal)
    print(f"BUDGET {name}: rms engine-vs-oracle {r_eng:.2e} | ideal-vs-oracle {r_ideal:.2e} | engine-vs-ideal "
          f"{r_kern:.2e} | floor {r_floor:.2e}")
    assert r_kern < 1.6 * r_floor + 1e-4, (r_kern, r_floor)      # B1
    assert r_eng < 1.25 * r_ideal + 1e-4, (r_eng, r_ideal)       # B2
