"""CaiT family on CPU: opt-in registration (and the registry left as it was found), the C entry points' argument checks,
the attention dispatch, the refusals, the host orchestration on the float64 statements, the float32 shadow rehearsal and
seeded defects."""
import dataclasses
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))

NAMES = ["cait_m36_384", "cait_m48_448", "cait_s24_224", "cait_s24_384", "cait_s36_384", "cait_xs24_384",
         "cait_xxs24_224", "cait_xxs24_384", "cait_xxs36_224", "cait_xxs36_384"]


@pytest.fixture
def cait():
    from cait_oracle import cait_registered

    with cait_registered() as mod:
        yield mod


def test_import_tfimm_registers_nothing_new():
    code = ("import sys; sys.path[:0] = ['{0}', '{0}/tensorflow-image-models_b200']; import tfimm; "
            "from tfimm.models.registry import list_modules; print(len(tfimm.list_models()), sorted(list_modules()), "
            "'tfimm.architectures.cait' in sys.modules)").format(ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == "False"
    assert "'cait'" not in " ".join(out)


def test_registration_on_import(cait):
    import tfimm

    assert sorted(tfimm.list_models(module="cait")) == NAMES
    m = tfimm.create_model("cait_m48_448", device="meta")
    assert isinstance(m, cait.CaiT) and m.cfg.grid_size == (28, 28) and m.cfg.nb_patches == 784
    assert len(m.feature_names) == 1 + 48 + 1 + 2 + 3
    init = {n: tfimm.models.registry.model_config(n).init_scale for n in NAMES}
    assert {n for n, s in init.items() if s == 1e-6} == {"cait_s36_384", "cait_m36_384", "cait_m48_448"}
    assert set(init.values()) == {1e-5, 1e-6}


def test_param_specs_initial_values(cait):
    """gamma_1 / gamma_2 start at the registration's init_scale, cls_token and pos_embed at zero, as the reference's
    Constant / "zeros" initialisers."""
    import tfimm

    for name in ("cait_xxs24_224", "cait_s36_384"):
        cfg = tfimm.models.registry.model_config(name)
        specs = cait.param_specs(cfg)
        assert specs["blocks/0/gamma_1"].init == f"const:{cfg.init_scale!r}"
        assert specs["blocks_token_only/1/gamma_2"].init == f"const:{cfg.init_scale!r}"
        assert specs["cls_token"].init == specs["pos_embed"].init == "zeros"
        assert tuple(specs["blocks/3/attn/proj_l/kernel"].shape) == (cfg.nb_heads, cfg.nb_heads)
    m = cait.CaiT(cait.CaiTConfig(name="t", input_size=(32, 32), embed_dim=96, nb_heads=2, nb_blocks=1,
                                  init_scale=1e-6), precision="fp32", device="cpu")
    assert torch.equal(m.params["blocks/0/gamma_2"], torch.full((96,), 1e-6))


PREFIX = "tfimm_b200_"


def test_entry_point_argument_checks_past_the_shape():
    """Shapes without an instantiation, misaligned or missing pointers are refused before any CUDA call."""
    from tfimm.backend import lib

    h = lib.load()
    assert h.tfimm_b200_cait_talking_heads_bf16(16, 16, 16, 16, 16, 16, 2, 197, 12, 64, None) == 1
    assert "head_dim 48 and H in {4, 6, 8, 16} (got H=12 dh=64)" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_cait_talking_heads_bf16(16, 16, 16, 16, 16, 16, 2, 197, 5, 48, None) == 1
    assert h.tfimm_b200_cait_talking_heads_bf16(16, 24, 16, 16, 16, 16, 2, 197, 4, 48, None) == 1
    assert "16-byte aligned" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_cait_talking_heads_bf16(16, 16, None, 16, 16, 16, 2, 197, 4, 48, None) == 1
    assert h.tfimm_b200_cait_talking_heads_f32(16, 16, 16, 16, 16, 16, 2, 197, 5, 48, None) == 1
    assert "H in {1, 2, 3, 4, 6, 8, 12, 16}" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_cait_talking_heads_f32(16, 16, 16, 16, 16, 16, 2, 197, 4, 50, None) == 1
    assert h.tfimm_b200_cait_talking_heads_f32(16, 16, 16, 16, 16, 16, 2, 197, 4, 68, None) == 1
    assert h.tfimm_b200_cait_class_attention(16, 16, 16, lib.F32, 2, 197, 4, 40, 0.1, None) == 1
    assert "head_dim must be 32, 48 or 64 (got 40)" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_cait_class_attention(16, 16, 16, lib.U8, 2, 197, 4, 48, 0.1, None) == 1
    assert h.tfimm_b200_cait_add_pos(16, 24, 2, 196, 192, None) == 1
    assert "16-byte aligned" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_cait_add_pos(16, 16, 2, 196, 190, None) == 1


def test_trace_family_names_and_counts():
    from tfimm.backend import cait_ops, ops

    sys.path.insert(0, str(ROOT / "tools"))
    import ncu_traffic

    ns = "void tfimm::(anonymous namespace)::"
    for kernel, fam in (("cait_talking_heads_bf16_kernel<16, 32, 16>(const __nv_bfloat16 *)", "cait_talking_heads_bf16"),
                        ("cait_talking_heads_f32_kernel<6>(const float *)", "cait_talking_heads_f32"),
                        ("cait_class_attn_kernel<float, 48>(const float *)", "cait_class_attention"),
                        ("cait_add_pos_kernel(float4 *)", "cait_add_pos")):
        assert ncu_traffic.family_of(ns + kernel) == fam == ops.TRACE_FAMILY[PREFIX + fam]
    # q k^T twice and P' V once (2 H dh FMA each per pair), the two H x H mixes (pre-mix twice)
    assert cait_ops.talking_heads_flops(2, 196, 4, 48) == 2.0 * 2 * 196 * 196 * (3 * 192 + 3 * 16)


def test_fold_premix():
    """dh^-0.5 log2 e multiplies proj_l's kernel; the bias takes log2 e only."""
    from tfimm.backend import cait_ops

    wl, bl = torch.randn(4, 4), torch.randn(4)
    fw, fb = cait_ops.fold_premix(wl, bl, 48)
    assert torch.equal(fw, (wl.double() * 48 ** -0.5 * cait_ops.LOG2E).float())
    assert torch.equal(fb, (bl.double() * cait_ops.LOG2E).float())


def test_attention_dispatch(monkeypatch):
    from tfimm.backend import cait_ops, lib

    calls = []
    monkeypatch.setattr(cait_ops, "talking_heads_bf16", lambda *a: calls.append(("bf16", a[-2], a[-1])))
    monkeypatch.setattr(cait_ops, "talking_heads_f32", lambda *a: calls.append(("f32", a[-2], a[-1])))
    w, b = torch.zeros(4, 4), torch.zeros(4)
    cait_ops.talking_heads(torch.zeros((5, 576), dtype=torch.bfloat16), w, b, w, b, 1, 5, 4, 48)
    cait_ops.talking_heads(torch.zeros((5, 576)), w, b, w, b, 1, 5, 4, 48)
    assert calls == [("bf16", 4, 48), ("f32", 4, 48)]
    with pytest.raises(lib.KernelLibraryError, match="no bf16 kernel for H=12"):
        cait_ops.talking_heads(torch.zeros((5, 3 * 768), dtype=torch.bfloat16), w, b, w, b, 1, 5, 12, 64)
    with pytest.raises(lib.KernelLibraryError, match="no fp32 kernel for H=5"):
        cait_ops.talking_heads(torch.zeros((5, 3 * 240)), w, b, w, b, 1, 5, 5, 48)


def test_refusals(cait):
    C = cait.CaiTConfig
    with pytest.raises(ValueError, match="normalization"):
        cait.CaiT(C(name="t", norm_layer="batch_norm"), device="meta")
    with pytest.raises(ValueError, match="activation"):
        cait.CaiT(C(name="t", act_layer="mish"), device="meta")
    with pytest.raises(ValueError, match="multiple of nb_heads"):
        cait.CaiT(C(name="t", embed_dim=200, nb_heads=3), device="meta")
    with pytest.raises(ValueError, match="no bf16 talking-heads kernel for nb_heads 12 at head_dim 64"):
        cait.CaiT(C(name="t"), device="meta")          # the config defaults: 768 / 12
    cait.CaiT(C(name="t"), precision="fp32", device="meta")
    with pytest.raises(ValueError, match="no fp32 talking-heads kernel"):
        cait.CaiT(C(name="t", embed_dim=240, nb_heads=5), precision="fp32", device="meta")
    with pytest.raises(ValueError, match="class attention needs head_dim"):
        cait.CaiT(C(name="t", embed_dim=64, nb_heads=4), precision="fp32", device="meta")


def test_input_smaller_than_a_patch_is_refused_before_any_launch(cait, cpu_engine):
    from tfimm.backend import ops

    m = cait.CaiT(cait.CaiTConfig(name="t", input_size=(32, 32), embed_dim=96, nb_heads=2, nb_blocks=1,
                                  interpolate_input=True), precision="fp32", device="cpu")
    before = ops.launch_count
    with pytest.raises(ValueError, match="smaller than the patch size"):
        m(torch.zeros((1, 12, 40, 3)))
    with pytest.raises(ValueError, match="does not match"):
        cait.CaiT(dataclasses.replace(m.cfg, interpolate_input=False), precision="fp32", device="cpu")(
            torch.zeros((1, 48, 32, 3)))
    assert ops.launch_count == before


def test_transform_pos_embed(cait):
    """transform_weights["pos_embed"] resizes the (1, N, D) table bicubically on its grid (nb_tokens = 0)."""
    import tfimm
    from oracle import cait as oc

    cfg = tfimm.models.registry.model_config("cait_xxs24_224")
    m = cait.CaiT(cfg, device="cpu")
    m.params["pos_embed"].copy_(torch.randn(m.params["pos_embed"].shape))
    tgt = dataclasses.replace(cfg, input_size=(288, 160))
    got = cfg.transform_weights["pos_embed"](m, m.params["pos_embed"], tgt)
    assert got.shape == (1, 18 * 10, 192)
    ref = oc.interpolate_pos_embeddings(m.params["pos_embed"].double(), (14, 14), (18, 10))
    assert (got.double() - ref).abs().max().item() < 1e-6


def test_timm_state_dict_loads(cait):
    """A timm CaiT state dict: (H, H) proj_l / proj_w Linear weights (transposed into Dense kernels), gamma_1 / gamma_2
    and the (1, 1, D) / (1, N, D) tokens, loaded strictly."""
    from tfimm.utils.timm import load_pytorch_weights_in_model, pytorch_key

    m = cait.CaiT(cait.CaiTConfig(name="t", input_size=(32, 48), embed_dim=96, nb_heads=2, nb_blocks=1,
                                  nb_classes=3), precision="fp32", device="cpu")
    gen = torch.Generator().manual_seed(3)
    sd = {}
    for k, v in m.params.items():
        shape = tuple(v.shape)
        if k.endswith("kernel"):
            shape = (shape[3], shape[2], shape[0], shape[1]) if len(shape) == 4 else shape[::-1]
        sd[pytorch_key(k)] = torch.randn(shape, generator=gen)
    assert "blocks.0.attn.proj_l.weight" in sd and "blocks_token_only.1.gamma_2" in sd
    missing, unexpected = load_pytorch_weights_in_model(m, sd)
    assert missing == [] and unexpected == []
    assert torch.equal(m.params["blocks/0/attn/proj_l/kernel"], sd["blocks.0.attn.proj_l.weight"].t())
    assert torch.equal(m.params["blocks/0/gamma_1"], sd["blocks.0.gamma_1"])
    with pytest.raises(Exception):
        m.load_weights_dict({k: v for k, v in m.params.items() if k != "blocks/0/gamma_1"})


# ---------------------------------------------------------------- host orchestration on emulated kernels
SMALL = {
    # 2 x 3 patches, H = 2 at head dim 48: the fp32 kernels' shapes
    "plain": dict(input_size=(32, 48), embed_dim=96, nb_heads=2, nb_blocks=2, nb_classes=5),
    # D = 192, H = 4 (the bf16 kernel's cait_xxs shape and the fused MLP), interpolated to a 3 x 5 grid, no head
    "xxs": dict(input_size=(32, 32), embed_dim=192, nb_heads=4, nb_blocks=1, nb_classes=0, interpolate_input=True),
    # D = 288, H = 6 (the unfused MLP in bf16), without qkv biases
    "xs": dict(input_size=(48, 32), embed_dim=288, nb_heads=6, nb_blocks=1, nb_classes=3, qkv_bias=False),
}
IMAGE = {"xxs": (48, 80)}


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def small(cait, kind, precision, batch=2):
    from cait_oracle import randomise
    from oracle import params

    cfg = cait.CaiTConfig(name="t", **SMALL[kind])
    m = cait.CaiT(cfg, precision=precision, device="cpu")
    w = randomise(params.random_params({k: tuple(v.shape) for k, v in m.params.items()}, seed=5), 6)
    m.load_weights_dict(w)
    return m, cfg, w, params.test_images(batch, *IMAGE.get(kind, cfg.input_size))


def test_randomised_weights_expose_the_defects(cait):
    m, cfg, w, _ = small(cait, "plain", "fp32")
    wl = w["blocks/0/attn/proj_l/kernel"]
    assert not torch.allclose(wl, wl.t()) and w["blocks/0/attn/proj_w/bias"].abs().min() > 0
    assert not torch.equal(w["blocks/0/gamma_1"], w["blocks/0/gamma_2"]) and w["cls_token"].abs().max() > 0


@pytest.mark.parametrize("kind", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(cait, cpu_engine, kind):
    """The host graph with every kernel replaced by its float64 statement (fp32 storage) is the oracle's forward, to
    1e-6 of each feature."""
    from cait_oracle import emulated_cait_ops
    from oracle import cait as oc

    m, cfg, w, x = small(cait, kind, "fp32")
    with emulated_cait_ops():
        y, feats = m(x, return_features=True)
    ref, rfeats = oc.forward(cfg, w, x, return_features=True)
    assert list(feats) == list(rfeats) == m.feature_names
    for k in rfeats:
        assert feats[k].shape == rfeats[k].shape, k
        assert (feats[k].double() - rfeats[k]).abs().max().item() <= 1e-6 * rfeats[k].abs().max().item(), k


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", ["xxs", "xs"])
def test_shadow_rehearsal_float32_stand_in(cait, cpu_engine, kind, precision):
    """The op-by-op harness on CPU: the float32 evaluation of every statement plays the kernels; every launch is inside
    its bound and the CaiT launchers of the precision are reached."""
    from cait_oracle import emulated_cait_ops, shadowed_cait_ops

    m, cfg, w, x = small(cait, kind, precision)
    with emulated_cait_ops(torch.float32), shadowed_cait_ops() as census:
        m(x)
    census.assert_ok()
    want = {"add_pos", "assemble_tokens", "im2col", "gemm", "layernorm", "class_attention",
            "talking_heads_bf16" if precision == "bf16" else "talking_heads_f32"}
    assert want <= census.ops(), census.ops()


# ---------------------------------------------------------------- seeded defects
def _th_variant(transpose_l=False, transpose_w=False, drop_bw=False, softmax_heads=False, mask_before=False,
                round_p=True):
    """A float32 stand-in of the talking-heads launcher with one seeded defect."""
    def f(qkv, wl, bl, ww, bw, B, N, H, dh):
        hp = torch.float32
        wl_, ww_ = (wl.t() if transpose_l else wl), (ww.t() if transpose_w else ww)
        bw_ = torch.zeros_like(bw) if drop_bw else bw
        out = []
        for b in range(B):
            q, k, v = qkv[b * N:(b + 1) * N].to(hp).view(N, 3, H, dh).permute(1, 2, 0, 3)
            S = q @ k.transpose(-1, -2)
            if mask_before:   # keys padded to the 32-key block, masked on S before the mix: -inf * w
                pad = -(-N // 32) * 32 - N
                S = torch.cat((S, torch.full((H, N, pad), -float("inf"))), -1)
                v = torch.cat((v, torch.zeros(H, pad, dh)), 1)
            L = torch.einsum("hqk,hg->gqk", S, wl_) + bl[:, None, None]
            P = torch.softmax(L * math.log(2), dim=0 if softmax_heads else -1)
            Pp = torch.einsum("gqk,gf->fqk", P, ww_) + bw_[:, None, None]
            Pp = Pp.to(torch.bfloat16).to(hp) if round_p else Pp
            out.append(torch.nan_to_num(Pp @ v).permute(1, 0, 2).reshape(N, H * dh))
        return torch.cat(out).to(qkv.dtype)
    return f



def _defect(name):
    """(launcher module, launcher name, float32 stand-in) of a seeded kernel defect."""
    from tfimm.backend import cait_ops

    th = {"proj_l_transposed": dict(transpose_l=True), "proj_w_transposed": dict(transpose_w=True),
          "bw_dropped": dict(drop_bw=True), "softmax_over_heads": dict(softmax_heads=True),
          "mask_before_mix": dict(mask_before=True)}
    if name in th:
        return cait_ops, "talking_heads_f32", _th_variant(round_p=False, **th[name])
    raise KeyError(name)


@pytest.mark.parametrize("defect", ["proj_l_transposed", "proj_w_transposed", "bw_dropped", "softmax_over_heads",
                                    "mask_before_mix"])
def test_seeded_kernel_defects_are_rejected(cait, cpu_engine, defect):
    """Each seeded kernel defect makes the harness fail, and the failing rows name the launcher that carries it."""
    from cait_oracle import emulated_cait_ops, shadowed_cait_ops

    m, cfg, w, x = small(cait, "plain", "fp32", batch=3)
    module, op, bad = _defect(defect)
    with emulated_cait_ops(torch.float32):
        setattr(module, op, bad)
        with shadowed_cait_ops() as census:
            m(x)
    fails = census.failures()
    assert fails and {r["op"] for r in fails} == {op}, census.table()


def _first_bad_feature(m, cfg, w, x):
    from cait_oracle import emulated_cait_ops
    from oracle import cait as oc

    with emulated_cait_ops():
        _, feats = m(x, return_features=True)
    _, rfeats = oc.forward(cfg, w, x, return_features=True)
    for k in rfeats:
        if (feats[k].double() - rfeats[k]).abs().max().item() > 1e-6 * rfeats[k].abs().max().item():
            return k
    return None


def test_seeded_plan_defects_are_caught_at_their_layer(cait, cpu_engine, monkeypatch):
    """Defects of the host graph, caught by the float64 orchestration against the oracle and named by the first
    feature they move: gamma_1 and gamma_2 swapped, the first position's embedding added to the class token, and the class blocks' MLP update landing on
    the patch rows."""
    from tfimm.backend import cait_ops

    m, cfg, w, x = small(cait, "plain", "fp32")
    assert _first_bad_feature(m, cfg, w, x) is None

    real_vec = type(m)._vec

    def swapped(self, key):
        if key.endswith("gamma_1"):
            key = key[:-1] + "2"
        elif key.endswith("gamma_2"):
            key = key[:-1] + "1"
        return real_vec(self, key)
    monkeypatch.setattr(type(m), "_vec", swapped)
    m._plan = None
    assert _first_bad_feature(m, cfg, w, x) == "block_0"
    monkeypatch.setattr(type(m), "_vec", real_vec)

    real_table = type(m)._pos_table

    def pos_on_cls(self, P, grid):
        pos, zeros = real_table(self, P, grid)
        bad = zeros.clone()
        bad[0] = pos[0]
        return pos, bad
    monkeypatch.setattr(type(m), "_pos_table", pos_on_cls)
    m._plan = None
    assert _first_bad_feature(m, cfg, w, x) == "features_cls_token"
    monkeypatch.setattr(type(m), "_pos_table", real_table)

    real_mlp = type(m)._mlp

    def mlp_on_all_rows(self, blk, xs):
        if xs.stride(0) != xs.shape[1]:   # the class rows: run the MLP on every row of the stream instead
            B = xs.shape[0]
            full = xs.as_strided((B * (xs.stride(0) // xs.shape[1]), xs.shape[1]), (xs.shape[1], 1))
            return real_mlp(self, blk, full)
        return real_mlp(self, blk, xs)
    monkeypatch.setattr(type(m), "_mlp", mlp_on_all_rows)
    m._plan = None
    assert _first_bad_feature(m, cfg, w, x) == "block_cls_token_0"


def test_scale_after_the_premix_is_invisible(cait, cpu_engine, monkeypatch):
    """The scale applied after the pre-mix differs from the reference only in proj_l's bias, which it would multiply
    by dh^-0.5 too.  That bias is one constant per (query, g) across all keys, so the softmax over keys cancels it: no
    output can show this defect.  The plan keeps the bias unscaled, as the reference computes it; this test records
    that the two agree to float64 rounding."""
    from cait_oracle import emulated_cait_ops
    from tfimm.backend import cait_ops

    m, cfg, w, x = small(cait, "plain", "fp32")
    with emulated_cait_ops():
        good = m(x)
    real_fold = cait_ops.fold_premix
    monkeypatch.setattr(cait_ops, "fold_premix", lambda wl, bl, dh: (real_fold(wl, bl, dh)[0],
                                                                      (bl.double() * dh ** -0.5 * cait_ops.LOG2E).float()))
    m._plan = None
    assert not torch.equal(m._ensure_plan()["blocks"][0]["bl"], real_fold(m.params["blocks/0/attn/proj_l/kernel"],
                                                                           m.params["blocks/0/attn/proj_l/bias"],
                                                                           48)[1])
    with emulated_cait_ops():
        bad = m(x)
    assert (good.double() - bad.double()).abs().max().item() <= 1e-6 * good.abs().max().item()


def test_pins_exist():
    pins = ROOT / "tests" / "golden" / "reference" / "cait_pins.npz"
    assert pins.exists()
    meta = __import__("json").loads(bytes(np.load(pins)["meta"]).decode())
    assert sorted(meta["registry"]) == NAMES
