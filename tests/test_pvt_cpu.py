"""PVT family on CPU: opt-in registration (and the registry left as it was found), the C entry points' argument checks,
the attention dispatch, refusals, the host orchestration on the float64 statements, the statements against the existing
attention statement, the float32 shadow rehearsal and seeded defects."""
import dataclasses
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))


@pytest.fixture
def pvt():
    from pvt_oracle import pvt_registered

    with pvt_registered() as mod:
        yield mod


def test_import_tfimm_registers_nothing_new():
    code = ("import sys; sys.path[:0] = ['{0}', '{0}/tensorflow-image-models_b200']; import tfimm; "
            "from tfimm.models.registry import list_modules; print(len(tfimm.list_models()), sorted(list_modules()), "
            "'tfimm.architectures.pvt' in sys.modules)").format(ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == "False"
    assert "'pvt'" not in " ".join(out)


def test_registration_on_import(pvt):
    import tfimm

    assert sorted(tfimm.list_models(module="pvt")) == ["pvt_large", "pvt_medium", "pvt_small", "pvt_tiny"]
    m = tfimm.create_model("pvt_small", device="meta")
    assert isinstance(m, pvt.PyramidVisionTransformer)
    assert m.cfg.grid_size == ((56, 56), (28, 28), (14, 14), (7, 7)) and m.cfg.nb_tokens == (0, 0, 0, 1)
    assert len(m.feature_names) == 4 * 3 + 16 + 3
    assert m.params["block1/0/attn/sr/kernel"].shape == (8, 8, 64, 64)
    assert m.params["pos_embed4"].shape == (1, 50, 512) and "block4/0/attn/sr/kernel" not in m.params


PREFIX = "tfimm_b200_"


def test_entry_point_argument_checks_past_the_shape():
    """Head dims other than 64, too many images or heads, misaligned pointers and a class row without cls are refused
    before any CUDA call."""
    from tfimm.backend import lib

    h = lib.load()
    assert h.tfimm_b200_pvt_sr_attention_bf16(16, 16, 16, 2, 197, 49, 4, 32, 0.1, None) == 1
    assert "head_dim must be 64 (got 32)" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pvt_sr_attention_bf16(16, 16, 16, 65536, 197, 49, 1, 64, 0.1, None) == 1
    assert "need B, H <= 65535" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pvt_sr_attention_bf16(16, 24, 16, 2, 197, 49, 4, 64, 0.1, None) == 1
    assert "16-byte aligned" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pvt_sr_attention_f32(16, 16, 8, 2, 197, 49, 4, 64, 0.1, None) == 1
    assert "16-byte aligned" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pvt_sr_attention_f32(16, 16, 16, 2, 197, 49, 4, 48, 0.1, None) == 1
    assert "head_dim must be 64 (got 48)" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pvt_embed_norm(16, 16, 16, 16, None, 16, 2, 49, 1, 512, 1e-5, None) == 1
    assert "ntok = 1 needs a 16-byte aligned cls" in h.tfimm_b200_last_error().decode()
    assert h.tfimm_b200_pvt_embed_norm(16, 16, 16, 16, None, 16, 2, 49, 0, 66, 1e-5, None) == 1
    assert h.tfimm_b200_pvt_embed_norm(16, 16, 16, 16, None, 16, 2, 49, 2, 64, 1e-5, None) == 1


def test_trace_family_names():
    from tfimm.backend import ops

    sys.path.insert(0, str(ROOT / "tools"))
    import ncu_traffic

    ns = "tfimm::(anonymous namespace)::"
    for kernel, fam in ((f"{ns}pvt_sr_attention_bf16_kernel(const __nv_bfloat16 *)", "pvt_sr_attention_bf16"),
                        (f"{ns}pvt_sr_attention_f32_kernel(const float *)", "pvt_sr_attention_f32"),
                        (f"void {ns}pvt_embed_norm_kernel<4>(const float *)", "pvt_embed_norm")):
        assert ncu_traffic.family_of(kernel) == fam == ops.TRACE_FAMILY[PREFIX + fam]


def test_byte_counts():
    from tfimm.backend import pvt_ops

    # pvt_small stage 0 at batch 256: q read and out written (3136 x 64 bf16 each), k and v read (49 x 64 each)
    assert pvt_ops.sr_attention_nbytes(256, 3136, 49, 1, 64, 2) == 2.0 * 256 * 64 * (2 * 3136 + 2 * 49)
    assert abs(pvt_ops.sr_attention_nbytes(256, 3136, 49, 1, 64, 2) / 1e6 - 208.7) < 0.1
    assert pvt_ops.embed_norm_nbytes(2, 49, 1, 512) == 4.0 * (2 * 49 * 512 + 2 * 50 * 512 + 50 * 512 + 3 * 512)


def test_attention_dispatch(monkeypatch):
    """bf16 -> the tensor-core kernel, fp32 (the fp32 and tf32 models) -> the fp32 kernel; other head dims refused."""
    from tfimm.backend import lib, pvt_ops

    calls = []
    monkeypatch.setattr(pvt_ops, "pvt_sr_attention_bf16", lambda q, kv, B, N, Nk, H, dh, s: calls.append("bf16"))
    monkeypatch.setattr(pvt_ops, "pvt_sr_attention_f32", lambda q, kv, B, N, Nk, H, dh, s: calls.append("f32"))
    pvt_ops.sr_attention(torch.zeros((5, 64), dtype=torch.bfloat16), torch.zeros((2, 128), dtype=torch.bfloat16),
                         1, 5, 2, 1, 64, 0.125)
    pvt_ops.sr_attention(torch.zeros((5, 64)), torch.zeros((2, 128)), 1, 5, 2, 1, 64, 0.125)
    assert calls == ["bf16", "f32"]
    with pytest.raises(lib.KernelLibraryError, match="head_dim 32"):
        pvt_ops.sr_attention(torch.zeros((5, 64), dtype=torch.bfloat16), torch.zeros((2, 128), dtype=torch.bfloat16),
                             1, 5, 2, 2, 32, 0.1)


def test_refusals(pvt):
    """Head dims other than 64, a spatial reduction in the class-token stage, grids smaller than their ratio and
    inputs of another size without interpolate_input are refused with ValueError before any launch."""
    C = pvt.PyramidVisionTransformerConfig
    P = pvt.PyramidVisionTransformer
    with pytest.raises(ValueError, match="normalization"):
        P(C(name="t", norm_layer="batch_norm"), device="meta")
    with pytest.raises(ValueError, match="head_dim 64/2 must be 64"):
        P(C(name="t", embed_dim=(64, 64, 320, 512)), device="meta")
    with pytest.raises(ValueError, match="sr_ratio"):
        P(C(name="t", embed_dim=(64, 128, 320, 512), sr_ratio=(8, 4, 2, 2)), device="meta")
    with pytest.raises(ValueError, match="one entry per stage"):
        P(C(name="t", embed_dim=(64, 128, 320, 512), sr_ratio=(8, 4, 1)), device="meta")
    m = P(C(name="t", embed_dim=(64, 128, 320, 512)), device="cpu")   # launches would fail on the CPU: none happens
    with pytest.raises(ValueError, match="does not match"):
        m(torch.zeros((1, 160, 224, 3)))
    m = P(C(name="t", embed_dim=(64, 128, 320, 512), interpolate_input=True), device="cpu")
    with pytest.raises(ValueError, match="stage 0's grid 7 x 8 is smaller than its patch or spatial-reduction ratio 8"):
        m(torch.zeros((1, 28, 32, 3)))
    m = P(C(name="t", embed_dim=(64, 128, 320, 512), sr_ratio=(2, 4, 2, 1), interpolate_input=True), device="cpu")
    with pytest.raises(ValueError, match="stage 1's grid 3 x 3 is smaller"):
        m(torch.zeros((1, 24, 24, 3)))
    with pytest.raises(NotImplementedError):
        m(torch.zeros((1, 64, 64, 3)), training=True)


def test_transform_pos_embed(pvt):
    """transform_weights["pos_embed{j}"] resizes each stage's table bicubically (tf.image.resize, float32) to the target
    grid, keeping the class row of the last stage."""
    import tfimm
    from oracle import pvt as op

    cfg = tfimm.models.registry.model_config("pvt_tiny")
    m = pvt.PyramidVisionTransformer(cfg, device="cpu")
    for k in m.params:
        if k.startswith("pos_embed"):
            m.params[k] = torch.randn(m.params[k].shape, generator=torch.Generator().manual_seed(3))
    tgt = dataclasses.replace(cfg, input_size=(200, 264))
    assert set(cfg.transform_weights) == {"pos_embed1", "pos_embed2", "pos_embed3", "pos_embed4"}
    for j, want in enumerate(((1, 50 * 66, 64), (1, 25 * 33, 128), (1, 12 * 16, 320), (1, 1 + 6 * 8, 512))):
        key = f"pos_embed{j + 1}"
        got = cfg.transform_weights[key](m, m.params[key], tgt)
        assert got.shape == want
        ref = op.interpolate_pos_embeddings(m.params[key].double(), cfg.grid_size[j], tgt.grid_size[j],
                                            cfg.nb_tokens[j])
        assert (got.double() - ref).abs().max().item() < 1e-6, key
    assert torch.equal(cfg.transform_weights["pos_embed4"](m, None, tgt)[:, 0], m.params["pos_embed4"][:, 0])


# ---------------------------------------------------------------- the statements
def _packed(B, N, H, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((B * N, 3 * H * 64), generator=g) * 1.5).to(dtype)


def _split_packed(qkv, B, N, H):
    """q and kv (the kv Dense's (2, H, dh) layout) cut from a packed [q | k | v] qkv."""
    x = qkv.view(B * N, 3, H * 64)
    return x[:, 0].contiguous(), x[:, 1:].reshape(B * N, 2 * H * 64).contiguous()


@pytest.mark.parametrize("N", [1, 17, 64, 65, 130])
def test_sr_statement_equals_the_attention_statement_on_a_packed_qkv(N):
    """Cut from one packed qkv (N' = N), the bf16 SRA statement is emulate_bf16.attention bit for bit, and its bound is
    shadow._blocked_attention_bound's."""
    import pvt_oracle as po
    from oracle import emulate_bf16 as emu
    from oracle import shadow

    B, H = 2, 3
    qkv = _packed(B, N, H, N, torch.bfloat16)
    q, kv = _split_packed(qkv, B, N, H)
    assert torch.equal(po.pvt_sr_attention_bf16(q, kv, B, N, N, H, 64, 0.125), emu.attention(qkv, B, N, H, 64, 0.125))
    got = po.sr_attention_bound(q, kv, B, N, N, H, 64, 0.125, emu.KEY_BLOCK, emu.round_bf16, shadow._UT, 67,
                                shadow._UT)
    assert torch.equal(got, shadow._blocked_attention_bound(qkv, B, N, H, 64, 0.125, emu.round_bf16))


def test_sr_statement_is_the_blocked_softmax_pv():
    """With N' != N the statement is _softmax_pv(scale q k^T, v, round_bf16, 64) per head, k / v read from the
    (2, H, dh) halves of kv."""
    import pvt_oracle as po
    from oracle import emulate_bf16 as emu

    B, N, Nk, H = 2, 70, 100, 2
    g = torch.Generator().manual_seed(1)
    q = torch.randn((B * N, H * 64), generator=g).to(torch.bfloat16)
    kv = torch.randn((B * Nk, 2 * H * 64), generator=g).to(torch.bfloat16)
    got = po.pvt_sr_attention_bf16(q, kv, B, N, Nk, H, 64, 0.125).view(B, N, H, 64)
    for b in range(B):
        for h in range(H):
            qh = q.view(B, N, H, 64)[b, :, h].double()
            k = kv.view(B, Nk, 2 * H, 64)[b, :, h].double()
            v = kv.view(B, Nk, 2 * H, 64)[b, :, H + h].double()
            want = emu._softmax_pv(0.125 * qh @ k.T, v, emu.round_bf16, 64)[0].to(torch.bfloat16)
            assert torch.equal(got[b, :, h], want)
    # fp32: the exact softmax, one rounding
    qf, kvf = q.float(), kv.float()
    want = torch.softmax(0.125 * qf.double().view(B, N, H, 64).transpose(1, 2) @
                         kvf.double().view(B, Nk, 2, H, 64)[:, :, 0].permute(0, 2, 3, 1), -1)
    want = (want @ kvf.double().view(B, Nk, 2, H, 64)[:, :, 1].transpose(1, 2)).transpose(1, 2).reshape(B * N, -1)
    assert torch.equal(po.pvt_sr_attention_f32(qf, kvf, B, N, Nk, H, 64, 0.125), want.float())


# ---------------------------------------------------------------- host orchestration on emulated kernels
_D = dict(embed_dim=(64, 128, 64, 64), nb_heads=(1, 2, 1, 1), nb_blocks=(1, 1, 1, 1), mlp_ratio=(2.0, 2.0, 2.0, 1.0))
SMALL = {
    # grids 16 x 16 -> 8 x 8 -> 4 x 4 -> 2 x 2 (+ class row); keys 16, 16, 4, 5; stage 1 runs the fused MLP in bf16
    "plain": (dict(input_size=(64, 64), sr_ratio=(4, 2, 2, 1), nb_classes=5, **_D), (64, 64)),
    # a 72 x 92 image: grids 18 x 23 -> 9 x 11 -> 4 x 5 -> 2 x 2; the sr convolutions drop rows and columns
    "odd": (dict(input_size=(64, 64), sr_ratio=(4, 2, 2, 1), interpolate_input=True, nb_classes=3, **_D), (72, 92)),
    # grids 8 x 8 -> 4 x 4 -> 2 x 2 -> 1 x 1; stages 2 and 3 attend to themselves; no head
    "noclass": (dict(input_size=(32, 32), sr_ratio=(2, 2, 1, 1), nb_classes=0, **_D), (32, 32)),
}


@pytest.fixture
def cpu_engine(monkeypatch):
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    monkeypatch.setattr(Model, "_ensure_plan", ensure_plan)


def _small(pvt, kind, precision, batch=2):
    from oracle import params
    from oracle import pvt as op

    fields, size = SMALL[kind]
    cfg = pvt.PyramidVisionTransformerConfig(name="t", **fields)
    m = pvt.PyramidVisionTransformer(cfg, precision=precision, device="cpu")
    w = params.random_params(op.param_shapes(cfg), seed=5)
    m.load_weights_dict(w)
    return m, cfg, w, params.test_images(batch, *size)


def test_param_specs_equal_the_oracle_tables(pvt):
    import tfimm
    from oracle import pvt as op

    for name in ("pvt_tiny", "pvt_large"):
        cfg = tfimm.models.registry.model_config(name)
        m = pvt.PyramidVisionTransformer(cfg, device="meta")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(op.param_shapes(cfg).items())
    for kind in SMALL:
        cfg = pvt.PyramidVisionTransformerConfig(name="t", **SMALL[kind][0])
        m = pvt.PyramidVisionTransformer(cfg, device="cpu")
        assert [(k, tuple(v.shape)) for k, v in m.params.items()] == list(op.param_shapes(cfg).items())


@pytest.mark.parametrize("kind", list(SMALL))
def test_fp32_orchestration_reproduces_the_oracle(pvt, cpu_engine, kind):
    """The host graph with every kernel replaced by its float64 statement (fp32 storage) is the oracle's forward, every
    feature with the reference's name and shape."""
    from oracle import pvt as op
    from pvt_oracle import emulated_pvt_ops

    m, cfg, w, x = _small(pvt, kind, "fp32")
    with emulated_pvt_ops():
        y, feats = m(x, return_features=True)
        y_plain = m(x)
    ref, rfeats = op.forward(cfg, w, x, return_features=True)
    assert list(feats) == list(rfeats) == m.feature_names
    for k in rfeats:
        assert feats[k].shape == rfeats[k].shape, k
        assert (feats[k].double() - rfeats[k]).abs().max().item() <= 1e-5 * rfeats[k].abs().max().item(), k
    assert torch.equal(y, y_plain)


@pytest.mark.parametrize("precision", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("kind", list(SMALL))
def test_shadow_rehearsal_float32_stand_in(pvt, cpu_engine, kind, precision):
    """The op-by-op harness on CPU: the float32 evaluation of every statement plays the kernels; every launch is inside
    its bound and the PVT launchers of the precision are reached."""
    from pvt_oracle import emulated_pvt_ops, shadowed_pvt_ops

    m, cfg, w, x = _small(pvt, kind, precision)
    with emulated_pvt_ops(torch.float32), shadowed_pvt_ops() as census:
        m(x)
    census.assert_ok()
    want = {"pvt_embed_norm", "im2col", "gemm", "layernorm",
            "pvt_sr_attention_bf16" if precision == "bf16" else "pvt_sr_attention_f32"}
    if precision == "bf16":
        want.add("mlp_fused")
    assert want <= census.ops(), census.ops()


def _defect(name):
    """A float32 stand-in of a launcher with one seeded defect: (launcher module, launcher name, function)."""
    import pvt_oracle as po
    from oracle import emulate_bf16 as emu
    from tfimm.backend import ops, pvt_ops

    def attention(q, kv, B, N, Nk, H, dh, scale, heads_outer=False):
        qh = q.float().view(B, N, H, dh).permute(0, 2, 1, 3)
        x = kv.float().view(B, Nk, *((H, 2) if heads_outer else (2, H)), dh)
        k, v = (x[:, :, :, 0], x[:, :, :, 1]) if heads_outer else (x[:, :, 0], x[:, :, 1])
        o = torch.softmax(scale * qh @ k.permute(0, 2, 3, 1), -1) @ v.permute(0, 2, 1, 3)
        return o.permute(0, 2, 1, 3).reshape(B * N, H * dh).to(q.dtype)

    if name == "k_v_swapped":
        def f(q, kv, B, N, Nk, H, dh, scale):
            swapped = kv.view(B * Nk, 2, H * dh).flip(1).reshape(B * Nk, -1)
            return attention(q, swapped, B, N, Nk, H, dh, scale)
        return pvt_ops, "pvt_sr_attention_bf16", f
    if name == "kv_split_h_2_dh":
        def f(q, kv, B, N, Nk, H, dh, scale):
            return attention(q, kv, B, N, Nk, H, dh, scale, heads_outer=True)
        return pvt_ops, "pvt_sr_attention_f32", f
    if name == "embed_norm_eps_1e-6":
        def f(tok, gamma, beta, pos, cls, B, P, eps):
            return po.pvt_embed_norm(tok, gamma, beta, pos, cls, B, P, 1e-6)
        return pvt_ops, "pvt_embed_norm", f
    if name == "sr_norm_eps_1e-6":
        def f(x, gamma, beta, eps, out_dtype, out=None):
            return emu.layernorm(x, gamma, beta, 1e-6 if eps == 1e-5 else eps, out_dtype, out)
        return ops, "layernorm", f
    if name == "pos_before_norm":
        def f(tok, gamma, beta, pos, cls, B, P, eps):
            ntok = 0 if cls is None else 1
            moved = (tok.view(B, P, -1) + pos[ntok:][None]).reshape(B * P, -1)
            return po.pvt_embed_norm(moved, gamma, beta, torch.zeros_like(pos), cls, B, P, eps)
        return pvt_ops, "pvt_embed_norm", f
    if name == "cls_without_pos":
        def f(tok, gamma, beta, pos, cls, B, P, eps):
            y = po.pvt_embed_norm(tok, gamma, beta, pos, cls, B, P, eps)
            if cls is not None:
                y.view(B, P + 1, -1)[:, 0] = cls
            return y
        return pvt_ops, "pvt_embed_norm", f
    if name == "sr_taps_transposed":
        def f(x, ks, stride, padding, out_dtype, groups=1, pre=None):
            cols, Ho, Wo = emu.im2col(x, ks, stride, padding, out_dtype, groups, pre)
            if pre is None:   # the sr convolutions (the patch embeddings at stages 1 .. 3 too)
                C = x.shape[-1]
                cols = cols[:, :ks * ks * C].view(-1, ks, ks, C).transpose(1, 2).reshape(cols.shape[0], -1)
            return cols.contiguous(), Ho, Wo
        return ops, "im2col", f
    if name == "sr_keeps_remainder":
        def f(x, ks, stride, padding, out_dtype, groups=1, pre=None):
            if pre is None and ks > 2 and (x.shape[1] % ks or x.shape[2] % ks):
                padding = "same"   # a partial last window, zero-filled, instead of VALID's floor
            return emu.im2col(x, ks, stride, padding, out_dtype, groups, pre)
        return ops, "im2col", f
    if name == "features_before_final_norm":
        def f(x, gamma, beta, eps, out_dtype, out=None):
            if eps == 1e-6 and out_dtype == torch.float32:   # only the final norm stores fp32 at eps 1e-6
                return x.to(out_dtype).clone()
            return emu.layernorm(x, gamma, beta, eps, out_dtype, out)
        return ops, "layernorm", f
    raise KeyError(name)


@pytest.mark.parametrize("defect,kind,precision", [
    ("k_v_swapped", "plain", "bf16"), ("kv_split_h_2_dh", "plain", "fp32"),
    ("embed_norm_eps_1e-6", "plain", "fp32"), ("sr_norm_eps_1e-6", "odd", "fp32"),
    ("pos_before_norm", "plain", "fp32"), ("cls_without_pos", "noclass", "fp32"),
    ("sr_taps_transposed", "plain", "fp32"), ("sr_keeps_remainder", "odd", "fp32"),
    ("features_before_final_norm", "noclass", "fp32")])
def test_seeded_defects_are_rejected(pvt, cpu_engine, defect, kind, precision):
    """Each seeded defect makes the harness fail, and the failing rows name the launcher that carries it."""
    from pvt_oracle import emulated_pvt_ops, shadowed_pvt_ops

    m, cfg, w, x = _small(pvt, kind, precision, batch=3)
    module, op, bad = _defect(defect)
    with emulated_pvt_ops(torch.float32):
        setattr(module, op, bad)
        with shadowed_pvt_ops() as census:
            m(x)
    fails = census.failures()
    assert fails and {r["op"] for r in fails} == {op}, census.table()
