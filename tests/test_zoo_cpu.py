"""CPU rehearsal of the zoo sweep (tests/test_zoo_gpu.py): its case list, its launch signatures, and its machinery --
recording, dedupe, the choice of shadow harness -- on small overrides of one registration per family, with the float32
emulation (``emulate_bf16.emulated_ops(torch.float32)`` and the Mixer / SAM statements) standing in for the kernels, as
tests/test_op_shadow_cpu.py does for the shadow harness itself.  Every launch of the stand-in must pass, and defects
seeded at shapes that only zoo registrations produce must be rejected, naming the launcher.
"""
from contextlib import ExitStack, contextmanager
from copy import deepcopy

import pytest
import torch

from test_zoo_gpu import (CASES, NO_TF32, NO_UINT8, PRECISIONS, Sweep, batch_of, check_registration, harness_launchers,
                          module_of, recording, registered_zoo)

FAMILIES = ("vit", "swin", "convnext", "efficientnet", "resnet", "mlp_mixer", "sam")


# ------------------------------------------------------------------------------------------------------ case list
def test_case_list_is_every_registration_times_its_accepted_precisions():
    import tfimm

    expected, refused = [], set()
    with registered_zoo() as registry:
        names = [n for n in tfimm.list_models() if module_of(registry, n) in FAMILIES]
        for n in names:
            module = module_of(registry, n)
            for p in PRECISIONS:
                try:
                    tfimm.create_model(n, precision=p, device="meta")
                except ValueError:
                    refused.add((module, p))
                    continue
                expected.append((n, module, p))
    assert CASES == expected
    assert refused == {(m, "tf32") for m in NO_TF32}
    assert len(names) == 215 and len(CASES) == 3 * 215 - 29 == 616


def test_raw_pixels_are_skipped_exactly_where_the_preprocessing_divides_by_zero():
    import tfimm

    with registered_zoo() as registry:
        zero_std = {n for n in tfimm.list_models() if 0.0 in registry.model_config(n).std}
    assert set(NO_UINT8) == zero_std


def test_registry_is_restored():
    from tfimm.models import registry

    before = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    with registered_zoo():
        assert {"mlp_mixer", "sam"} <= set(registry._by_module)
        assert len(registry._classes) == len(before[0]) + 29
    assert registry._classes == before[0] and registry._configs == before[1]
    assert registry._by_module == before[2] and registry._with_url == before[3]
    assert not {"mlp_mixer", "sam"} & set(registry._by_module)


def test_every_launcher_is_recorded():
    """The recorded launchers are every launcher of ops / mixer_ops / sam_ops (shape predicates and host helpers
    aside), so no launch escapes its signature."""
    from tfimm.backend import mixer_ops, ops, sam_ops

    def public(mod, skip):
        return {n for n in dir(mod) if not n.startswith("_") and callable(getattr(mod, n))
                and getattr(getattr(mod, n), "__module__", "") == mod.__name__ and n not in skip}

    want = (public(ops, ("act_code", "same_pad", "conv_geometry", "attention_bf16_supported", "mlp_fused_supported"))
            | public(mixer_ops, ("glu_interleave",)) | public(sam_ops, ("relpos_attention_bf16_supported",)))
    assert harness_launchers() == want


# ------------------------------------------------------------------------------------------------------ signatures
def _gemm_signature(a, w, tf32=False, **kw):
    from oracle import emulate_bf16
    from tfimm.backend import lib, ops

    log = []
    token = lib.tf32_mode.set(tf32)
    try:
        with emulate_bf16.emulated_ops(torch.float32), recording(log):
            ops.gemm(a, w, **kw)
    finally:
        lib.tf32_mode.reset(token)
    assert len(log) == 1
    return log[0]


def _operands(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(16, 40, generator=g), torch.randn(24, 32, generator=g), torch.randn(16, 24, generator=g)


VARIANTS = {
    "row_stride": lambda a, w, r: dict(a=a[:, :32].contiguous(), w=w, residual=r),
    "alignment": lambda a, w, r: dict(a=a[:, 2:34], w=w, residual=r),                     # 8 bytes off
    "dtype": lambda a, w, r: dict(a=a[:, :32].bfloat16(), w=w.bfloat16(), residual=r),
    "flag": lambda a, w, r: dict(a=a[:, :32], w=w, residual=r, act_after_residual=True),
    "tf32_mode": lambda a, w, r: dict(a=a[:, :32], w=w, residual=r, tf32=True),
}


def test_signature_ignores_values():
    (a, w, r), (a2, w2, r2) = _operands(0), _operands(1)
    assert not torch.equal(a, a2)
    assert _gemm_signature(a[:, :32], w, residual=r) == _gemm_signature(a2[:, :32], w2, residual=r2)


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_signature_separates(variant):
    a, w, r = _operands(0)
    assert a.data_ptr() % 16 == 0
    base = _gemm_signature(a[:, :32], w, residual=r)
    assert _gemm_signature(**VARIANTS[variant](a, w, r)) != base


# ------------------------------------------------------------------------------------------------------- rehearsal
@pytest.fixture(scope="module")
def cpu_zoo():
    """The registry of the sweep, and the engine's host orchestration on CPU tensors (``cpu_engine`` of
    tests/test_orchestration_cpu.py)."""
    from tfimm.models.model import Model

    def ensure_plan(self):
        if self._plan is None:
            self._plan = self._compile()
        return self._plan

    with registered_zoo() as registry, pytest.MonkeyPatch.context() as mp:
        mp.setattr(Model, "_ensure_plan", ensure_plan)
        yield registry


@contextmanager
def standin(module, precision):
    """The float32 emulation of every launcher a family uses, in place of the kernels (TF32 rounding in tf32)."""
    from mixer_oracle import emulated_mixer_ops
    from oracle import emulate_bf16
    from sam_oracle import emulated_sam_ops
    from tf32_oracle import tf32_oracle

    with ExitStack() as stack:
        if precision == "tf32":
            stack.enter_context(tf32_oracle())
        emulated = {"mlp_mixer": emulated_mixer_ops, "sam": emulated_sam_ops}.get(module, emulate_bf16.emulated_ops)
        stack.enter_context(emulated(torch.float32))
        yield


# one registration per family, shrunk
REHEARSAL = {
    "deit_tiny_distilled_patch16_224": {"nb_blocks": 2, "input_size": (64, 64)},
    "swin_tiny_patch4_window7_224": {"input_size": (56, 56), "nb_blocks": (2, 2), "nb_heads": (3, 6)},
    "convnext_tiny": {"input_size": (64, 96), "nb_blocks": (1, 1, 1, 1)},
    "efficientnet_b0": {"input_size": (64, 64)},
    "seresnext26d_32x4d": {"input_size": (64, 64)},
    "gmixer_12_224": {"input_size": (20, 24), "patch_size": 4, "embed_dim": 16, "nb_blocks": 2, "nb_classes": 5},
    "sam_vit_b": {"input_size": (32, 32), "encoder_patch_size": 4, "encoder_embed_dim": 160, "encoder_nb_heads": 2,
                  "encoder_nb_blocks": 2, "encoder_global_attn_indices": (1,), "encoder_window_size": 3,
                  "embed_dim": 64},
}


def _small(registry, name, precision, overrides):
    import importlib

    import tfimm
    from oracle import params

    module = module_of(registry, name)
    model = tfimm.create_model(name, precision=precision, device="cpu", **overrides)
    omod = importlib.import_module(f"oracle.{module}")
    model.load_weights_dict(params.random_params(omod.param_shapes(model.cfg), seed=3))
    return model, module


def _run(sweep, registry, name, precision, overrides, mutate=None):
    from oracle import params
    from tfimm.backend import ops

    model, module = _small(registry, name, precision, overrides)
    cfg = model.cfg
    x = params.test_images(batch_of(cfg), *cfg.input_size, cfg.in_channels)
    with standin(module, precision):
        if mutate is not None:
            mutate(ops)
        check_registration(sweep, name, module, precision, model, x)
    return module


@pytest.fixture(scope="module")
def rehearsal(cpu_zoo):
    """One sweep over REHEARSAL x the precisions of each family: {(name, precision): None or the exception}."""
    sweep, out = Sweep(), {}
    for name, overrides in REHEARSAL.items():
        for precision in PRECISIONS:
            if precision == "tf32" and module_of(cpu_zoo, name) in NO_TF32:
                continue
            try:
                _run(sweep, cpu_zoo, name, precision, overrides)
                out[(name, precision)] = None
            except Exception as e:   # reported by the test of that case
                out[(name, precision)] = e
    return sweep, out


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(REHEARSAL))
def test_float32_standin_passes_the_sweep(rehearsal, cpu_zoo, name, precision):
    sweep, out = rehearsal
    if precision == "tf32" and module_of(cpu_zoo, name) in NO_TF32:
        assert (name, precision) not in out
        return
    if out[(name, precision)] is not None:
        raise out[(name, precision)]


def test_sweep_reaches_each_family_and_dedupes(rehearsal, cpu_zoo):
    sweep, _ = rehearsal
    assert {"token_gemm", "gemm_glu", "relpos_attention", "dwconv_ln", "attention_cls", "window_attention_tc",
            "gemm_gated", "grouped_conv", "im2col", "patchify"} <= sweep.reached
    # the same registration again: every signature is checked already, nothing is shadowed
    passes, shadowed = sweep.passes, sweep.shadowed
    name = "deit_tiny_distilled_patch16_224"
    _run(sweep, cpu_zoo, name, "bf16", REHEARSAL[name])
    assert sweep.passes == passes + 2 and sweep.shadowed == shadowed
    # another class count is a new head GEMM signature: the fp32-image pass is shadowed again
    _run(sweep, cpu_zoo, name, "bf16", dict(REHEARSAL[name], nb_classes=7))
    assert sweep.shadowed == shadowed + 1


# --------------------------------------------------------------------------------- defects only the zoo reaches
def _gemm_last_column_lost(ops):
    f = ops.gemm

    def gemm(*a, **k):
        out = f(*a, **k)
        if out.shape[1] % 8:
            out[:, -1] = 0
        return out
    ops.gemm = gemm


def _attention_scale_of_head_dim_64(ops):
    f = ops.attention

    def attention(qkv, B, N, H, dh, scale, *a, **k):
        return f(qkv, B, N, H, dh, 64 ** -0.5 if dh == 80 else scale, *a, **k)
    ops.attention = attention


def _dwconv_ln_beta_lost_on_wide_rows(ops):
    f = ops.dwconv_ln

    def dwconv_ln(x, wgt, bias, gamma, beta, eps, out_dtype):
        if x.shape[-1] >= 2048:
            beta = beta.clone()
            beta[-64:] = 0
        return f(x, wgt, bias, gamma, beta, eps, out_dtype)
    ops.dwconv_ln = dwconv_ln


DEFECTS = [
    # vit_*_in21k heads: 21843 columns, the logits a padded-stride view
    ("gemm_last_column_when_n_is_not_a_multiple_of_8", "vit_tiny_patch16_224",
     {"nb_blocks": 1, "input_size": (32, 32), "nb_classes": 21843}, "gemm", _gemm_last_column_lost),
    # vit_huge_patch14_224_in21k: head dim 80
    ("attention_scaled_for_head_dim_64_at_80", "vit_tiny_patch16_224",
     {"nb_blocks": 1, "input_size": (32, 32), "embed_dim": 160, "nb_heads": 2}, "attention",
     _attention_scale_of_head_dim_64),
    # convnext_xlarge_*: stage 3 at C = 2048
    ("dwconv_ln_last_channels_lose_beta_at_2048", "convnext_tiny",
     {"input_size": (64, 64), "nb_blocks": (1, 1, 1, 1), "embed_dim": (16, 32, 64, 2048)}, "dwconv_ln",
     _dwconv_ln_beta_lost_on_wide_rows),
]


@pytest.mark.parametrize("defect,name,overrides,op,mutate", DEFECTS, ids=[d[0] for d in DEFECTS])
def test_seeded_defect_at_a_zoo_shape_is_rejected(cpu_zoo, defect, name, overrides, op, mutate, capsys):
    sweep = Sweep()
    with pytest.raises(AssertionError, match=rf"FAIL {op} "):
        _run(sweep, cpu_zoo, name, "bf16", overrides, mutate=mutate)
    failed = {line.split()[1] for line in capsys.readouterr().out.splitlines() if line.startswith("FAIL ")}
    assert failed == {op}
    # the same registration without the defect passes
    _run(Sweep(), cpu_zoo, name, "bf16", overrides)
