"""precision="tf32" on CPU: the TF32 rounding against an independent reference, the precision switch, and a rehearsal of
every tf32 forward of tests/test_orchestration_cpu.py through the op-by-op shadow harness (tests/tf32_oracle.py on
oracle/shadow.py), with the emulation evaluated in float32 standing in for the kernels -- as tests/test_op_shadow_cpu.py
does for bf16 and fp32.  tests/test_tf32_gpu.py runs the real kernels.
"""
import numpy as np
import pytest
import torch

from test_op_shadow_cpu import _images, cpu_models  # noqa: F401  (fixture)
from test_orchestration_cpu import CASES, _build
from tf32_oracle import tf32_oracle


def _ref_round_tf32(x):
    """Nearest TF32 value, ties away from zero, computed in float64 arithmetic (no bit manipulation): the spacing of
    TF32 numbers at |x| is 2^(e - 10) for |x| in [2^e, 2^(e+1)), 2^-136 below the smallest normal; results of 2^128 or
    more are infinite.  Non-finite values are returned as they are."""
    x = np.asarray(x, dtype=np.float32)
    out = x.copy()
    fin = np.isfinite(x)
    a = np.abs(x[fin].astype(np.float64))
    _, e = np.frexp(a)                                   # a = m 2^e, m in [0.5, 1): leading bit 2^(e-1)
    spacing = np.ldexp(1.0, np.maximum(e - 1, -126) - 10)
    r = np.floor(a / spacing + 0.5) * spacing            # exact: a / spacing < 2^12
    r = np.where(r >= 2.0 ** 128, np.inf, r)
    with np.errstate(over="ignore"):
        out[fin] = np.copysign(r, x[fin]).astype(np.float32)
    return out


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.uint32)


def _from_bits(u):
    return np.asarray(u, dtype=np.uint32).view(np.float32)


def _check_round(x):
    from tfimm.backend.lib import round_tf32

    got = round_tf32(torch.from_numpy(x.copy())).numpy()
    want = _ref_round_tf32(x)
    nan = np.isnan(x)
    assert np.array_equal(_bits(got)[nan], _bits(x)[nan])           # NaN payloads pass through
    mism = np.nonzero(_bits(got)[~nan] != _bits(want)[~nan])[0]
    assert mism.size == 0, [(hex(int(_bits(x)[~nan][i])), got[~nan][i], want[~nan][i]) for i in mism[:5]]
    assert np.all((_bits(got)[np.isfinite(got)] & 0x1FFF) == 0)
    return got


def test_round_tf32_ties_go_away_from_zero():
    half = 2.0 ** -11                     # half a TF32 ulp at 1
    x = np.array([1 + half, -(1 + half), 1 + 3 * half, -(1 + 3 * half), 1 + half / 2, 1 + 1.5 * half,
                  3 * 2.0 ** -140, -(3 * 2.0 ** -140)], dtype=np.float32)
    got = _check_round(x)
    assert got[0] == 1 + 2 * half and got[1] == -(1 + 2 * half)        # round-to-even would give 1 and -1
    assert got[2] == 1 + 4 * half and got[3] == -(1 + 4 * half)
    assert got[4] == 1 and got[5] == 1 + 2 * half


def test_round_tf32_at_the_top_of_the_range():
    top = 0x7F7FE000                      # largest TF32 value, (2 - 2^-10) 2^127
    u = np.array([top, top + 0xFFF, top + 0x1000, 0x7F7FFFFF, top - 0x2000 + 0x1000], dtype=np.uint32)
    u = np.concatenate([u, u | 0x80000000])
    got = _check_round(_from_bits(u))
    assert _bits(got[0]) == top and _bits(got[1]) == top
    assert np.isposinf(got[2]) and np.isposinf(got[3])                 # the tie and float max round up to inf
    assert _bits(got[4]) == top and np.isneginf(got[7]) and np.isneginf(got[8])


def test_round_tf32_keeps_representable_values_and_non_finite():
    rng = np.random.default_rng(0)
    u = rng.integers(0, 2 ** 32, size=4096, dtype=np.uint64).astype(np.uint32) & np.uint32(0xFFFFE000)
    x = _from_bits(u)
    got = _check_round(x)
    fin = np.isfinite(x)
    assert np.array_equal(_bits(got)[fin], u[fin])
    special = np.array([np.inf, -np.inf, np.nan, 0.0, -0.0], dtype=np.float32)
    special = np.concatenate([special, _from_bits(np.array([0x7FC01234, 0xFF800001], dtype=np.uint32))])
    got = _check_round(special)
    assert np.array_equal(_bits(got), _bits(special))


def test_round_tf32_random_values():
    rng = np.random.default_rng(1)
    u = rng.integers(0, 2 ** 32, size=200_000, dtype=np.uint64).astype(np.uint32)   # every binade, subnormals, NaN
    _check_round(_from_bits(u))
    _check_round(rng.standard_normal(100_000).astype(np.float32))


def test_tf32_precision_is_accepted_and_unknown_ones_are_not():
    import tfimm

    model = tfimm.create_model("vit_tiny_patch16_224", precision="tf32", device="cpu", nb_blocks=1)
    assert model.precision == "tf32" and model.act_dtype == torch.float32
    with pytest.raises(ValueError, match="precision"):
        tfimm.create_model("vit_tiny_patch16_224", precision="fp16", device="cpu", nb_blocks=1)


# --------------------------------------------------------------------------------------------- shadow rehearsal
def _shadowed_tf32_forward(model, x, return_features=False):
    """One forward with the float32 emulation standing in for the kernels; records the weight operands of the
    contractions as the kernels receive them."""
    from oracle import emulate_bf16, shadow
    from tfimm.backend import ops

    weights = []

    def record(name):
        f = getattr(ops, name)

        def launcher(*a, **k):
            weights.append((name, a[1] if len(a) > 1 else k["w"]))
            return f(*a, **k)
        setattr(ops, name, launcher)

    with tf32_oracle(), emulate_bf16.emulated_ops(arithmetic=torch.float32):
        record("gemm")
        record("conv_gemm")
        with shadow.shadowed_ops() as census:
            model(x, return_features=return_features)
    return census, weights


@pytest.fixture(scope="module")
def tf32_rehearsal(cpu_models):  # noqa: F811
    out = {}
    for family, name, overrides, batch in CASES:
        model, _, _ = _build(family, name, overrides, "tf32")
        runs = [_shadowed_tf32_forward(model, _images(model, batch))]
        if model.accepts_uint8:
            runs.append(_shadowed_tf32_forward(model, _images(model, batch, uint8=True)))
        runs.append(_shadowed_tf32_forward(model, _images(model, batch), return_features=True))
        out[name] = runs
    return out


@pytest.mark.parametrize("name", [c[1] for c in CASES])
def test_tf32_standin_passes_every_shadowed_launch(tf32_rehearsal, name):
    for census, weights in tf32_rehearsal[name]:
        assert census.rows
        census.assert_ok()
        assert all(r["cite"] is None for r in census.rows)
        assert weights and all(w.dtype == torch.float32 for _, w in weights)
        for op, w in weights:     # rounded once at plan time: the kernels do not round W
            assert not bool(((w.contiguous().view(torch.int32) & 0x1FFF) != 0).any()), op


def test_tf32_rehearsal_reaches_the_tf32_branches(tf32_rehearsal):
    ops = {r["op"] for runs in tf32_rehearsal.values() for census, _ in runs for r in census.rows}
    assert {"gemm", "conv_gemm", "attention"} <= ops
    assert not ops & {"mlp_fused", "gemm_gated", "window_attention", "window_attention_tc", "attention_cls"}


def test_tf32_mode_does_not_leak(cpu_models):  # noqa: F811
    """After a tf32 forward -- also one that raises -- bf16 and fp32 models dispatch as before."""
    from oracle import emulate_bf16
    from tfimm.backend import lib, ops

    family, name, overrides, batch = CASES[0]
    tf32, _, _ = _build(family, name, overrides, "tf32")
    x = _images(tf32, batch)
    seen = []
    with emulate_bf16.emulated_ops(arithmetic=torch.float32):
        f = ops.gemm

        def gemm(*a, **k):
            seen.append(lib.tf32_mode.get())
            return f(*a, **k)
        ops.gemm = gemm
        tf32(x)
        assert seen and all(seen)
        with pytest.raises(ValueError, match="Input size"):
            tf32(torch.zeros(1, 32, 32, 3))          # raises inside the forward, after the mode was set
        assert lib.tf32_mode.get() is False
        for precision in ("bf16", "fp32"):
            seen.clear()
            model, _, _ = _build(family, name, overrides, precision)
            model(x)
            assert seen and not any(seen)


@pytest.mark.parametrize("entry", ["call", "forward_features"])
@pytest.mark.parametrize("name", [c[1] for c in CASES])
def test_every_public_forward_entry_point_runs_in_tf32_mode(cpu_models, name, entry):  # noqa: F811
    """``model.call`` and ``model.forward_features`` called directly (not through ``model(x)``) dispatch the
    contractions of a tf32 model to the TF32 kernels, and leave the switch off afterwards."""
    from oracle import emulate_bf16
    from tfimm.backend import lib, ops

    family, _, overrides, batch = next(c for c in CASES if c[1] == name)
    model, _, _ = _build(family, name, overrides, "tf32")
    x = _images(model, batch)
    seen = []
    with tf32_oracle(), emulate_bf16.emulated_ops(arithmetic=torch.float32):
        for op in ("gemm", "conv_gemm", "attention"):
            f = getattr(ops, op)

            def launcher(*a, _f=f, _op=op, **k):
                seen.append((_op, lib.tf32_mode.get()))
                return _f(*a, **k)
            setattr(ops, op, launcher)
        getattr(model, entry)(x)
    assert seen and all(mode for _, mode in seen), seen
    assert lib.tf32_mode.get() is False
