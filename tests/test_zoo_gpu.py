"""Every registered model, in every precision it accepts, run on the H100 with each launch checked against its float64
statement where the suite has not checked that launch yet.

The kernel tests pick their shapes from hand-made lists and the op-by-op shadow tests (tests/test_op_shadow_gpu.py,
tests/test_tf32_gpu.py, tests/test_mixer_gpu.py, tests/test_sam_gpu.py) run a dozen configurations; the registry has
215 models.  A kernel that is wrong only at a shape the zoo produces -- C = 2048 in ConvNeXt-XL's LayerNorm, head dim 80
in ViT-H, a 21843-column head, 384 channels per ResNeXt group, 12 x 12 Swin windows at 48 heads -- or a registration
that raises in one of its precisions passes all of them.  Here every registration x precision (616 cases; MLP-Mixer and
SAM refuse tf32) builds with random weights (``oracle.params.random_params``: nonzero BN statistics, LN affine terms and
biases), runs on test images at batch 3 (1 above 320 px: an odd batch, so tiles span images and the last one is partial)
and, if it takes them, on raw uint8 pixels.  Each output must have its shape and be finite; in fp32 the stem's output for
uint8 pixels must equal its output for ``create_preprocessing(name)`` of them (the ``_ap`` / ``_ns`` / ``tv_`` variants
differ only in these statistics).

Every launch of ``tfimm.backend.ops`` / ``mixer_ops`` / ``sam_ops`` is recorded by its signature: launcher, tf32 mode,
and for each argument its dtype, shape, strides and ``data_ptr() % 16`` if it is a tensor, its value otherwise.  A pass
with a signature no earlier case of the session has had checked is run again under its family's shadow harness
(oracle/shadow.py with tests/mixer_oracle.py, tests/sam_oracle.py, and tests/tf32_oracle.py for tf32), which checks every
launch of that pass within the bounds those tests already use.  So each distinct launch of the zoo is checked at least
once, and the registrations that only change weights or preprocessing cost one plain forward.  ``-k <name>`` runs
a case alone, shadowed.  ``-s`` prints, per pass, its launch count, its new signatures and whether it was shadowed,
with the census rows of the new launches; the last test prints the signatures per launcher, the shadowed passes, the
peak allocated memory and the wall time.

Measured on an H100 80GB HBM3 (400 W power limit): the whole file in 16 min (958 s; 1232 passes, 463 of them shadowed,
7664 distinct signatures), peak allocated memory 10.6 GiB.
"""
import importlib
import inspect
import sys
import time
from collections import Counter
from contextlib import contextmanager
from copy import deepcopy

import pytest
import torch

pytestmark = pytest.mark.gpu

# Registered on import only (as in the reference); the fixture below restores the registry afterwards, because
# tests/test_api_cpu.py pins the default list of models.
OPTIONAL_MODULES = ("tfimm.architectures.mlp_mixer", "tfimm.architectures.segment_anything.sam")
PRECISIONS = ("bf16", "tf32", "fp32")
# Registry modules whose models refuse precision="tf32" with a ValueError (pinned by tests/test_zoo_cpu.py).
NO_TF32 = {
    "mlp_mixer": "TF32 wgmma has no transposed operand form for the token-mixing GEMM",
    "sam": "the relative-position attention has no TF32 kernel",
}
# Registrations whose preprocessing the reference itself cannot evaluate, so they run on float images only (pinned by
# tests/test_zoo_cpu.py): their registered std is (0, 0, 0), as in the reference, and create_preprocessing divides by it.
NO_UINT8 = {
    "vit_base_patch16_224_miil": "registered std (0, 0, 0): create_preprocessing divides by zero",
    "vit_base_patch16_224_miil_in21k": "registered std (0, 0, 0): create_preprocessing divides by zero",
}
SEED = 17
MAX_INPUT_FOR_BATCH_3 = 320
PEAK_LIMIT = 16 * 10 ** 9          # bytes: the share of a card that other jobs use too


@contextmanager
def registered_zoo():
    """The registry with the optional families registered; restored on exit."""
    from tfimm.models import registry

    saved = (dict(registry._classes), dict(registry._configs), deepcopy(registry._by_module), set(registry._with_url))
    try:
        for name in OPTIONAL_MODULES:
            if name in sys.modules:
                importlib.reload(sys.modules[name])
            else:
                importlib.import_module(name)
        yield registry
    finally:
        registry._classes.clear(), registry._classes.update(saved[0])
        registry._configs.clear(), registry._configs.update(saved[1])
        registry._by_module.clear(), registry._by_module.update(saved[2])
        registry._with_url.clear(), registry._with_url.update(saved[3])


def module_of(registry, name):
    """Registry module of a model ("vit", ..., "mlp_mixer", "sam"): also the name of its oracle module."""
    return next(stem for stem, names in registry._by_module.items() if name in names)


def zoo_cases():
    """[(name, module, precision)]: every registered model x every precision it accepts, in list_models() order."""
    import tfimm

    with registered_zoo() as registry:
        return [(n, module_of(registry, n), p) for n in tfimm.list_models() for p in PRECISIONS
                if not (p == "tf32" and module_of(registry, n) in NO_TF32)]


CASES = zoo_cases()


# ------------------------------------------------------------------------------------------------ launch signatures
def _statements():
    """{launcher: its float64 statement}, the functions whose parameters name the launchers' arguments."""
    import mixer_oracle
    import sam_oracle
    from oracle import emulate_bf16, shadow

    out = {n: getattr(emulate_bf16, n) for n in shadow.SHADOWED}
    out.update({n: f for n, (f, _) in mixer_oracle._MIXER.items()})
    out["relpos_attention"] = sam_oracle.relpos_attention
    return out


def launchers():
    """[(module, name)] of every launcher the harnesses check."""
    import mixer_oracle
    from tfimm.backend import mixer_ops, ops, sam_ops

    mods = {n: mixer_ops for n in mixer_oracle._MIXER}
    mods["relpos_attention"] = sam_ops
    return [(mods.get(n, ops), n) for n in _statements()]


def _arg(v):
    if torch.is_tensor(v):
        return (v.dtype, tuple(v.shape), v.stride(), v.data_ptr() % 16)
    if isinstance(v, (tuple, list)):
        return tuple(_arg(e) for e in v)
    return v


def signature(name, arguments):
    """What selects a kernel's code path: the launcher, the tf32 mode, the tensors' dtype / shape / strides / 16-byte
    alignment and every other argument's value -- not the tensors' contents."""
    from tfimm.backend import lib

    return (name, bool(lib.tf32_mode.get())) + tuple((k, _arg(v)) for k, v in arguments.items())


@contextmanager
def recording(log):
    """Appends the signature of every launch to ``log``; whatever each launcher is on entry still runs."""
    statements = _statements()
    saved = [(mod, n, getattr(mod, n)) for mod, n in launchers()]

    def wrap(n, f):
        sig = inspect.signature(statements[n])

        def launcher(*a, **k):
            b = sig.bind(*a, **k)
            b.apply_defaults()
            log.append(signature(n, b.arguments))
            return f(*a, **k)
        return launcher

    for mod, n, f in saved:
        setattr(mod, n, wrap(n, f))
    try:
        yield log
    finally:
        for mod, n, f in saved:
            setattr(mod, n, f)


def harness(module, precision):
    """The shadow harness of a family and precision."""
    from oracle import shadow

    if module == "mlp_mixer":
        from mixer_oracle import shadowed_mixer_ops
        return shadowed_mixer_ops()
    if module == "sam":
        from sam_oracle import shadowed_sam_ops
        return shadowed_sam_ops()
    if precision == "tf32":
        from test_tf32_gpu import _shadowed_tf32
        return _shadowed_tf32()
    return shadow.shadowed_ops()


def harness_launchers():
    """Every launcher some harness checks: shadow.SHADOWED, the Mixer and the SAM launchers."""
    return {n for _, n in launchers()}


class Sweep:
    """Signatures seen and checked over a session, and the census of what was shadowed."""

    def __init__(self):
        self.seen, self.checked, self.reached = set(), set(), set()
        self.passes = self.shadowed = 0
        self.cases = set()

    def run(self, title, forward, module, precision):
        """One plain pass ``forward()`` with its launches recorded, then -- if it launched a signature not yet checked
        -- the same pass under the family's shadow harness, whose census must be clean.  Returns the plain output."""
        log = []
        with recording(log):
            y = forward()
        self.passes += 1
        self.seen.update(log)
        new = set(log) - self.checked
        print(f"\n{title}: {len(log)} launches, {len(set(log))} signatures, {len(new)} new, "
              f"{'shadowed' if new else 'not shadowed'}")
        if new:
            with harness(module, precision) as census:
                forward()
            self.shadowed += 1
            self.reached |= census.ops()
            fresh = {i for i, s in enumerate(log) if s in new}
            rows = [r for r in census.rows if r["index"] in fresh and r["ok"]]
            if rows:
                print("\n".join(census._fmt(r) for r in rows))
            bad = census.failures()
            if bad:
                print("\n".join(census._fmt(r) for r in bad))
            census.assert_ok()
            self.checked.update(log)
        return y


def nerr(a, b):
    a, b = a.double(), b.double()
    return (a - b).abs().max().item() / (b.abs().max().item() + 1e-12)


def batch_of(cfg):
    return 3 if max(cfg.input_size) <= MAX_INPUT_FOR_BATCH_3 else 1


def expected_shape(model, module, batch):
    c = model.cfg
    if module == "sam":
        return (batch, c.input_size[0] // c.encoder_patch_size, c.input_size[1] // c.encoder_patch_size, c.embed_dim)
    if getattr(c, "distilled", False):
        return (batch, 2, c.nb_classes)      # DeiT distilled: the class and the distillation head
    return (batch, c.nb_classes)


def check_registration(sweep, name, module, precision, model, x):
    """Everything one case checks, on ``model`` (the registration; on CPU, a small override of it) fed images ``x``."""
    import tfimm

    target = model.image_encoder if module == "sam" else model
    runs = [("fp32 images", x)]
    if target.accepts_uint8 and name not in NO_UINT8:
        runs.append(("uint8 pixels", (x * 255).round().to(torch.uint8)))
    outs = {}
    for what, inp in runs:
        y = sweep.run(f"{name}-{precision} {what}", lambda: target(inp), module, precision)
        want = expected_shape(model, module, x.shape[0])
        assert tuple(y.shape) == want, (what, tuple(y.shape), want)
        assert bool(torch.isfinite(y).all()), f"{what}: non-finite outputs"
        outs[what] = y
    if precision == "fp32" and len(runs) == 2:
        # Compared where the statistics enter, at the stem: deeper, random-weight networks amplify the one-ulp
        # difference of the two pixel paths (the logits of resnetrs420 move by 0.19, of gmixer_24_224 by 3e-3).
        px = runs[1][1]
        op_u8, fused = first_launch(lambda: target(px))
        op_f, ref = first_launch(lambda: target(tfimm.create_preprocessing(name)(px)))
        assert op_u8 == op_f and fused.shape == ref.shape, (op_u8, op_f, fused.shape, ref.shape)
        err = nerr(fused, ref)
        assert err <= 1e-5, f"{op_u8} of uint8 pixels vs of create_preprocessing({name!r}): normalised error {err:.3e}"
    sweep.cases.add((name, precision))


def first_launch(forward):
    """(launcher, output) of the first launch of ``forward()``."""
    first = []
    saved = [(mod, n, getattr(mod, n)) for mod, n in launchers()]

    def wrap(n, f):
        def launcher(*a, **k):
            out = f(*a, **k)
            if not first:
                first.append((n, (out[0] if isinstance(out, tuple) else out).clone()))
            return out
        return launcher

    for mod, n, f in saved:
        setattr(mod, n, wrap(n, f))
    try:
        forward()
    finally:
        for mod, n, f in saved:
            setattr(mod, n, f)
    return first[0]


# ------------------------------------------------------------------------------------------------------ the sweep
_WEIGHTS = {}


def _weights(registry, name, module):
    """Random weights of a registration, drawn once and reused by its precisions (cases run name by name)."""
    from oracle import params

    if name not in _WEIGHTS:
        _WEIGHTS.clear()
        omod = importlib.import_module(f"oracle.{module}")
        _WEIGHTS[name] = params.random_params(omod.param_shapes(registry.model_config(name)), seed=SEED)
    return _WEIGHTS[name]


@pytest.fixture(scope="module")
def zoo():
    with registered_zoo() as registry:
        torch.cuda.reset_peak_memory_stats()
        sweep = Sweep()
        sweep.registry, sweep.t0 = registry, time.time()
        yield sweep
    _WEIGHTS.clear()


@pytest.mark.parametrize("name,module,precision", CASES, ids=[f"{n}-{p}" for n, _, p in CASES])
def test_registration(zoo, name, module, precision):
    import tfimm
    from oracle import params

    torch.cuda.empty_cache()
    w = _weights(zoo.registry, name, module)
    model = tfimm.create_model(name, precision=precision, device="cpu")   # built on the host, moved once
    model.load_weights_dict(w)
    model.to("cuda")
    cfg = model.cfg
    x = params.test_images(batch_of(cfg), *cfg.input_size, cfg.in_channels).cuda()
    check_registration(zoo, name, module, precision, model, x)


def test_zoo_summary(zoo):
    """Runs last: what the sweep reached, its peak memory and its wall time."""
    peak = torch.cuda.max_memory_allocated()
    per = Counter(s[0] for s in zoo.seen)
    print(f"\n=== zoo sweep: {len(zoo.cases)} cases, {zoo.passes} passes, {zoo.shadowed} shadowed, "
          f"{len(zoo.seen)} distinct signatures, peak allocated {peak / 2 ** 30:.2f} GiB, "
          f"wall time {(time.time() - zoo.t0) / 60:.1f} min")
    for n, k in sorted(per.items()):
        print(f"  {n:<22} {k:6d} signatures")
    assert peak <= PEAK_LIMIT, f"peak allocated {peak / 1e9:.2f} GB"
    if len(zoo.cases) < len(CASES):
        pytest.skip(f"{len(zoo.cases)} of {len(CASES)} cases ran; the launcher coverage needs all of them")
    assert harness_launchers() - zoo.reached == set()
