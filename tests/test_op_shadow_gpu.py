"""Every kernel launch of the benchmark models against its float64 statement, op by op (oracle/shadow.py).

The model-level tests compare logits, where one flipped bf16 rounding spreads through the layers and the floor is
~2-3e-3; a kernel that is wrong only at one tile, one channel tail or one head count can hide below it.  Here each
launch of an eager forward pass is checked where it happens, on exactly the inputs the engine produced, against the
bound ``shadow.check`` derives for it -- at the shapes and dispatch branches the models take: the small configurations
of tests/test_parity_budget_gpu.py (plus the 12 x 12 windows of swin_base_patch4_window12_384) in both precisions, with
fp32 images and raw uint8 pixels, one ``return_features=True`` pass per family, and the benchmark configurations at
their benchmark batch.  ``-s`` prints the census: op, call site, launch index, worst error / bound, flip %, arguments.
"""
import pytest
import torch

from test_parity_budget_gpu import SMALL, _model

pytestmark = pytest.mark.gpu

SMALL_CASES = SMALL + [("swin", "swin_base_patch4_window12_384", {})]   # window_attention: 12 x 12 windows, 4-32 heads

# EfficientNet-B4 runs at 380 px.  Its largest launch -- the 1 x 1 expansion to 144 channels at 190 x 190 -- has a
# 5.2 M-element output per image, and the float64 reference of that one op (the product, the activation's temporaries,
# the arithmetic bound, the comparison) holds ~10 tensors of that size: ~0.4 GB per image.  Batch 32 keeps it near
# 13 GB (peak allocated 12.7 GiB, measured on an H100 80GB HBM3 at 700 W), under ~16 GB on a card that others share;
# the other configurations run at the benchmark's batch of 256.  The whole file took 51 s there.
EFFICIENTNET_B4_BATCH = 32
BENCH = [
    ("vit", "vit_base_patch16_224", 256),
    ("convnext", "convnext_base", 256),
    ("swin", "swin_base_patch4_window7_224", 256),
    ("resnet", "resnet50", 256),
    ("efficientnet", "efficientnet_b4", EFFICIENTNET_B4_BATCH),
]

_REACHED = set()


def _shadowed(model, x, title, return_features=False):
    from oracle import shadow

    torch.cuda.reset_peak_memory_stats()
    with shadow.shadowed_ops() as census:
        model(x.cuda(), return_features=return_features)
    torch.cuda.synchronize()
    print(f"\n=== {title}: {census.launches} launches, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB\n"
          + census.table())
    _REACHED.update(census.ops())
    return census


def _inputs(model, batch):
    from oracle import params

    x = params.test_images(batch, *model.cfg.input_size, model.cfg.in_channels)
    runs = [("fp32 images", x)]
    if model.accepts_uint8:
        runs.append(("uint8 pixels", (x * 255).round().to(torch.uint8)))
    return runs


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("family,name,overrides", SMALL_CASES, ids=[c[1] for c in SMALL_CASES])
def test_small_config_every_launch_within_its_bound(family, name, overrides, precision):
    model, _, _ = _model(name, family, precision, overrides)
    batch = 1 if name == "swin_base_patch4_window12_384" else 2
    for what, x in _inputs(model, batch):
        _shadowed(model, x, f"{name} {precision} {what}").assert_ok()


RETURN_FEATURES = [("vit", "vit_tiny_patch16_224", {"nb_blocks": 4}),      # fp32 attention writing probs
                   ("swin", "swin_tiny_patch4_window7_224", SMALL[2][2]),
                   ("convnext", "convnext_tiny", SMALL[3][2]),
                   ("efficientnet", "efficientnet_b0", SMALL[4][2]),
                   ("resnet", "resnet50", SMALL[6][2])]


@pytest.mark.parametrize("family,name,overrides", RETURN_FEATURES, ids=[c[1] for c in RETURN_FEATURES])
def test_return_features_every_launch_within_its_bound(family, name, overrides):
    model, _, _ = _model(name, family, "bf16", overrides)
    _, x = _inputs(model, 2)[0]
    _shadowed(model, x, f"{name} bf16 return_features", return_features=True).assert_ok()


@pytest.mark.parametrize("family,name,batch", BENCH, ids=[c[1] for c in BENCH])
def test_benchmark_config_at_its_batch_every_launch_within_its_bound(family, name, batch):
    """bf16, eager, at the batch bench.py runs (tile widths, wave counts and grid sizes of the benchmark), fed fp32
    images and -- as bench.py's end-to-end pass -- raw uint8 pixels."""
    model, _, _ = _model(name, family, "bf16", seed=29)
    for what, x in _inputs(model, batch):
        census = _shadowed(model, x, f"{name} bf16 batch {batch} {what}")
        census.assert_ok()
        del census
        torch.cuda.empty_cache()


def test_census_reaches_every_launcher():
    """Every shadowed launcher of tfimm.backend.ops was reached by the configurations above (run with the module)."""
    from oracle import shadow

    if not _REACHED:
        pytest.skip("runs after the shadowed configurations of this module")
    assert set(shadow.SHADOWED) - _REACHED == set()
