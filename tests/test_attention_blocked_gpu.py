"""The tensor-core attention kernels against the float64 statement of their own algorithm, on the H100.

The ViT bf16 and TF32 kernels (csrc/attention.cu), the PiT kernel (csrc/pit.cu) and the Segment Anything relpos kernel
(csrc/relpos_attention.cu) run an online softmax over 64-key blocks and round P per block, relative to the running
maximum.  Each is held here, through the shadow harness, to ``emulate_bf16._softmax_pv`` in 64-key blocks within
``shadow._blocked_softmax_err`` (+ one bf16 ulp of the output), and to the flip criterion (under ``FLIP_LIMIT`` of the
outputs not correctly rounded):

* over the score cases of tests/test_attention_blocked_cpu.py (randn, logits near 80, the maximum on the last or on the
  first key for every query, all scores equal, all scores near -40) and lengths at the 16-key tile, 64-key block,
  query-chunk (128 / 224 rows) and resident-K/V (832) edges of each kernel;
* at a batch and head count of several waves of CTAs;
* called through the C entry point with the output in the middle of a canary buffer: nothing outside it is written
  and nothing in it is NaN; two runs are bit-identical, and image i of a batch equals image i run alone.

``-s`` prints the census of every case: worst error / bound and flip %.
"""
import sys
from contextlib import contextmanager
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
if str(HERE) not in sys.path:
    sys.path.insert(0, str(HERE))

import pit_oracle as po  # noqa: E402
import sam_oracle  # noqa: E402
from test_attention_blocked_cpu import KINDS, scored_qkv  # noqa: E402
from test_pit_gpu import LENGTHS as PIT_LENGTHS  # noqa: E402
from test_sam_gpu import GEOMETRY as RELPOS_GEOMETRY  # noqa: E402
from test_sam_gpu import _inputs as relpos_inputs  # noqa: E402
from tf32_oracle import tf32_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

# the 16-key tile and 64-key block edges; the 128-row (N <= 128) / 224-row (128 < N <= 784) / 128-row (N > 784) query
# chunks of the bf16 launcher and its resident-K/V limit of 832 keys
VIT_LENGTHS = [1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 197, 223, 224, 225, 448, 449, 577, 784, 785, 831, 832]
TF32_LENGTHS = VIT_LENGTHS + [1100]     # K / V stream through the TF32 kernel: no length limit


@contextmanager
def _tf32_mode():
    from tfimm.backend import lib

    token = lib.tf32_mode.set(True)
    try:
        yield
    finally:
        lib.tf32_mode.reset(token)


def _report(census, title):
    print(f"\n=== {title}\n" + census.table())
    census.assert_ok()
    assert census.rows and all(r["flips"] < 0.02 for r in census.rows)


def _bh(N):
    return (1, 2) if N > 1000 else (2, 4)


# ------------------------------------------------------------------------------------------- against the statement
@pytest.mark.parametrize("N", VIT_LENGTHS)
def test_vit_bf16_within_the_blocked_bound(N):
    from oracle import shadow
    from tfimm.backend import ops

    B, H = _bh(N)
    with shadow.shadowed_ops() as census:
        for kind in KINDS:
            ops.attention(scored_qkv(kind, B, N, H, 64, seed=N).cuda(), B, N, H, 64, 0.125)
    _report(census, f"attention bf16 N={N}: {KINDS}")
    assert census.ops() == {"attention"} and len(census.rows) == len(KINDS)


@pytest.mark.parametrize("N", TF32_LENGTHS)
def test_vit_tf32_within_the_blocked_bound(N):
    from oracle import shadow
    from tfimm.backend import ops

    B, H = _bh(N)
    calls = []
    call = ops._call

    def recording_call(name, *a, **k):
        calls.append(name)
        return call(name, *a, **k)

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "_call", recording_call)
        with tf32_oracle(), _tf32_mode(), shadow.shadowed_ops() as census:
            for kind in KINDS:
                ops.attention(scored_qkv(kind, B, N, H, 64, seed=N, dtype=torch.float32).cuda(), B, N, H, 64, 0.125)
    _report(census, f"attention tf32 N={N}: {KINDS}")
    assert set(calls) == {"tfimm_b200_attention_tf32"}


@pytest.mark.parametrize("T", PIT_LENGTHS)
@pytest.mark.parametrize("dh", [32, 48, 64])
def test_pit_within_the_blocked_bound(dh, T):
    from tfimm.backend import pit_ops

    B, H = _bh(T)
    with po.shadowed_pit_ops() as census:
        for kind in KINDS:
            pit_ops.pit_attention_bf16(scored_qkv(kind, B, T, H, dh, seed=T + dh).cuda(), B, T, H, dh, dh ** -0.5)
    _report(census, f"pit_attention_bf16 dh={dh} T={T}: {KINDS}")


@pytest.mark.parametrize("B,gh,gw,H,dh,window", RELPOS_GEOMETRY)
def test_relpos_within_the_blocked_bound(B, gh, gw, H, dh, window):
    """randn qkv, and the same scaled by 3: logits of std ~9, with the relative-position terms on top."""
    from tfimm.backend import sam_ops

    qkv, rh, rw, pad = relpos_inputs(B, gh, gw, H, dh, window, torch.bfloat16)
    with sam_oracle.shadowed_sam_ops() as census:
        for gain in (1.0, 3.0):
            sam_ops.relpos_attention((qkv.float() * gain).to(torch.bfloat16), B, gh, gw, H, dh, dh ** -0.5, rh, rw,
                                     window, pad)
    _report(census, f"relpos_attention B={B} grid={gh}x{gw} H={H} dh={dh} window={window}")
    assert census.ops() == {"relpos_attention"}


def test_several_waves_within_the_blocked_bound():
    """Grids of 1152 - 1344 CTAs (several waves of the 132 SMs at two CTAs each), randn and large logits."""
    from oracle import shadow
    from tfimm.backend import ops, pit_ops

    torch.cuda.reset_peak_memory_stats()
    with shadow.shadowed_ops() as census:
        for kind in ("randn", "large"):
            ops.attention(scored_qkv(kind, 32, 577, 12, 64, seed=1).cuda(), 32, 577, 12, 64, 0.125)   # 3 x 12 x 32
    _report(census, "attention bf16 B=32 N=577 H=12")
    with tf32_oracle(), _tf32_mode(), shadow.shadowed_ops() as census:
        qkv = scored_qkv("randn", 16, 785, 12, 64, seed=2, dtype=torch.float32).cuda()
        ops.attention(qkv, 16, 785, 12, 64, 0.125)                                                  # 7 x 12 x 16
    _report(census, "attention tf32 B=16 N=785 H=12")
    with po.shadowed_pit_ops() as census:
        for kind in ("randn", "large"):
            pit_ops.pit_attention_bf16(scored_qkv(kind, 16, 731, 6, 48, seed=3).cuda(), 16, 731, 6, 48, 48 ** -0.5)
    _report(census, "pit_attention_bf16 B=16 T=731 H=6 dh=48")                                       # 12 x 6 x 16
    peak = torch.cuda.max_memory_allocated()
    print(f"peak allocated {peak / 1e9:.2f} GB")
    assert peak < 16e9


# --------------------------------------------------------------------------------------- entry points and invariants
def _relpos_tables(H, dh, window, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rh = 0.5 * torch.randn(2 * window - 1, dh, device="cuda", generator=g)
    rw = 0.5 * torch.randn(2 * window - 1, dh, device="cuda", generator=g)
    pad = (0.5 * torch.randn(3 * H * dh, device="cuda", generator=g)).to(torch.bfloat16)
    return rh, rw, pad


# name: (sequence length, heads, head dim, dtype); relpos: a 10 x 13 grid in 4 x 4 windows of 16 tokens (padded)
KERNELS = {
    "attention_bf16": (197, 3, 64, torch.bfloat16),                   # 224-query chunks
    "attention_bf16_128_row_chunks": (785, 2, 64, torch.bfloat16),    # above 784 keys: 128-query chunks
    "attention_tf32": (197, 3, 64, torch.float32),
    "pit_attention_bf16": (731, 3, 48, torch.bfloat16),
    "relpos_attention_bf16": (130, 4, 64, torch.bfloat16),
}
_RELPOS = dict(gh=10, gw=13, window=4)


def _launch(name, qkv, B, out=None):
    """The launcher's output (``out`` None) or the C entry point's status writing into ``out``."""
    from tfimm.backend import lib, ops, pit_ops, sam_ops

    N, H, dh, _ = KERNELS[name]
    scale = dh ** -0.5
    if name.startswith("relpos"):
        rh, rw, pad = _relpos_tables(H, dh, _RELPOS["window"], seed=1)
        gh, gw, window = _RELPOS["gh"], _RELPOS["gw"], _RELPOS["window"]
        if out is None:
            return sam_ops.relpos_attention(qkv, B, gh, gw, H, dh, scale, rh, rw, window, pad)
        return lib.load().tfimm_b200_relpos_attention_bf16(qkv.data_ptr(), out.data_ptr(), pad.data_ptr(),
                                                           rh.data_ptr(), rw.data_ptr(), B, gh, gw, H, dh, window,
                                                           scale, None)
    if name.startswith("pit"):
        if out is None:
            return pit_ops.pit_attention_bf16(qkv, B, N, H, dh, scale)
        return lib.load().tfimm_b200_pit_attention_bf16(qkv.data_ptr(), out.data_ptr(), B, N, H, dh, scale, None)
    entry = "tfimm_b200_attention_tf32" if name == "attention_tf32" else "tfimm_b200_attention_bf16"
    with _tf32_mode():
        if out is None:
            return ops.attention(qkv, B, N, H, dh, scale)
        return getattr(lib.load(), entry)(qkv.data_ptr(), out.data_ptr(), B, N, H, dh, scale, None)


def _qkv(name, B, seed):
    N, H, dh, dtype = KERNELS[name]
    return scored_qkv("randn", B, N, H, dh, seed, dtype=dtype).cuda()


@pytest.mark.parametrize("name", list(KERNELS))
def test_entry_point_writes_only_its_output(name):
    N, H, dh, dtype = KERNELS[name]
    B, G = 3, 4096                                   # guard elements on each side (16-byte multiples)
    pattern = -1232.0                                # exact in bf16
    qkv = _qkv(name, B, seed=11)
    n = B * N * H * dh
    buf = torch.full((n + 2 * G,), pattern, device="cuda", dtype=dtype)
    out = buf[G:G + n]
    assert _launch(name, qkv, B, out) == 0
    torch.cuda.synchronize()
    assert (buf[:G] == pattern).all() and (buf[-G:] == pattern).all()
    assert not out.isnan().any() and not (out == pattern).any()
    assert torch.equal(out.view(B * N, H * dh), _launch(name, qkv, B))


@pytest.mark.parametrize("name", list(KERNELS))
def test_two_runs_are_bit_identical(name):
    qkv = _qkv(name, 8, seed=12)
    a, b = _launch(name, qkv, 8), _launch(name, qkv, 8)
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize("name", list(KERNELS))
def test_image_of_a_batch_equals_the_image_alone(name):
    N = KERNELS[name][0]
    B = 5
    qkv = _qkv(name, B, seed=13)
    batch = _launch(name, qkv, B).view(B, N, -1)
    for i in (0, 2, B - 1):
        alone = _launch(name, qkv.view(B, N, -1)[i].contiguous().view(N, -1), 1)
        assert torch.equal(batch[i].view(torch.uint8), alone.view(N, -1).view(torch.uint8)), i
