"""Swin window attention against the float64 statement of its own algorithm, on the H100.

Both entry points of csrc/window_attention.cu -- region labels + [H][N][N] bias (the <64> and <144> instantiations), and
64-bit mask words + the padded [H][64][64] bias (N <= 52) -- are held here, through the shadow harness, to
``emulate_bf16.window_attention{,_tc}`` within ``shadow._window_attention_bound`` (+ one bf16 ulp of the output) and to
the flip criterion (under ``FLIP_LIMIT`` of the outputs not correctly rounded):

* over the score cases of tests/test_window_attention_cpu.py -- among them ``ties``, where every exact output is a bf16
  rounding midpoint, which a kernel that multiplies by a rounded 1 / l breaks at N = 15, 52 or 121 -- at every N of the
  8-key and 16-row tiles up to 64 and 144 tokens; square N on real Swin layouts, shifted and unshifted, the others on
  a random row map and random region labels; head counts 1, 3, 4 and 32, with pair counts off the 4 warps of a CTA;
* the padded-table entry bit-identical to the labels entry on equivalent tables (it changes only where the bias and
  the mask are read from);
* at Swin-B's stage-1 shape, batch 32: 2,048 CTAs;
* called through the C entry points with the output in the middle of a canary buffer: nothing outside it is written
  and nothing in it is NaN; two runs are bit-identical, and image i of a batch equals image i run alone.

``-s`` prints the census of every case: worst error / bound and flip %.
"""
import math
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
if str(HERE) not in sys.path:
    sys.path.insert(0, str(HERE))

from test_window_attention_cpu import DH, KINDS, SCALE, padded_tables, scattered, square, window_case  # noqa: E402

pytestmark = pytest.mark.gpu


def _geometries(N):
    """Real layouts for square N (shifted where the window has room, 28 x 21 tokens for 7 x 7), else a random one."""
    ws = math.isqrt(N)
    if ws * ws != N:
        return [scattered(N, 3, seed=N)]
    geos = [square(ws, 2 * ws, ws, 0)]
    if ws > 1:
        geos.append(square(2 * ws, 2 * ws, ws, ws // 2))
    if ws == 7:
        geos.append(square(28, 21, 7, 3))
    return geos


def _cuda(c):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()}


def _run(N, H, B=1):
    """Every kind on every geometry of N, shadowed; N <= 52 also through the padded-table entry, which must match the
    labels entry bit for bit."""
    from oracle import shadow
    from tfimm.backend import ops

    rows = {}
    with shadow.shadowed_ops() as census:
        for geo in _geometries(N):
            for j, kind in enumerate(KINDS):
                c = _cuda(window_case(kind, geo, B, H, seed=N * 31 + j))
                args = (c["B"], c["nw"], N, H, DH, SCALE)
                out = ops.window_attention(c["qkv"], c["bias"], c["row_map"], c["labels"], *args)
                rows[("labels", kind, geo["name"])] = census.rows[-1]
                if N <= 52:   # a table entry outside N x N, if read, would dominate its row
                    bias_pad, bits = padded_tables(c["bias"], c["labels"], c["nw"], N, fill=1e4)
                    out_tc = ops.window_attention_tc(c["qkv"], bias_pad, c["row_map"], bits, *args)
                    rows[("padded", kind, geo["name"])] = census.rows[-1]
                    assert torch.equal(out_tc.view(torch.int16), out.view(torch.int16)), (kind, geo["name"])
    print(f"\n=== window attention N={N} H={H}")
    for (entry, kind, name), r in rows.items():
        print(f"{'ok  ' if r['ok'] else 'FAIL'} {entry:<7} {kind:<14} {name:<16} worst {r['worst']:7.3f} x bound  "
              f"flips {100 * r['flips']:6.3f} %")
    failed = [key for key, r in rows.items() if not r["ok"]]
    assert not failed, failed
    assert census.ops() == ({"window_attention", "window_attention_tc"} if N <= 52 else {"window_attention"})


HEADS = [1, 3, 4, 32]
N_64 = [1, 4, 9, 15, 16, 17, 25, 36, 49, 52, 63, 64]
N_144 = [65, 81, 100, 121, 143, 144]


@pytest.mark.parametrize("N", N_64)
def test_labels_entry_64_rows_within_the_bound(N):
    _run(N, HEADS[N_64.index(N) % 4])


@pytest.mark.parametrize("N", N_144)
def test_labels_entry_144_rows_within_the_bound(N):
    _run(N, HEADS[N_144.index(N) % 4])


def test_several_waves_within_the_bound():
    """Swin-B stage 1 at batch 32 (56 x 56 tokens, 7 x 7 windows, 4 heads): 8,192 (window, head) pairs, 2,048 CTAs,
    shifted, through both entry points; randn and large logits."""
    from oracle import shadow
    from tfimm.backend import ops

    torch.cuda.reset_peak_memory_stats()
    geo = square(56, 56, 7, 3)
    with shadow.shadowed_ops() as census:
        for kind in ("randn", "large"):
            c = _cuda(window_case(kind, geo, 32, 4, seed=5))
            args = (32, geo["nw"], 49, 4, DH, SCALE)
            out = ops.window_attention(c["qkv"], c["bias"], c["row_map"], c["labels"], *args)
            bias_pad, bits = padded_tables(c["bias"], c["labels"], geo["nw"], 49)
            assert torch.equal(ops.window_attention_tc(c["qkv"], bias_pad, c["row_map"], bits, *args), out)
    print("\n=== Swin-B stage 1, batch 32\n" + census.table())
    census.assert_ok()
    assert len(census.rows) == 4
    peak = torch.cuda.max_memory_allocated()
    print(f"peak allocated {peak / 1e9:.2f} GB")
    assert peak < 16e9


# --------------------------------------------------------------------------------------- entry points and invariants
# name: (entry, h, w, ws, shift, heads): the <64> and <144> instantiations of the labels entry, and the padded entry
ENTRIES = {
    "labels_64": ("labels", 28, 21, 7, 3, 3),
    "labels_144": ("labels", 24, 36, 12, 6, 4),
    "padded": ("padded", 28, 21, 7, 3, 3),
}


def _inputs(name, B, seed):
    entry, h, w, ws, shift, H = ENTRIES[name]
    geo = square(h, w, ws, shift)
    c = _cuda(window_case("randn", geo, B, H, seed))
    if entry == "padded":
        c["bias"], c["labels"] = padded_tables(c["bias"], c["labels"], geo["nw"], geo["N"])
    return c


def _launch(name, c, out=None):
    """The launcher's output (``out`` None) or the C entry point's status writing into ``out``."""
    from tfimm.backend import lib, ops

    padded = ENTRIES[name][0] == "padded"
    args = (c["B"], c["nw"], c["N"], c["H"], DH, SCALE)
    if out is None:
        fn = ops.window_attention_tc if padded else ops.window_attention
        return fn(c["qkv"], c["bias"], c["row_map"], c["labels"], *args)
    entry = "tfimm_b200_window_attention_tc_bf16" if padded else "tfimm_b200_window_attention_bf16"
    return getattr(lib.load(), entry)(c["qkv"].data_ptr(), out.data_ptr(), c["bias"].data_ptr(),
                                      c["row_map"].data_ptr(), c["labels"].data_ptr(), *args, None)


@pytest.mark.parametrize("name", list(ENTRIES))
def test_entry_point_writes_only_its_output(name):
    B, G = 3, 4096                                   # guard elements on each side (16-byte multiples)
    pattern = -1232.0                                # exact in bf16
    c = _inputs(name, B, seed=11)
    n = c["qkv"].numel() // 3
    buf = torch.full((n + 2 * G,), pattern, device="cuda", dtype=torch.bfloat16)
    out = buf[G:G + n]
    assert _launch(name, c, out) == 0
    torch.cuda.synchronize()
    assert (buf[:G] == pattern).all() and (buf[-G:] == pattern).all()
    assert not out.isnan().any() and not (out == pattern).any()
    assert torch.equal(out.view(c["qkv"].shape[0], -1), _launch(name, c))


@pytest.mark.parametrize("name", list(ENTRIES))
def test_two_runs_are_bit_identical(name):
    c = _inputs(name, 8, seed=12)
    a, b = _launch(name, c), _launch(name, c)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("name", list(ENTRIES))
def test_image_of_a_batch_equals_the_image_alone(name):
    B = 5
    c = _inputs(name, B, seed=13)
    L = c["nw"] * c["N"]
    batch = _launch(name, c).view(B, L, -1)
    for i in (0, 2, B - 1):
        alone = dict(c, B=1, qkv=c["qkv"].view(B, L, -1)[i].contiguous().view(L, -1))
        assert torch.equal(batch[i].view(torch.int16), _launch(name, alone).view(torch.int16)), i
