"""The persistent 128 x 256 instance of the plain bf16 GEMM (block_n=1) against the per-tile instances.

Every output element is the same fp32 sum over the same k16 steps, with the same epilogue operations in the same order,
so each case must match the 256-wide fragment-epilogue kernel and the 128-wide staged kernel bit for bit over the whole
buffer: the output is a column slice of a wider buffer with a padded row stride and rows past M, all canaries, and
nothing outside the view may change.  Each case also checks the float64 statement within the bounds of
tests/test_gemm_staged_epilogue_gpu.py.
"""
import pytest
import torch

from test_gemm_staged_epilogue_gpu import ACTS, _act64, _inputs, _run

pytestmark = pytest.mark.gpu

PERSISTENT = 1   # force_block_n of the persistent instance
# M, N, K, in order: M and N tails (N % 256 != 0; the fp32 tile's second 128-column half is partial in one tile and
# wholly past N in another, and the last tile's second warpgroup has no rows); one k-block; two k-blocks (fewer than
# the three ring stages); K % 64 != 0; fewer tiles than SMs; 71 x 4 = 284 tiles, more than twice the SMs and not a
# multiple of them, with 7 k-blocks per tile, so ring phases and the staging handoff wrap across the tiles of a CTA.
SHAPES = [(300, 328, 192), (200, 264, 64), (130, 512, 128), (256, 256, 200), (1000, 520, 256), (9000, 776, 448)]


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("res_mode", ["none", "separate", "inplace"])
def test_persistent_matches_per_tile_instances(M, N, K, out_dtype, res_mode):
    a, w, bias, gamma_all, canvas, res = _inputs(M, N, K, out_dtype, res_mode, seed=M * 5 + N * 3 + K)
    y = a.double() @ w.double().t() + bias.double()
    r = (canvas[:M, 24:24 + N] if res_mode == "inplace" else res).double() if res_mode != "none" else 0.0
    outside = torch.ones(canvas.shape, dtype=torch.bool, device=canvas.device)
    outside[:M, 24:24 + N] = False
    for gamma in (None, gamma_all):
        s = gamma.double() if gamma is not None else 1.0
        for act_post in (False, True):
            for act in ACTS:
                got = _run(a, w, bias, gamma, canvas, res, res_mode, N, act, act_post, PERSISTENT)
                for block_n in (256, 128):
                    want = _run(a, w, bias, gamma, canvas, res, res_mode, N, act, act_post, block_n)
                    assert torch.equal(_bits(got), _bits(want)), (act, gamma is not None, act_post, block_n)
                assert torch.equal(got[outside], canvas[outside]), act
                ref = _act64(r + s * y, act) if act_post else r + s * _act64(y, act)
                err = (got[:M, 24:24 + N].double() - ref).abs().max().item()
                tol = 2e-3 if out_dtype == torch.float32 else 2e-2 + 4e-3 * ref.abs().max().item()
                assert err < tol, (act, gamma is not None, act_post, err, tol)


@pytest.mark.parametrize("res_mode", ["none", "inplace"])
def test_persistent_bf16_ragged_rows_keep_fragment_epilogue(res_mode):
    """bf16 rows of N = 100 do not end on a 16-byte boundary, where a TMA store would not clip them: forcing the
    persistent instance there must give the fragment epilogue's bits, canaries included."""
    M, N, K = 77, 100, 256
    a, w, bias, gamma, canvas, res = _inputs(M, N, K, torch.bfloat16, res_mode, seed=11)
    for act in ACTS:
        got = _run(a, w, bias, gamma, canvas, res, res_mode, N, act, False, PERSISTENT)
        want = _run(a, w, bias, gamma, canvas, res, res_mode, N, act, False, 256)
        assert torch.equal(_bits(got), _bits(want)), act
