"""The blocked statement of the tensor-core attention kernels and its error bound, on the CPU.

The bf16 / TF32 attention kernels (csrc/attention.cu, pit.cu, relpos_attention.cu) run an online softmax over 64-key
blocks and round P per block, relative to the running maximum.  ``emulate_bf16._softmax_pv`` states that algorithm in
float64 and ``shadow._blocked_softmax_err`` bounds a float32 implementation of it, with the flip criterion on.  Here:

* with one block covering the row the blocked statement is the global one, bit for bit;
* the statement evaluated in float32 -- an honest implementation that only rounds differently -- and a float32 model
  of the kernel's own loop (log2 units, exp2, padded key tiles) pass the rule on every score case below;
* each seeded defect of that kernel model is rejected by the shadow harness on at least one case, naming the op.
"""
import math

import pytest
import torch

LOG2E = 1.4426950408889634


# ----------------------------------------------------------------------------------------------------- score cases
def scored_qkv(kind, B, N, H, dh, seed, dtype=torch.bfloat16):
    """qkv (B * N, 3 * H * dh) in ``dtype`` whose scores scale q.k have the named shape (scale = dh^-0.5):
    randn            q, k, v ~ N(0, 1);
    large            score std ~10, query 0's score of key N // 2 exactly 80 (before the bf16 rounding of qkv);
    late_max         every query's maximum on the last key (inside the partial last block when N % 64 != 0);
    first_max        every query's maximum on key 0;
    equal            q = 0: every score 0, P = 1 exactly;
    neg40            every score -40 +- ~0.1 (a pad key scored 0, or a finite sentinel, would dominate)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, 3, H, dh, generator=g, dtype=torch.float64)
    if kind == "large":
        x[:, :, :2] *= 10.0 ** 0.5                                # q, k entries of variance 10: scores of std ~10
        x[:, N // 2, 1] = x[:, 0, 0] * 80.0 * dh ** 0.5 / x[:, 0, 0].pow(2).sum(-1, keepdim=True)   # query 0: 80
    elif kind in ("late_max", "first_max"):
        key = N - 1 if kind == "late_max" else 0
        # key j's k along the mean direction of all queries, others orthogonal to it: a margin of ~6 in every row
        x[:, :, 0] += 2.0
        x[:, :, 1] -= x[:, :, 1].mean(-1, keepdim=True)
        x[:, key, 1] = 3.0
    elif kind == "equal":
        x[:, :, 0] = 0.0
    elif kind == "neg40":
        # q = 1, k = -5 (1 + noise): scores = -40 + a spread of ~0.1
        x[:, :, 0] = 1.0
        x[:, :, 1] = -40.0 * dh ** 0.5 / dh + 0.3 * x[:, :, 1] * dh ** -0.25
    return x.reshape(B * N, 3 * H * dh).to(dtype)


KINDS = ["randn", "large", "late_max", "first_max", "equal", "neg40"]


def _scores(qkv, B, N, H, dh):
    q, k, _ = qkv.double().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    return dh ** -0.5 * q @ k.transpose(-1, -2)


@pytest.mark.parametrize("N", [17, 65, 197])
def test_score_cases_have_their_shape(N):
    B, H, dh = 2, 2, 64
    s = {kind: _scores(scored_qkv(kind, B, N, H, dh, seed=N), B, N, H, dh) for kind in KINDS}
    if N > 1:
        assert s["large"].amax() > 70 and s["large"].std() > 6
    assert (s["late_max"].argmax(-1) == N - 1).all()
    assert (s["first_max"].argmax(-1) == 0).all()
    assert (s["equal"] == 0).all()
    assert s["neg40"].amax() < -35 and s["neg40"].amin() > -45


# ---------------------------------------------------------------------------------------------- the blocked statement
@pytest.mark.parametrize("N", [1, 63, 64, 65, 197])
@pytest.mark.parametrize("rounded", [False, True])
def test_one_block_equals_the_global_form_bit_for_bit(N, rounded):
    from oracle import emulate_bf16 as emu

    g = torch.Generator().manual_seed(N)
    s = 4 * torch.randn(2, 3, N, N, generator=g, dtype=torch.float64)
    v = torch.randn(2, 3, N, 64, generator=g, dtype=torch.float64)
    rnd = emu.round_bf16 if rounded else None
    # the global form: exp(s - row max), the row sum of the unrounded p, rounded p @ v, divided at the end
    p = torch.exp(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    pr = rnd(p) if rounded else p
    want = (pr @ v) / l
    for key_block in (None, N, N + 1, 1024):
        o, probs = emu._softmax_pv(s, v, rnd, key_block)
        assert torch.equal(o, want) and torch.equal(probs, pr / l), key_block


def test_blocks_differ_from_the_global_form_only_by_the_rounding_of_p():
    """Unrounded, the online softmax is the softmax (to float64 rounding); rounded per block, it is not the global
    rounding -- the reason the statement has to follow the kernel's blocks."""
    from oracle import emulate_bf16 as emu

    g = torch.Generator().manual_seed(1)
    s = 4 * torch.randn(2, 3, 197, 197, generator=g, dtype=torch.float64)
    v = torch.randn(2, 3, 197, 64, generator=g, dtype=torch.float64)
    exact = torch.softmax(s, -1) @ v
    assert (emu._softmax_pv(s, v, None, 64)[0] - exact).abs().max().item() < 1e-13
    blocked = emu._softmax_pv(s, v, emu.round_bf16, 64)[0]
    assert not torch.equal(blocked, emu._softmax_pv(s, v, emu.round_bf16, None)[0])


# ------------------------------------------------------------------------------------ a float32 model of the kernel
def _trunc_bf16(p):
    return (p.float().view(torch.int32) & -65536).view(torch.float32)


def kernel_model(qkv, B, N, H, dh, scale, defect=None):
    """The bf16 tensor-core kernel's loop in float32 (csrc/attention.cu): scores times fp32(scale log2 e), keys padded
    to a multiple of 16 and masked to -inf, 64-key blocks, m = running max, alpha = exp2(m_old - m), p = exp2(s - m),
    l = alpha l + sum p, O = alpha O + bf16(p) V, O / l rounded to bf16.  ``defect`` seeds one mistake."""
    q, k, v = qkv.float().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    c = torch.tensor(scale * LOG2E, dtype=torch.float32)
    if defect == "scale_log2e_in_bf16":
        c = c.to(torch.bfloat16).float()
    npad = (N + 15) // 16 * 16
    t = torch.nn.functional.pad((q @ k.transpose(-1, -2)) * c, (0, npad - N),
                                value=0.0 if defect == "pad_keys_scored_0" else -math.inf)
    v = torch.nn.functional.pad(v, (0, 0, 0, npad - N))                     # zero-filled key rows
    rnd = _trunc_bf16 if defect == "p_truncated" else (lambda p: p.to(torch.bfloat16).float())
    m = torch.full(t.shape[:-1] + (1,), -math.inf)
    l = torch.zeros_like(m)
    o = torch.zeros(t.shape[:-1] + (dh,))
    for j0 in range(0, npad, 64):
        if defect == "last_partial_block_dropped" and N % 64 and j0 + 64 > N:
            break
        tb = t[..., j0:j0 + 64]
        m_new = torch.maximum(m, tb.amax(-1, keepdim=True))
        alpha = torch.exp2(m - m_new)
        p = torch.exp2(tb - m_new)
        pr = rnd(p)
        l = (l if defect == "l_not_rescaled" else l * alpha) + (pr if defect == "l_from_rounded_p" else p).sum(-1, True)
        o = o * alpha + pr @ v[..., j0:j0 + 64, :]
        m = m_new
    return (o / l).permute(0, 2, 1, 3).reshape(B * N, H * dh).to(torch.bfloat16)


DEFECTS = ["p_truncated", "l_from_rounded_p", "l_not_rescaled", "pad_keys_scored_0", "scale_log2e_in_bf16",
           "last_partial_block_dropped"]
LENGTHS = [1, 15, 17, 63, 64, 65, 129, 197]
CASES = [(kind, N) for kind in KINDS for N in LENGTHS]


def _shadowed(attention, cases, B=2, H=3, dh=64):
    """{(kind, N): census row} of ``attention`` (installed as ops.attention) under the shadow harness."""
    from oracle import shadow
    from tfimm.backend import ops

    rows = {}
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "attention", attention)
        with shadow.shadowed_ops() as census:
            for kind, N in cases:
                ops.attention(scored_qkv(kind, B, N, H, dh, seed=N), B, N, H, dh, dh ** -0.5)
                rows[(kind, N)] = census.rows[-1]
    return rows, census


def test_float32_statement_passes_the_rule_on_every_case():
    from oracle import emulate_bf16 as emu

    with emu.emulated_ops(arithmetic=torch.float32):
        standin = emu.attention
        rows, census = _shadowed(lambda *a, **k: standin(*a, **k), CASES)
    print("\n" + census.table())
    census.assert_ok()
    assert len(rows) == len(CASES) and all(r["op"] == "attention" for r in rows.values())


def test_float32_kernel_model_passes_the_rule_on_every_case():
    rows, census = _shadowed(kernel_model, CASES)
    print("\n" + census.table())
    census.assert_ok()
    # the rule is tight enough to see the model's own rounding: some case uses a visible share of its bound
    assert max(r["worst"] for r in rows.values()) > 0.1


@pytest.mark.parametrize("defect", DEFECTS)
def test_seeded_defect_is_rejected(defect):
    rows, census = _shadowed(lambda *a, **k: kernel_model(*a, defect=defect, **k), CASES)
    failed = [case for case, r in rows.items() if not r["ok"]]
    print(f"\n{defect}: rejected on {len(failed)} / {len(rows)} cases: {failed}")
    with pytest.raises(AssertionError, match="attention"):
        census.assert_ok()
    assert failed


def test_tf32_form_passes_the_rule():
    """The same rule with P rounded to TF32 (tests/tf32_oracle.py; fp32 output, so no ulp term and no flip count): the
    statement evaluated in float32 from fp32 scores passes on every score case."""
    from oracle import emulate_bf16 as emu
    from oracle import shadow
    from tf32_oracle import round_p_tf32, round_tf32

    B, H, dh = 2, 3, 64
    for kind, N in CASES:
        qkv = round_tf32(scored_qkv(kind, B, N, H, dh, seed=N, dtype=torch.float32))
        q, k, v = qkv.double().view(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
        s = dh ** -0.5 * q @ k.transpose(-1, -2)
        ref = emu._softmax_pv(s, v, round_p_tf32, 64)[0]
        o = emu._softmax_pv(s.float(), v.float(), round_tf32, 64)[0]
        bound = shadow._blocked_attention_bound(qkv, B, N, H, dh, dh ** -0.5, round_p_tf32)
        worst = ((o.double() - ref).abs() / bound.view(B, N, H, dh).permute(0, 2, 1, 3)).max().item()
        assert worst <= 1.0, (kind, N, worst)
