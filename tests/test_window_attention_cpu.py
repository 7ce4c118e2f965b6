"""Swin window attention's float64 statement and its error bound, on the CPU.

The mma.sync window kernel (csrc/window_attention.cu) runs the shared core's softmax as one block over the whole window:
logits fma(q.k, scale, bias) (+ -100 between shift regions) in log2 units, p = exp2(s - row max), l the fp32 sum of the
unrounded p, bf16(p) V, O / l correctly rounded.  ``emulate_bf16.window_attention{,_tc}`` state it in float64 and
``shadow._window_attention_bound`` bounds a float32 implementation of it, with the flip criterion on.  Here:

* the statement equals an explicit roll -> partition -> bias + mask -> softmax -> reverse -> roll, for both entry
  formats (region labels + [H][N][N] bias, or 64-bit mask words + the padded [H][64][64] bias);
* the statement evaluated in float32 and a float32 model of the kernel pass the rule on every case below;
* each seeded defect of that model is rejected by the shadow harness on at least one case, naming the op.
"""
import math

import numpy as np
import pytest
import torch

from test_attention_blocked_cpu import KINDS as SCORE_KINDS
from test_attention_blocked_cpu import _trunc_bf16, scored_qkv

LOG2E = 1.4426950408889634
DH = 32
SCALE = DH ** -0.5
KINDS = SCORE_KINDS + ["ties", "bias_dominant", "lone_region"]


# ------------------------------------------------------------------------------------------------------- geometries
def square(h, w, ws, shift):
    """A Swin layout: the row map and region labels of ``window_tables`` (labels None when unshifted)."""
    from tfimm.architectures.swin import window_tables

    row_map, labels = window_tables(h, w, ws, shift)
    return dict(N=ws * ws, nw=(h // ws) * (w // ws), row_map=row_map, labels=labels, name=f"{h}x{w}/{ws}/{shift}")


def scattered(N, nw, seed):
    """Any N: a random permutation of the image's tokens as the row map, and random labels of 3 regions."""
    rng = np.random.default_rng(seed)
    return dict(N=N, nw=nw, row_map=rng.permutation(nw * N).astype(np.int32),
                labels=rng.integers(0, 3, nw * N).astype(np.int32), name=f"perm N={N} nw={nw}")


def _ties_v(Bw, N, H, seed):
    """v (Bw, N, H, dh) whose every exact output is a bf16 rounding midpoint m: with P = 1 and l = N, two keys of each
    column carry the bf16 parts hi + lo = N m (exact: m has 9 significant bits, N at most 8) and the others are 0."""
    g = torch.Generator().manual_seed(seed)
    b = (torch.rand(Bw, H, DH, generator=g, dtype=torch.float64) * 3.9 + 0.1).to(torch.bfloat16).double()
    b = b * torch.where(torch.rand(Bw, H, DH, generator=g) < 0.5, -1.0, 1.0).double()
    from oracle.shadow import ulp_bf16

    m = b + 0.5 * ulp_bf16(b) * b.sign()
    hi = (N * m).to(torch.bfloat16).double()
    lo = (N * m - hi).to(torch.bfloat16).double()
    assert torch.equal(hi + lo, N * m) and (m.to(torch.bfloat16).double() != m).all()
    v = torch.zeros(Bw, N, H, DH, dtype=torch.float64)
    col = torch.arange(DH)
    v[:, col % N, :, col] = hi.permute(2, 0, 1)
    if N > 1:      # (N = 1: the output is v itself, a bf16 value; there is no tie to make)
        v[:, (col + 1) % N, :, col] = lo.permute(2, 0, 1)
    return v


def window_case(kind, geo, B, H, seed):
    """Inputs of one launch: qkv built per window, in window order, by ``kind`` and scattered to token order through
    the row map; the [H][N][N] bias; row map and labels (torch int32).  Score kinds as tests/test_attention_blocked_cpu.py
    (bias std 1 on top), and
    ties           q = 0, no bias and no mask: P = 1, l = N, every exact output a bf16 rounding midpoint;
    bias_dominant  bias std 5 over q.k of std ~0.3;
    lone_region    the last token of every window in a region of its own: its row's mass sits on itself."""
    N, nw = geo["N"], geo["nw"]
    Bw = B * nw
    g = torch.Generator().manual_seed(seed + 1)
    labels = geo["labels"]
    if kind in ("equal", "ties"):
        bias = torch.zeros(H, N, N)
    else:
        bias = (5.0 if kind == "bias_dominant" else 1.0) * torch.randn(H, N, N, generator=g)
    if kind == "ties":
        labels = None
        x = torch.zeros(Bw, N, 3, H, DH, dtype=torch.float64)
        x[:, :, 1] = torch.randn(Bw, N, H, DH, generator=g, dtype=torch.float64)
        x[:, :, 2] = _ties_v(Bw, N, H, seed)
        win = x.reshape(Bw * N, 3 * H * DH).to(torch.bfloat16)
    else:
        win = scored_qkv("randn" if kind in ("bias_dominant", "lone_region") else kind, Bw, N, H, DH, seed)
        if kind == "bias_dominant":
            win = (win.float() * 0.3).to(torch.bfloat16)
    if kind == "lone_region":
        labels = (np.zeros(nw * N, np.int32) if labels is None else labels.copy())
        labels[N - 1::N] = 99
    row_map = torch.from_numpy(geo["row_map"])
    idx = (torch.arange(B)[:, None] * (nw * N) + row_map.long()[None, :]).reshape(-1)
    qkv = torch.empty_like(win)
    qkv[idx] = win
    return dict(qkv=qkv, bias=bias, row_map=row_map, labels=None if labels is None else torch.from_numpy(labels),
                B=B, nw=nw, N=N, H=H)


def padded_tables(bias, labels, nw, N, fill=0.0):
    """The padded-table entry's equivalents: bias in [H][64][64] (``fill`` outside N x N) and one 64-bit word per
    query row, bit j set where tokens i and j lie in different regions (None without labels)."""
    H = bias.shape[0]
    bias_pad = torch.full((H, 64, 64), fill, dtype=torch.float32, device=bias.device)
    bias_pad[:, :N, :N] = bias
    if labels is None:
        return bias_pad, None
    lab = labels.view(nw, N).long()
    diff = (lab[:, :, None] != lab[:, None, :]).to(torch.int64)
    bits = torch.zeros(nw, 64, dtype=torch.int64, device=bias.device)
    bits[:, :N] = (diff << torch.arange(N, device=bias.device)[None, None, :]).sum(-1)
    return bias_pad, bits


def launch(c, entry, fn=None):
    """Runs ``fn`` (default: ops.window_attention / window_attention_tc) on case ``c`` through ``entry``
    ("labels" or "padded")."""
    from tfimm.backend import ops

    args = (c["B"], c["nw"], c["N"], c["H"], DH, SCALE)
    if entry == "labels":
        return (fn or ops.window_attention)(c["qkv"], c["bias"], c["row_map"], c["labels"], *args)
    bias_pad, bits = padded_tables(c["bias"], c["labels"], c["nw"], c["N"])
    return (fn or ops.window_attention_tc)(c["qkv"], bias_pad, c["row_map"], bits, *args)


# --------------------------------------------------------------------------------------------- the statement itself
def _explicit(qkv, B, h, w, ws, shift, bias, labels, H, round_p):
    """roll(-shift) -> window_partition -> softmax(scale q k^T + bias + mask) V -> window_reverse -> roll(shift), in
    float64, with the window kernels' single-block softmax: P rounded by ``round_p``, l the sum of the unrounded p."""
    C = H * DH
    x = qkv.double().view(B, h, w, 3 * C)
    x = torch.roll(x, (-shift, -shift), (1, 2))
    nh, nwx, n = h // ws, w // ws, ws * ws
    xw = x.view(B, nh, ws, nwx, ws, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(B * nh * nwx, n, 3, H, DH)
    q, k, v = xw.permute(2, 0, 3, 1, 4)
    s = SCALE * q @ k.transpose(-1, -2) + bias.double()
    if labels is not None:
        lab = torch.from_numpy(labels).view(nh * nwx, n)
        mask = torch.where(lab[:, None, :] != lab[:, :, None], -100.0, 0.0).double()
        s = (s.view(B, nh * nwx, H, n, n) + mask[None, :, None]).view(s.shape)
    p = torch.exp(s - s.amax(-1, keepdim=True))
    o = round_p(p) @ v / p.sum(-1, keepdim=True)
    o = o.permute(0, 2, 1, 3).reshape(B, nh, nwx, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, h, w, C)
    return torch.roll(o, (shift, shift), (1, 2)).reshape(B * h * w, C)


EXPLICIT = [(14, 14, 7, 3), (14, 14, 7, 0), (28, 21, 7, 3), (8, 8, 4, 2), (21, 14, 7, 3), (24, 24, 12, 6),
            (24, 12, 12, 0), (33, 22, 11, 5)]


@pytest.mark.parametrize("h,w,ws,shift", EXPLICIT)
def test_statement_equals_explicit_roll_partition_softmax(h, w, ws, shift):
    from oracle import emulate_bf16 as emu

    B, H = 2, 3
    geo = square(h, w, ws, shift)
    c = window_case("randn", geo, B, H, seed=h * w + shift)
    N, nw = geo["N"], geo["nw"]
    for dt, round_p in ((torch.float64, lambda p: p), (torch.bfloat16, emu.round_bf16)):
        qkv = c["qkv"].to(dt)
        want = _explicit(qkv, B, h, w, ws, shift, c["bias"], geo["labels"], H, round_p)
        entries = [emu.window_attention(qkv, c["bias"], c["row_map"], c["labels"], B, nw, N, H, DH, SCALE)]
        if N <= 52:
            bias_pad, bits = padded_tables(c["bias"], c["labels"], nw, N, fill=float("nan"))
            entries.append(emu.window_attention_tc(qkv, bias_pad, c["row_map"], bits, B, nw, N, H, DH, SCALE))
        for got in entries:
            if dt == torch.float64:
                assert (got - want).abs().max().item() < 1e-12
            else:       # the same single-block algorithm; the output rounded once
                assert torch.equal(got, want.to(dt))


# ------------------------------------------------------------------------------------ a float32 model of the kernel
def kernel_model(qkv, bias, row_map, masked, B, nw_img, N, H, dh, scale, defect=None):
    """The window kernel in float32 (csrc/window_attention.cu): keys padded to a multiple of 8 and scored -inf, query
    rows to a multiple of 16 (scored 0, discarded); logits fl(fl(fma(q.k, fl(scale), bias)) + -100 where ``masked``)
    * fl(log2 e); p = exp2(s - row max); l = the fp32 sum of the unrounded p; bf16(p) V; O / l correctly rounded; rows
    scattered back through the row map.  ``masked`` (nw_img, N, N) bool or None.  ``defect`` seeds one mistake."""
    Bw = B * nw_img
    idx = (torch.arange(B)[:, None] * (nw_img * N) + row_map.long()[None, :]).reshape(-1)
    q, k, v = qkv[idx].float().view(Bw, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    kp, qp = -(-N // 8) * 8, -(-N // 16) * 16
    pad = torch.nn.functional.pad
    q, k, v = pad(q, (0, 0, 0, qp - N)), pad(k, (0, 0, 0, kp - N)), pad(v, (0, 0, 0, kp - N))
    acc = q @ k.transpose(-1, -2)                                              # (Bw, H, qp, kp)
    b = bias.float()
    if defect == "bias_transposed":
        b = b.transpose(-1, -2)
    b = pad(b, (0, kp - N, 0, qp - N))
    sc = torch.tensor(scale, dtype=torch.float32).double()
    fma = (lambda a, c: (a.double() * sc + c.double()).float())              # one rounding
    val = fma(acc, torch.zeros_like(b) if defect == "bias_after_log2e" else b)
    if masked is not None and defect != "region_mask_ignored":
        mw = pad(masked, (0, kp - N, 0, qp - N))[torch.arange(Bw) % nw_img][:, None]
        val = torch.where(mw, val + (-math.inf if defect == "mask_minus_inf" else -100.0), val)
    s = val * torch.tensor(LOG2E, dtype=torch.float32)
    if defect == "bias_after_log2e":
        s = s + b
    keys, rows = torch.arange(kp), torch.arange(qp)[:, None]
    s = torch.where(keys >= N, 0.0 if defect == "pad_keys_scored_0" else -math.inf, s)
    s = torch.where((rows >= N) & (keys < N), 0.0, s)
    p = torch.exp2(s - s.amax(-1, keepdim=True))
    pr = _trunc_bf16(p) if defect == "p_truncated" else p.to(torch.bfloat16).float()
    l = (pr if defect == "l_from_rounded_p" else p).sum(-1, keepdim=True)
    o = pr @ v
    o = o * (1.0 / l) if defect == "o_times_inv_l" else o / l
    o = o[:, :, :N].permute(0, 2, 1, 3).reshape(Bw * N, H * dh).to(torch.bfloat16)
    if defect == "row_map_off_by_one":
        idx = (torch.arange(B)[:, None] * (nw_img * N) + torch.roll(row_map, -1).long()[None, :]).reshape(-1)
    out = torch.empty_like(o)
    out[idx] = o
    return out


def model_entries(defect=None):
    """The kernel model behind both entry points' signatures."""
    def labels_entry(qkv, bias, row_map, labels, B, nw_img, N, H, dh, scale):
        masked = None
        if labels is not None:
            lab = labels.view(nw_img, N)
            masked = lab[:, None, :] != lab[:, :, None]
        return kernel_model(qkv, bias, row_map, masked, B, nw_img, N, H, dh, scale, defect)

    def padded_entry(qkv, bias_pad, row_map, maskbits, B, nw_img, N, H, dh, scale):
        masked = None
        if maskbits is not None:
            masked = ((maskbits[:, :N, None] >> torch.arange(N)[None, None, :]) & 1).bool()
        return kernel_model(qkv, bias_pad[:, :N, :N], row_map, masked, B, nw_img, N, H, dh, scale, defect)

    return labels_entry, padded_entry


# every edge of N the kernel has (the 8-key and 16-row tiles, 64 and 144 rows); the tie case's N = 15, 52 and 121
GEOMETRIES = [square(14, 14, 7, 3), square(14, 14, 7, 0), square(28, 21, 7, 3), square(8, 8, 4, 2), square(9, 9, 3, 1),
              square(22, 22, 11, 5), square(24, 24, 12, 6), square(14, 14, 7, 1),
              scattered(1, 3, 1), scattered(15, 3, 2), scattered(17, 2, 3), scattered(52, 2, 4),
              scattered(63, 2, 5), scattered(65, 2, 6), scattered(121, 1, 7), scattered(143, 1, 8)]
CASES = [(kind, i) for kind in KINDS for i in range(len(GEOMETRIES))]


def _shadowed(entries, cases, B=2, H=3):
    """{(entry, kind, geometry index): census row} of ``entries`` = (labels entry, padded entry), installed as
    ops.window_attention / window_attention_tc, under the shadow harness; the padded entry on N <= 52."""
    from oracle import shadow
    from tfimm.backend import ops

    rows = {}
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "window_attention", entries[0])
        mp.setattr(ops, "window_attention_tc", entries[1])
        with shadow.shadowed_ops() as census:
            for kind, i in cases:
                c = window_case(kind, GEOMETRIES[i], B, H, seed=100 * i + KINDS.index(kind))
                for entry in ("labels", "padded") if c["N"] <= 52 else ("labels",):
                    launch(c, entry)
                    rows[(entry, kind, i)] = census.rows[-1]
    return rows, census


def _failed(rows):
    return sorted({(e, kind, GEOMETRIES[i]["name"]) for (e, kind, i), r in rows.items() if not r["ok"]})


def test_score_cases_have_their_shape():
    from oracle import emulate_bf16 as emu

    for i in (0, 9, 11, 14):                                  # N = 49, 15, 52, 121
        geo = GEOMETRIES[i]
        c = window_case("ties", geo, 2, 3, seed=i)
        o = emu.window_attention(c["qkv"].double(), c["bias"], c["row_map"], c["labels"], 2, geo["nw"], geo["N"], 3,
                                 DH, SCALE)                   # float64 in, float64 out: the exact outputs
        assert c["labels"] is None and (o.abs() >= 0.1).all() and (o.to(torch.bfloat16).double() != o).all()
        lab = window_case("lone_region", geo, 2, 3, seed=i)["labels"].view(geo["nw"], geo["N"])
        assert (lab[:, -1:] != lab[:, :-1]).all()
    bd = window_case("bias_dominant", GEOMETRIES[0], 2, 3, seed=3)
    q, k, _ = bd["qkv"].double().view(-1, 3, 3, DH).permute(1, 0, 2, 3)
    assert bd["bias"].std() > 4 and (SCALE * (q * k).sum(-1)).std() < 0.5


def test_float32_statement_passes_the_rule_on_every_case():
    from oracle import emulate_bf16 as emu

    with emu.emulated_ops(arithmetic=torch.float32):
        lab, pad = emu.window_attention, emu.window_attention_tc
        rows, census = _shadowed((lambda *a: lab(*a), lambda *a: pad(*a)), CASES)
    print("\n" + census.table())
    census.assert_ok()
    assert {r["op"] for r in rows.values()} == {"window_attention", "window_attention_tc"}


def test_float32_kernel_model_passes_the_rule_on_every_case():
    rows, census = _shadowed(model_entries(), CASES)
    print("\n" + census.table())
    assert not _failed(rows), _failed(rows)
    # the rule is tight enough to see the model's own rounding: some case uses a visible share of its bound
    assert max(r["worst"] for r in rows.values()) > 0.1
    assert max(r["flips"] for (_, kind, _), r in rows.items() if kind == "ties") == 0.0


def test_minus_inf_for_the_region_mask_is_accepted():
    """-inf in place of -100 is a legitimate kernel: exp2 of a masked logit, (-100 - spread) log2 e < -144, is below
    2^-126 either way -- under the bound's allowance for fp32 underflow -- and a row's own token always survives."""
    rows, census = _shadowed(model_entries("mask_minus_inf"), CASES)
    assert not _failed(rows), _failed(rows)


DEFECTS = ["o_times_inv_l", "p_truncated", "l_from_rounded_p", "bias_transposed", "bias_after_log2e",
           "region_mask_ignored", "pad_keys_scored_0", "row_map_off_by_one"]


@pytest.mark.parametrize("defect", DEFECTS)
def test_seeded_defect_is_rejected(defect):
    rows, census = _shadowed(model_entries(defect), CASES)
    failed = _failed(rows)
    print(f"\n{defect}: rejected on {len(failed)} / {len(rows)} cases: {failed}")
    with pytest.raises(AssertionError, match="window_attention"):
        census.assert_ok()
    assert failed
    if defect == "o_times_inv_l":
        # the multiply by a rounded 1 / l breaks ties at exactly these window sizes (and not at N = 49, 144, ...)
        n_of = {g["name"]: g["N"] for g in GEOMETRIES}
        assert {n_of[name] for _, kind, name in failed if kind == "ties"} >= {15, 52, 121}
