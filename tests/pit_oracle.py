"""TEST INFRASTRUCTURE ONLY -- the PiT launchers (``tfimm.backend.pit_ops``) on top of oracle/emulate_bf16.py and
oracle/shadow.py.

Each launcher gets
* a statement at the kernels' storage points, in the emulation's arithmetic (float64 by default):
  - ``pit_attention_bf16``: the bf16 qkv as stored, softmax(scale q k^T) v with P rounded to bf16 per 64-key block
    of an online softmax (the emulation's attention), one rounding of the output to bf16;
  - ``pit_pool``: the reference's ConvHeadPooling on the grid rows -- reshape to (B, H, W, C), ZeroPadding2D(1), a
    VALID 3 x 3 / 2 Conv2D with groups = C (torch's grouped convolution: output channel o reads input o // 2), plus
    bias -- one rounding to fp32; and the token rows rounded to bf16 when asked.  The output's token rows belong to
    the token Dense that runs next: the statement leaves them NaN, so an orchestration that does not overwrite them
    shows.
* a derived error bound for the op-by-op shadow harness (``_rule_*``):
  - the attention: the bound of the ViT tensor-core kernel (``shadow._rule_attention``), the same algorithm: fp32
    scores accumulated in the tensor cores, fp32 online softmax over 64-key blocks with P rounded to bf16 per block
    against the running maximum, as the statement does (``shadow._blocked_softmax_err``), the output's own bf16
    rounding and the flip criterion;
  - the pool: nine fp32 fmas onto the bias, gamma_10 (|b| + sum |w| |x|); the bf16 token rows exactly.

``emulated_pit_ops()`` / ``shadowed_pit_ops()`` are ``emulated_ops()`` / ``shadowed_ops()`` with these launchers
added.
"""
from contextlib import contextmanager

import torch
import torch.nn.functional as F

from oracle import emulate_bf16 as emu
from oracle import shadow

_F64 = torch.float64


def pit_attention_bf16(qkv, B, T, H, dh, scale):
    return emu.attention(qkv, B, T, H, dh, scale)


def _grid_conv(x, w, bias, B, nb_tokens, H, W, dtype):
    """The grouped 3 x 3 / 2 convolution of the grid rows of x, (B, Ho * Wo, 2C) in dtype."""
    C = x.shape[1]
    grid = x.to(dtype).view(B, nb_tokens + H * W, C)[:, nb_tokens:].reshape(B, H, W, C).permute(0, 3, 1, 2)
    kernel = w.to(dtype).view(3, 3, 1, 2 * C).permute(3, 2, 0, 1)          # (2C, 1, 3, 3)
    y = F.conv2d(grid, kernel, bias.to(dtype), stride=2, padding=1, groups=C)
    return y.permute(0, 2, 3, 1).reshape(B, -1, 2 * C)


def pit_pool(x, w, bias, B, nb_tokens, H, W, tokens_bf16=False):
    C = x.shape[1]
    y = _grid_conv(x, w, bias, B, nb_tokens, H, W, emu._HP)
    out = torch.full((B, nb_tokens + y.shape[1], 2 * C), float("nan"), dtype=torch.float32, device=x.device)
    out[:, nb_tokens:] = y.to(torch.float32)
    tokens = None
    if tokens_bf16:
        tokens = x.view(B, -1, C)[:, :nb_tokens].reshape(B * nb_tokens, C).to(torch.bfloat16)
    return out.view(-1, 2 * C), tokens


# ------------------------------------------------------------------------------------------------------ the bounds
def _rule_pit_attention_bf16(A):
    return shadow._rule_attention(dict(qkv=A["qkv"], B=A["B"], N=A["T"], H=A["H"], dh=A["dh"], scale=A["scale"]))


def _grid_rows(B, nb_tokens):
    def get(s):
        out = s.ret[0]
        return out.view(B, -1, out.shape[1])[:, nb_tokens:]
    return get


def _rule_pit_pool(A):
    B, nb = A["B"], A["nb_tokens"]
    mag = _grid_conv(A["x"].abs(), A["w"].abs(), A["bias"].abs(), B, nb, A["H"], A["W"], _F64)
    outs = [("grid rows", _grid_rows(B, nb), shadow._bounded(shadow._gamma(10) * mag, flips=False))]
    if A["tokens_bf16"]:
        outs.append(("tokens_bf16", lambda s: s.ret[1], shadow._exact()))
    return outs


_PIT = {"pit_attention_bf16": (pit_attention_bf16, _rule_pit_attention_bf16),
        "pit_pool": (pit_pool, _rule_pit_pool)}


@contextmanager
def emulated_pit_ops(arithmetic=torch.float64):
    """``emulate_bf16.emulated_ops()`` plus the statements of the ``pit_ops`` launchers."""
    from tfimm.backend import pit_ops

    saved = {n: getattr(pit_ops, n) for n in _PIT}
    with emu.emulated_ops(arithmetic):
        for n, (f, _) in _PIT.items():
            setattr(pit_ops, n, f)
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(pit_ops, n, f)


@contextmanager
def shadowed_pit_ops():
    """``shadow.shadowed_ops()`` plus every ``pit_ops`` launcher checked against its statement within its bound; yields
    the shared ``Census``.  Whatever ``pit_ops.<name>`` is on entry is "the kernel"."""
    from tfimm.backend import pit_ops

    saved = {n: getattr(pit_ops, n) for n in _PIT}
    for n, (f, rule) in _PIT.items():
        setattr(emu, n, f)
        shadow._RULES[n] = rule
    try:
        with shadow.shadowed_ops() as census:
            for n in _PIT:
                setattr(pit_ops, n, shadow._shadow(n, saved[n], census))
            yield census
    finally:
        for n, f in saved.items():
            setattr(pit_ops, n, f)
            delattr(emu, n)
            del shadow._RULES[n]
