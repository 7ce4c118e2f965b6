"""CaiT throughput, and its talking-heads kernel against the unfused torch chain and its data-sheet bounds.

    python tools/bench_cait.py [--models cait_xxs24_224,...] [--precisions bf16,tf32,fp32] [--batch 256]
                               [--warmup 3] [--iters 10] [--skip-models] [--skip-attention] [--out DIR]

Models (their own input size, random weights): one forward captured with ``cuda_graph`` per model and precision,
``--warmup`` replays, ``--iters`` replays timed with CUDA events -> images / s.  fp32 and tf32 take one warm-up and
``max(1, iters // 4)`` timed replays.

Talking-heads attention at batch --batch at each family shape (H, N), each timed with CUDA events over ``--iters``
launches in the same run:
  talking_heads_bf16   the fused two-pass kernel on the packed bf16 qkv
  talking_heads_f32    the fp32 SIMT kernel on the same values in fp32
  torch_chain_bf16     the unfused chain in bf16: q k^T (matmul), einsum mix over heads, softmax, einsum mix, P V
                       (matmul), chunked over the batch so that the (b, H, N, N) logits fit; the comparison only
and three lower bounds per (query, key) pair from the H100 SXM data sheet: the tensor cores (3 D MACs: q k^T twice,
P V once, at 989 TFLOP/s dense bf16), the CUDA cores (2 H^2 FMAs of the two mixes at 67 TFLOP/s fp32) and the MUFU
(2 H ex2 at 16 per clock per SM, 132 SMs, at the card's maximum SM clock).  They are bounds, not rates reached.

The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line and writes it to
--out.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tensorflow-image-models_b200"))

import tfimm  # noqa: E402
import tfimm.architectures.cait  # noqa: E402,F401
from tfimm.backend import cait_ops  # noqa: E402

BF16_TFLOPS, FP32_TFLOPS = 989.0, 67.0   # dense, H100 SXM data sheet
SMS, EX2_PER_CLK_SM = 132, 16

NAMES = ["cait_xxs24_224", "cait_xxs24_384", "cait_xxs36_224", "cait_xxs36_384", "cait_xs24_384", "cait_s24_224",
         "cait_s24_384", "cait_s36_384", "cait_m36_384", "cait_m48_448"]
# (label, H, N): every (heads, tokens) pair of the family
SHAPES = [("xxs_224", 4, 196), ("xxs_384", 4, 576), ("xs_384", 6, 576), ("s_224", 8, 196), ("s_384", 8, 576),
          ("m_384", 16, 576), ("m_448", 16, 784)]


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", f"--query-gpu={fields}",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        return [v.strip() for v in out.strip().split(",")]
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_models(names, precisions, batch, warmup, iters):
    res = {}
    for precision in precisions:
        w, it = (warmup, iters) if precision == "bf16" else (1, max(1, iters // 4))
        for name in names:
            m = tfimm.create_model(name, precision=precision, device="cuda")
            x = torch.rand((batch, *m.cfg.input_size, 3), device="cuda")
            run = m.cuda_graph(batch)
            ms = timed(lambda: run(x), w, it)
            res.setdefault(precision, {})[name] = {"img_per_s": round(batch / ms * 1e3, 1), "step_ms": round(ms, 3)}
            print(precision, name, res[precision][name], flush=True)
            del m, run, x
            torch.cuda.empty_cache()
    return res


def torch_chain(qkv, wl, bl, ww, bw, B, N, H, dh, chunk):
    """The unfused bf16 chain, ``chunk`` images at a time."""
    out = torch.empty((B, N, H * dh), device=qkv.device, dtype=torch.bfloat16)
    x = qkv.view(B, N, 3, H, dh)
    wlb, blb, wwb, bwb = (t.to(torch.bfloat16) for t in (wl, bl, ww, bw))
    for s in range(0, B, chunk):
        q, k, v = x[s:s + chunk].permute(2, 0, 3, 1, 4)
        a = torch.einsum("bhqk,hg->bgqk", q @ k.transpose(-1, -2), wlb) + blb[:, None, None]
        a = torch.softmax(a, dim=-1)
        a = torch.einsum("bgqk,gf->bfqk", a, wwb) + bwb[:, None, None]
        out[s:s + chunk] = (a @ v).permute(0, 2, 1, 3).reshape(-1, N, H * dh)
    return out


def bench_attention(batch, warmup, iters, sm_clock_mhz):
    res = {}
    for label, H, N in SHAPES:
        B, dh = batch, 48
        D = H * dh
        qkv = torch.randn((B * N, 3 * D), device="cuda").to(torch.bfloat16)
        qkv32 = qkv.float()
        wl, ww = torch.randn((H, H), device="cuda") * 0.3, torch.randn((H, H), device="cuda") * 0.3
        bl, bw = torch.randn((H,), device="cuda"), torch.randn((H,), device="cuda")
        pairs = float(B) * N * N
        chunk = max(1, int(2 ** 31 // (H * N * N * 2 * 4)))   # ~2 GB of bf16 logits per chunk, four live copies
        row = {"B": B, "H": H, "N": N, "dh": dh}
        t_bf16 = timed(lambda: cait_ops.talking_heads_bf16(qkv, wl, bl, ww, bw, B, N, H, dh), warmup, iters)
        t_f32 = timed(lambda: cait_ops.talking_heads_f32(qkv32, wl, bl, ww, bw, B, N, H, dh), 1, max(1, iters // 4))
        t_chain = timed(lambda: torch_chain(qkv, wl, bl, ww, bw, B, N, H, dh, chunk), 1, max(1, iters // 2))
        row["talking_heads_bf16_us"] = round(t_bf16 * 1e3, 1)
        row["talking_heads_f32_us"] = round(t_f32 * 1e3, 1)
        row["torch_chain_bf16_us"] = round(t_chain * 1e3, 1)
        row["chain_chunk"] = min(chunk, B)
        row["bound_tensor_us"] = round(2.0 * 3 * D * pairs / (BF16_TFLOPS * 1e12) * 1e6, 1)
        row["bound_mix_fma_us"] = round(2.0 * 2 * H * H * pairs / (FP32_TFLOPS * 1e12) * 1e6, 1)
        row["bound_ex2_us"] = (round(2 * H * pairs / (SMS * EX2_PER_CLK_SM * sm_clock_mhz * 1e6) * 1e6, 1)
                               if sm_clock_mhz else None)
        bounds = {k: row[k] for k in ("bound_tensor_us", "bound_mix_fma_us", "bound_ex2_us") if row[k]}
        row["nearest_bound"] = max(bounds, key=bounds.get)
        row["x_nearest_bound"] = round(row["talking_heads_bf16_us"] / bounds[row["nearest_bound"]], 2)
        row["speedup_vs_torch_chain"] = round(t_chain / t_bf16, 2)
        res[label] = row
        print(label, row, flush=True)
        del qkv, qkv32
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(NAMES))
    ap.add_argument("--precisions", default="bf16,tf32,fp32")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--skip-models", action="store_true")
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cait needs a CUDA device")
    card = smi("name,power.limit,clocks.max.sm")
    try:
        sm_clock = float(card[2])
    except (TypeError, IndexError, ValueError):
        sm_clock = None
    res = {"card": card, "batch": args.batch}
    if not args.skip_attention:
        res["talking_heads"] = bench_attention(args.batch, args.warmup, args.iters, sm_clock)
    if not args.skip_models:
        res["models"] = bench_models(args.models.split(","), args.precisions.split(","), args.batch, args.warmup,
                                     args.iters)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_cait.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
