"""PiT throughput, its attention against the kernels it replaces, and the bandwidth of the pooling kernel.

    python tools/bench_pit.py [--models pit_ti_224,...] [--precisions bf16,tf32,fp32] [--batch 256]
                              [--warmup 3] [--iters 10] [--out DIR]

Models (224 x 224, random weights): one forward captured with ``cuda_graph`` per model and precision, ``--warmup``
replays, ``--iters`` replays timed with CUDA events -> images / s.

Attention, at batch --batch, at the stage-0 and stage-1 shapes of each model size (plain token counts), each timed with
CUDA events over ``--iters`` launches, in the same run:
  pit_attention_bf16   the new kernel on the packed bf16 qkv
  attention_f32        the fp32 SIMT kernel a bf16 model would otherwise fall back to (on the same values in fp32)
  sdpa_flash           torch.nn.functional.scaled_dot_product_attention, bf16, flash backend, on q, k, v already in
                       (B, H, T, dh) layout: the comparison only
  vit_attention_bf16   the ViT kernel, at the head-dim-64 shapes it also takes (pit_b stages 1 and 2, and T = 129 and 197
                       between them): pit_ops.vit_kernel_preferred is set from these rows
Each row also gives two lower bounds on the kernel's time from the H100 SXM data sheet figures: the tensor-core bound
(4 dh FLOPs per score at 989 TFLOP/s dense bf16) and the exponential bound (one MUFU ex2 per score at 16 per clock per
SM, 132 SMs, at the card's maximum SM clock).  They are bounds, not rates reached.

pit_pool at the stage-0 shapes of pit_ti and pit_b (one token row, the bf16 token copy on): bytes from the shapes
(pit_ops.pool_nbytes) over kernel time, against the 3.35 TB/s HBM3 figure of the data sheet.

The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line and writes it to
--out.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tensorflow-image-models_b200"))

import tfimm  # noqa: E402
import tfimm.architectures.pit  # noqa: E402,F401
from tfimm.backend import ops, pit_ops  # noqa: E402

HBM_TBPS = 3.35        # H100 SXM data sheet
BF16_TFLOPS = 989.0    # dense
SMS, EX2_PER_CLK_SM = 132, 16

NAMES = ["pit_ti_224", "pit_xs_224", "pit_s_224", "pit_b_224",
         "pit_ti_distilled_224", "pit_xs_distilled_224", "pit_s_distilled_224", "pit_b_distilled_224"]
# (label, T, H, dh)
ATTN_SHAPES = [("ti_s0", 730, 2, 32), ("ti_s1", 197, 4, 32), ("xs_s0", 730, 2, 48), ("xs_s1", 197, 4, 48),
               ("s_s0", 730, 3, 48), ("s_s1", 197, 6, 48), ("b_s0", 962, 4, 64), ("b_s1", 257, 8, 64),
               ("b_s2", 65, 16, 64), ("d64_t129", 129, 8, 64), ("d64_t197", 197, 8, 64)]


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
        for name in names:
            m = tfimm.create_model(name, precision=precision, device="cuda")
            x = torch.rand((batch, 224, 224, 3), device="cuda")
            run = m.cuda_graph(batch)
            ms = timed(lambda: run(x), warmup, iters)
            res.setdefault(precision, {})[name] = {"img_per_s": round(batch / ms * 1e3, 1), "step_ms": round(ms, 3)}
            print(precision, name, res[precision][name], flush=True)
            del m, run
            torch.cuda.empty_cache()
    return res


def bench_attention(batch, warmup, iters, sm_clock_mhz):
    from torch.nn.attention import SDPBackend, sdpa_kernel

    res = {}
    for label, T, H, dh in ATTN_SHAPES:
        B = batch
        scale = dh ** -0.5
        qkv = (torch.randn((B * T, 3 * H * dh), device="cuda")).to(torch.bfloat16)
        qkv32 = qkv.float()
        q, k, v = (t.contiguous() for t in qkv.view(B, T, 3, H, dh).permute(2, 0, 3, 1, 4))
        scores = float(B) * H * T * T
        row = {"B": B, "T": T, "H": H, "dh": dh}
        t_pit = timed(lambda: pit_ops.pit_attention_bf16(qkv, B, T, H, dh, scale), warmup, iters)
        t_f32 = timed(lambda: ops.attention(qkv32, B, T, H, dh, scale), 1, max(1, iters // 4))
        with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
            t_sdpa = timed(lambda: F.scaled_dot_product_attention(q, k, v, scale=scale), warmup, iters)
        row["pit_attention_bf16_us"] = round(t_pit * 1e3, 1)
        row["attention_f32_us"] = round(t_f32 * 1e3, 1)
        row["sdpa_flash_us"] = round(t_sdpa * 1e3, 1)
        if ops.attention_bf16_supported(T, dh):
            t_vit = timed(lambda: ops.attention(qkv, B, T, H, dh, scale), warmup, iters)
            row["vit_attention_bf16_us"] = round(t_vit * 1e3, 1)
        tensor_us = 4.0 * dh * scores / (BF16_TFLOPS * 1e12) * 1e6
        ex2_us = scores / (SMS * EX2_PER_CLK_SM * sm_clock_mhz * 1e6) * 1e6 if sm_clock_mhz else None
        row["tflops"] = round(4.0 * dh * scores / (t_pit * 1e-3) / 1e12, 1)
        row["bound_tensor_us"] = round(tensor_us, 1)
        row["bound_ex2_us"] = round(ex2_us, 1) if ex2_us else None
        row["speedup_vs_attention_f32"] = round(t_f32 / t_pit, 1)
        row["vs_sdpa_flash"] = round(t_sdpa / t_pit, 2)
        res[label] = row
        print(label, row, flush=True)
        del qkv, qkv32, q, k, v
        torch.cuda.empty_cache()
    return res


def bench_pool(batch, warmup, iters):
    res = {}
    for label, H, W, C in (("ti_s0", 27, 27, 64), ("b_s0", 31, 31, 256)):
        B, nb = batch, 1
        x = torch.randn((B * (nb + H * W), C), device="cuda")
        w = torch.randn((9, 2 * C), device="cuda")
        b = torch.randn((2 * C,), device="cuda")
        t = timed(lambda: pit_ops.pit_pool(x, w, b, B, nb, H, W, tokens_bf16=True), warmup, iters)
        nbytes = pit_ops.pool_nbytes(B, nb, H, W, C, True)
        res[label] = {"shape": [B, nb, H, W, C], "us": round(t * 1e3, 1), "gbytes": round(nbytes / 1e9, 4),
                      "tb_per_s": round(nbytes / t / 1e9, 3), "of_hbm": round(nbytes / t / 1e9 / HBM_TBPS, 3)}
        print(label, res[label], flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(NAMES))
    ap.add_argument("--precisions", default="bf16,tf32,fp32")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--skip-models", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pit needs a CUDA device")
    card = smi("name,power.limit,clocks.max.sm")
    try:
        sm_clock = float(card[2])
    except (TypeError, IndexError, ValueError):
        sm_clock = None
    res = {"card": card, "batch": args.batch}
    res["attention"] = bench_attention(args.batch, args.warmup, args.iters, sm_clock)
    res["pit_pool"] = bench_pool(args.batch, args.warmup, args.iters)
    if not args.skip_models:
        res["models"] = bench_models(args.models.split(","), args.precisions.split(","), args.batch, args.warmup,
                                     args.iters)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_pit.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
