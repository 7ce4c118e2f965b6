"""ConvMixer throughput and the rate of its depthwise token-mixer kernel.

    python tools/bench_convmixer.py [--models convmixer_768_32,convmixer_1024_20_ks9_p14,convmixer_1536_20]
                                    [--batch 256] [--warmup 5] [--iters 20] [--repeats 2] [--out DIR]

For each model (bf16, 224 x 224): one forward captured with ``cuda_graph``, ``--warmup`` replays, ``--iters`` replays
timed with CUDA events -> images / s, ``--repeats`` times.  Then one eager forward under ``ops.trace`` -> kernel time
per family.  Then, at each model's block shape (B = --batch), each timed with CUDA events over ``--iters`` launches,
``--repeats`` times:
  convmixer_dwconv   the fused kernel (bf16 output, the model's activation)
  torch_eager        F.conv2d(groups=C) + act + affine + add in fp32 from torch's eager kernels, only as a comparison
FMAs are B H W C k^2, bytes the launcher's count (convmixer_ops.dwconv_nbytes); both over kernel time, against the H100
SXM data sheet's 67 TFLOP/s FP32 (33.5 T FMA/s) and 3.35 TB/s HBM3.  The larger of the two shares names the bound.
The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line, writes it to --out.
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
import tfimm.architectures.convmixer  # noqa: E402,F401
from tfimm.backend import convmixer_ops, ops  # noqa: E402

FP32_TFLOPS = 67.0   # H100 SXM data sheet, dense FP32
HBM_TBPS = 3.35      # H100 SXM data sheet


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


def kernel_rows(name, B, warmup, iters, repeats):
    cfg = tfimm.models.registry.model_config(name)
    C, k, act = cfg.embed_dim, cfg.kernel_size, cfg.act_layer
    H = W = 224 // cfg.patch_size[0]
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.relu(torch.randn((B, H, W, C), generator=g, device="cuda"))
    s_in, s1 = torch.rand(C, device="cuda") + 0.5, torch.rand(C, device="cuda") + 0.5
    t_in, bias, t1 = torch.randn(C, device="cuda"), torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    taps = torch.randn((k * k, C), device="cuda") / k
    wt = taps.t().reshape(C, 1, k, k).contiguous()
    act_fn = F.relu if act == "relu" else F.gelu

    def eager():
        x = (s_in * a + t_in).permute(0, 3, 1, 2)           # NCHW view of channels-last memory
        z = F.conv2d(x, wt, bias, padding=(k - 1) // 2, groups=C)
        return x + s1[:, None, None] * act_fn(z) + t1[:, None, None]

    fmas = float(B * H * W * C * k * k)
    nbytes = convmixer_ops.dwconv_nbytes(B, H, W, C, k, torch.bfloat16)
    t_k = [timed(lambda: convmixer_ops.dwconv(a, s_in, t_in, taps, bias, s1, t1, act, torch.bfloat16), warmup, iters)
           for _ in range(repeats)]
    t_e = [timed(eager, warmup, iters) for _ in range(repeats)]
    best = min(t_k)
    fma_share = fmas / (best * 1e-3) / (FP32_TFLOPS / 2 * 1e12)
    hbm_share = nbytes / (best * 1e-3) / (HBM_TBPS * 1e12)
    return {"shape": [B, H, W, C], "k": k, "act": act,
            "convmixer_dwconv_us": [round(t * 1e3, 1) for t in t_k],
            "tflops_fp32": round(2 * fmas / (best * 1e-3) / 1e12, 2), "of_fp32_peak": round(fma_share, 3),
            "tb_per_s": round(nbytes / (best * 1e-3) / 1e12, 3), "of_hbm": round(hbm_share, 3),
            "bound": "FP32 FMA" if fmas / (FP32_TFLOPS / 2 * 1e12) > nbytes / (HBM_TBPS * 1e12) else "HBM",
            "torch_eager_fp32_us": [round(t * 1e3, 1) for t in t_e],
            "speedup_vs_eager": round(min(t_e) / best, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="convmixer_768_32,convmixer_1024_20_ks9_p14,convmixer_1536_20")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_convmixer needs a CUDA device")
    res = {"card": smi("name,power.limit,clocks.max.sm"), "batch": args.batch, "models": {}, "kernel": {}}

    for name in args.models.split(","):
        m = tfimm.create_model(name, precision="bf16", device="cuda")
        x = torch.rand((args.batch, 224, 224, 3), device="cuda")
        run = m.cuda_graph(args.batch)
        ms = [timed(lambda: run(x), args.warmup, args.iters) for _ in range(args.repeats)]
        ops.trace = []
        m(x)
        torch.cuda.synchronize()
        fam = {}
        for f, e0, e1, _, nb in ops.trace:
            d = fam.setdefault(f, {"ms": 0.0, "launches": 0})
            d["ms"] += e0.elapsed_time(e1)
            d["launches"] += 1
        ops.trace = None
        res["models"][name] = {"img_per_s": [round(args.batch / t * 1e3, 1) for t in ms],
                               "step_ms": [round(t, 3) for t in ms],
                               "families_eager": {k: {"ms": round(v["ms"], 3), "launches": v["launches"]}
                                                  for k, v in sorted(fam.items(), key=lambda kv: -kv[1]["ms"])}}
        del m, run
        torch.cuda.empty_cache()
        res["kernel"][name] = kernel_rows(name, args.batch, args.warmup, args.iters, args.repeats)
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_convmixer.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
