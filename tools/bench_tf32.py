"""bf16 / tf32 / fp32 throughput of the benchmark models, and the TF32 GEMM's tensor-core throughput.

    python tools/bench_tf32.py [--batch 256] [--warmup 3] [--iters 10] [--models vit_base_patch16_224,...]

For each model and precision: one forward of the given batch captured with ``model.cuda_graph``, ``--warmup`` replays,
then ``--iters`` replays timed with CUDA events -> images / s.  Then the TF32 GEMM alone at the ViT-B/16 shapes of batch
256 (M = 256 * 197 = 50432 tokens: qkv, proj, fc1, fc2) -> TFLOP/s and its share of the H100 SXM data-sheet TF32 peak
(495 dense TFLOP/s).  The card's name and power limit are read in the same run and printed with the numbers: they are
part of them.  Prints one JSON line at the end.
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
from tfimm.backend import lib, ops  # noqa: E402

MODELS = ["vit_base_patch16_224", "convnext_base", "swin_base_patch4_window7_224", "efficientnet_b4"]
TF32_PEAK_TFLOPS = 495.0   # H100 SXM data sheet, dense
VIT_B_SHAPES = [(50432, 2304, 768), (50432, 768, 768), (50432, 3072, 768), (50432, 768, 3072)]


def card():
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        idx = torch.cuda.current_device()
        out = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return info


def _time(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters   # ms


def model_throughput(name, precision, batch, warmup, iters):
    """(images / s, batch used).  A precision whose kernels refuse the batch (the fp32 SIMT GEMM's grid is limited to
    65535 row tiles: EfficientNet-B4's 190 x 190 maps at batch 256 exceed it) is measured at the largest halved batch
    that runs."""
    model = tfimm.create_model(name, precision=precision, device="cuda")   # native input size (B4: 380 px)
    h, w = model.cfg.input_size
    while True:
        x = torch.rand(batch, h, w, model.cfg.in_channels, device="cuda",
                       generator=torch.Generator("cuda").manual_seed(0))
        try:
            fwd = model.cuda_graph(batch)
            break
        except lib.KernelLibraryError as e:
            if batch == 1:
                raise
            print(f"  {name} {precision} batch {batch}: {e}; halving the batch")
            torch.cuda.synchronize()
            batch //= 2
    ms = _time(lambda: fwd(x), warmup, iters)
    del fwd, model
    torch.cuda.empty_cache()
    return batch / (ms * 1e-3), batch


def gemm_tf32_tflops(M, N, K, warmup, iters):
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = lib.round_tf32(torch.randn(N, K, device="cuda", generator=g) / K ** 0.5)
    bias = torch.randn(N, device="cuda", generator=g)
    out = torch.empty(M, N, device="cuda")
    token = lib.tf32_mode.set(True)
    try:
        ms = _time(lambda: ops.gemm(a, w, bias=bias, out=out), warmup, iters)
    finally:
        lib.tf32_mode.reset(token)
    return 2.0 * M * N * K / (ms * 1e-3) * 1e-12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--models", default=",".join(MODELS))
    args = ap.parse_args()
    dev = card()
    print(f"card: {dev['name']}, power limit {dev['power_limit_w']} W")
    res = {"card": dev, "batch": args.batch, "img_per_s": {}, "gemm_tf32": []}
    for name in args.models.split(","):
        runs = {p: model_throughput(name, p, args.batch, args.warmup, args.iters) for p in ("bf16", "tf32", "fp32")}
        row = {p: r[0] for p, r in runs.items()}
        res["img_per_s"][name] = row
        res.setdefault("batch_used", {})[name] = {p: r[1] for p, r in runs.items()}
        print(f"{name:32s} img/s  bf16 {row['bf16']:8.0f}  tf32 {row['tf32']:8.0f}  fp32 {row['fp32']:8.0f}  "
              f"tf32/fp32 {row['tf32'] / row['fp32']:.2f}x  tf32/bf16 {row['tf32'] / row['bf16']:.2f}x  "
              f"(batch {'/'.join(str(r[1]) for r in runs.values())})")
    for M, N, K in VIT_B_SHAPES:
        t = gemm_tf32_tflops(M, N, K, args.warmup, 4 * args.iters)
        res["gemm_tf32"].append({"M": M, "N": N, "K": K, "tflops": t, "share_of_peak": t / TF32_PEAK_TFLOPS})
        print(f"gemm_tf32 M={M} N={N} K={K}: {t:6.1f} TFLOP/s = {100 * t / TF32_PEAK_TFLOPS:.1f} % of "
              f"{TF32_PEAK_TFLOPS:.0f}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
