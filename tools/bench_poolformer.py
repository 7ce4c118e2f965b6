"""PoolFormer throughput and the bandwidth of its GroupNorm / token-mixer kernels.

    python tools/bench_poolformer.py [--models poolformer_s12,poolformer_s36,poolformer_m48] [--batch 256]
                                     [--warmup 5] [--iters 20] [--out DIR]

For each model (bf16, 224 x 224): one forward captured with ``cuda_graph``, ``--warmup`` replays, ``--iters`` replays
timed with CUDA events -> images / s.  Then one eager forward under ``ops.trace`` -> kernel time per family.  Then, at
poolformer_s12's stage-0 shape (56 x 56 x 64 at --batch), each timed with CUDA events over ``--iters`` launches:
  poolformer_mixer   the fused token mixer (x + ls1 gamma rstd mean_j (x_j - x), and its output's partials)
  gn1_apply_bf16     GN(x) -> the bf16 fc1 operand
  torch_eager        F.group_norm(x, 1) -> avg_pool2d(3, 1, 1, count_include_pad=False) -> sub, scale, add: the same
                     mixer from torch's eager kernels, only as the comparison
Bytes are the shape-derived counts the launchers pass to ``nbytes`` (poolformer_ops.mixer_nbytes / apply_nbytes) over
kernel time, against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet: the kernels are bandwidth-bound.  The card's
name, power limit and SM clock are read in the same run.  Prints one JSON line and writes it to --out.
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
import tfimm.architectures.poolformer  # noqa: E402,F401
from tfimm.backend import ops, poolformer_ops  # noqa: E402

HBM_TBPS = 3.35   # H100 SXM data sheet


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="poolformer_s12,poolformer_s36,poolformer_m48")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_poolformer needs a CUDA device")
    res = {"card": smi("name,power.limit,clocks.max.sm"), "batch": args.batch, "models": {}}

    for name in args.models.split(","):
        m = tfimm.create_model(name, precision="bf16", device="cuda")
        x = torch.rand((args.batch, 224, 224, 3), device="cuda")
        run = m.cuda_graph(args.batch)
        ms = timed(lambda: run(x), args.warmup, args.iters)
        ops.trace = []
        m(x)
        torch.cuda.synchronize()
        fam = {}
        for f, e0, e1, _, nb in ops.trace:
            d = fam.setdefault(f, {"ms": 0.0, "launches": 0, "gbytes": 0.0})
            d["ms"] += e0.elapsed_time(e1)
            d["launches"] += 1
            d["gbytes"] += nb / 1e9
        ops.trace = None
        res["models"][name] = {"img_per_s": round(args.batch / ms * 1e3, 1), "step_ms": round(ms, 3),
                               "families_eager": {k: {"ms": round(v["ms"], 3), "launches": v["launches"],
                                                      "gbytes": round(v["gbytes"], 3)}
                                                  for k, v in sorted(fam.items(), key=lambda kv: -kv[1]["ms"])}}
        del m, run
        torch.cuda.empty_cache()

    B, H, W, C = args.batch, 56, 56, 64
    x = torch.randn((B, H, W, C), device="cuda")
    gamma, beta, ls1 = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda"), torch.rand(C, device="cuda")
    p = poolformer_ops.gn1_partials(x)
    t_mix = timed(lambda: poolformer_ops.poolformer_mixer(x, p, gamma, beta, ls1, 1e-5), args.warmup, args.iters)
    t_app = timed(lambda: poolformer_ops.gn1_apply(x, p, gamma, beta, 1e-5, torch.bfloat16), args.warmup, args.iters)
    t_par = timed(lambda: poolformer_ops.gn1_partials(x), args.warmup, args.iters)

    xc = x.permute(0, 3, 1, 2)   # the same memory seen as NCHW (channels_last strides)

    def eager():
        n = F.group_norm(xc, 1, gamma, beta, 1e-5)
        return xc + ls1[:, None, None] * (F.avg_pool2d(n, 3, 1, 1, count_include_pad=False) - n)

    t_eager = timed(eager, args.warmup, args.iters)
    mix_b = poolformer_ops.mixer_nbytes(B, H, W, C)
    app_b = poolformer_ops.apply_nbytes(B, H, W, C, torch.bfloat16)
    par_b = 4.0 * B * H * W * C
    res["kernels_s12_stage0"] = {
        "shape": [B, H, W, C],
        "poolformer_mixer": {"us": round(t_mix * 1e3, 1), "gbytes": round(mix_b / 1e9, 4),
                             "tb_per_s": round(mix_b / t_mix / 1e9, 3), "of_hbm": round(mix_b / t_mix / 1e9 / HBM_TBPS, 3)},
        "gn1_apply_bf16": {"us": round(t_app * 1e3, 1), "gbytes": round(app_b / 1e9, 4),
                           "tb_per_s": round(app_b / t_app / 1e9, 3), "of_hbm": round(app_b / t_app / 1e9 / HBM_TBPS, 3)},
        "gn1_partials": {"us": round(t_par * 1e3, 1), "tb_per_s": round(par_b / t_par / 1e9, 3)},
        "torch_eager_mixer": {"us": round(t_eager * 1e3, 1), "speedup_of_poolformer_mixer": round(t_eager / t_mix, 2)},
        "bound": "HBM bandwidth: bytes from the shapes over 3.35 TB/s (data sheet)",
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_poolformer.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
