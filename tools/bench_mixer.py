"""MLP-Mixer family throughput and the token-mixing GEMM's tensor-core throughput.

    python tools/bench_mixer.py [--models mixer_b16_224,resmlp_24_224,gmlp_s16_224] [--batch 256] [--warmup 5]
                                [--iters 20] [--out DIR]

For each model (bf16, 224 x 224): one forward captured with ``cuda_graph``, ``--warmup`` replays, ``--iters`` replays
timed with CUDA events -> images / s.  Then the token-mixing contraction at Mixer-B/16 shapes (196 tokens, 768 channels,
token hidden 384) three ways, each timed with CUDA events over ``--iters`` launches:
  token_gemm       mixer_ops.token_gemm, X read where it is stored (MN-major wgmma operand)
  transpose_gemm   a transpose copy of X (torch), ops.gemm, a transpose copy back (torch) -- the same contraction built
                   from the engine's row-major GEMM; the copies are torch's and only serve as the comparison
with FLOPs computed here from the shapes (2 B M K C) against the 989 TFLOP/s dense bf16 peak of the H100 SXM data sheet.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON line and writes it to --out.
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
import tfimm.architectures.mlp_mixer  # noqa: E402,F401
from tfimm.backend import mixer_ops, ops  # noqa: E402

BF16_PEAK_TFLOPS = 989.0   # H100 SXM data sheet, dense


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
    ap.add_argument("--models", default="mixer_b16_224,resmlp_24_224,gmlp_s16_224")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mixer.py needs a CUDA device")
    res = {"gpu": torch.cuda.get_device_name(), "batch": a.batch, "models": {}, "token_mixing": {}}
    for name in a.models.split(","):
        m = tfimm.create_model(name, precision="bf16", device="cuda")
        x = torch.rand((a.batch, *m.cfg.input_size, 3), device="cuda")
        run = m.cuda_graph(a.batch)
        ms = timed(lambda: run(x), a.warmup, a.iters)
        res["models"][name] = {"ms_per_batch": round(ms, 3), "img_per_s": round(a.batch * 1e3 / ms, 1)}
        print(f"{name}: {a.batch * 1e3 / ms:.0f} img/s (bf16, batch {a.batch}, cuda_graph)", flush=True)
        del m, run
    B, N, C, Ht = a.batch, 196, 768, 384
    g = torch.Generator(device="cuda").manual_seed(0)
    for label, M, K in (("fc1", Ht, N), ("fc2", N, Ht)):
        x = torch.randn((B, K, C), generator=g, device="cuda").to(torch.bfloat16)
        wt = torch.randn((M, (K + 7) // 8 * 8), generator=g, device="cuda").to(torch.bfloat16)
        w = wt[:, :K].contiguous() if K % 8 == 0 else torch.nn.functional.pad(wt[:, :K], (0, (-K) % 8))
        bias = torch.randn(M, generator=g, device="cuda")
        flops = 2.0 * B * M * K * C

        def token():
            mixer_ops.token_gemm(wt[:, :K], x, bias=bias)

        def transposed():
            xt = x.transpose(1, 2).reshape(B * C, K)
            if K % 8:
                xt = torch.nn.functional.pad(xt, (0, (-K) % 8))
            y = ops.gemm(xt.contiguous(), w, bias=bias)
            return y.view(B, C, M).transpose(1, 2).contiguous()

        ref = transposed().float()
        out = mixer_ops.token_gemm(wt[:, :K], x, bias=bias).float()
        diff = ((out - ref).abs().max() / ref.abs().max()).item()
        t_tok = timed(token, a.warmup, a.iters)
        t_tr = timed(transposed, a.warmup, a.iters)
        res["token_mixing"][label] = {
            "shape": {"B": B, "M": M, "K": K, "C": C},
            "token_gemm_ms": round(t_tok, 4), "token_gemm_tflops": round(flops / t_tok / 1e9, 1),
            "transpose_gemm_ms": round(t_tr, 4), "transpose_gemm_tflops": round(flops / t_tr / 1e9, 1),
            "token_gemm_share_of_bf16_peak": round(flops / t_tok / 1e9 / BF16_PEAK_TFLOPS, 3),
            "max_rel_diff_vs_transpose_path": diff,
        }
        print(label, res["token_mixing"][label], flush=True)
    info = smi("name,power.limit,clocks.sm,clocks.max.sm")
    res["card"] = info
    print(json.dumps(res))
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "bench_mixer.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
