"""PVT v2 on the GPU: the fused ConvFFN against the three unfused launches (fc1 GEMM, dwconv_bias_act, fc2 GEMM) at
every stage-0 / 1 shape of the family at batch 256, with the HBM byte floor of each, and bf16 throughput of the six
models at batch 256 (CUDA graph).  Prints one line per measurement; medians of CUDA-event timings.

    python tools/bench_pvt_v2.py [--batch 256] [--reps 20]
"""
import argparse
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tensorflow-image-models_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

# (gh, gw, C, hidden): stages 0 / 1 of b0, of b1-b4 (mlp_ratio 8) and of b5 (mlp_ratio 4)
SHAPES = [(56, 56, 32, 256), (28, 28, 64, 512), (56, 56, 64, 512), (28, 28, 128, 1024), (56, 56, 64, 256),
          (28, 28, 128, 512)]
HBM = 3.35e12   # H100 SXM HBM3 bytes / s


def _time(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    fn()
    torch.cuda.synchronize()
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ev) * 1e-3


def bench_conv_mlp(B, reps):
    from tfimm.backend import ops, pvt_v2_ops

    for gh, gw, C, hidden in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        M = B * gh * gw
        h = torch.randn((M, C), device="cuda", generator=g).to(torch.bfloat16)
        w1 = (torch.randn((hidden, C), device="cuda", generator=g) * C ** -0.5).to(torch.bfloat16)
        w2 = (torch.randn((C, hidden), device="cuda", generator=g) * hidden ** -0.5).to(torch.bfloat16)
        b1, bdw = torch.randn(hidden, device="cuda"), torch.randn(hidden, device="cuda")
        wdw, b2 = torch.randn((9, hidden), device="cuda") / 3, torch.randn(C, device="cuda")
        res = torch.randn((M, C), device="cuda")

        def fused():
            pvt_v2_ops.pvt_v2_conv_mlp_bf16(h, w1, b1, wdw, bdw, w2, b2, res, B, gh, gw, "gelu", out=res)

        def unfused():
            hid = ops.gemm(h, w1, bias=b1)
            hid = ops.dwconv_bias_act(hid.view(B, gh, gw, hidden), wdw, bdw, 3, 1, "symmetric", act="gelu")
            ops.gemm(hid.view(M, hidden), w2, bias=b2, residual=res, out=res)

        tf, tu = _time(fused, reps), _time(unfused, reps)
        ff = pvt_v2_ops.conv_mlp_nbytes(B, gh, gw, C, hidden) / HBM
        fu = pvt_v2_ops.unfused_conv_mlp_nbytes(B, gh, gw, C, hidden) / HBM
        print(f"CONV_MLP B={B} {gh}x{gw} C={C} hidden={hidden}: fused {tf * 1e6:8.1f} us (byte floor {ff * 1e6:7.1f}) "
              f"| unfused {tu * 1e6:8.1f} us (byte floor {fu * 1e6:7.1f}) | speedup {tu / tf:.2f}x", flush=True)


def bench_models(B, reps):
    import tfimm
    import tfimm.architectures.pvt_v2  # noqa: F401

    for name in tfimm.list_models(module="pvt_v2"):
        m = tfimm.create_model(name, precision="bf16", device="cuda")
        run = m.cuda_graph(B)
        x = torch.rand((B, *m.cfg.input_size, 3), device="cuda")
        t = _time(lambda: run(x), reps)
        print(f"MODEL {name} bf16 B={B}: {t * 1e3:8.2f} ms/step, {B / t:8.0f} img/s", flush=True)
        del run, m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(f"CARD {q}", flush=True)
    bench_conv_mlp(args.batch, args.reps)
    bench_models(args.batch, args.reps)
