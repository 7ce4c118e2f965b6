"""GEMM micro-benchmark.

    python tools/bench_gemm.py M N K [act] [out=bf16|f32] [res=0|1] [block_n]
    python tools/bench_gemm.py vit [block_n ...]

The first form times one shape.  The second times the four GEMMs of a vit_base_patch16_224 block at the benchmark's
batch (M = 256 x 197 rows) with their real epilogues, once per listed block_n (default: 0 = the library's choice, 64,
128, 256), and prints the card, its power limit and its SM clock first.  Times are device time per launch (CUDA events
around back-to-back launches after warm-up); TFLOP/s counts 2 M N K.  The "ran" column is the tile width of the kernel
that actually ran, read from its name in a separate profiled launch."""
import re
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tensorflow-image-models_b200"))

from tfimm.backend import ops  # noqa: E402

# name, N, K, act, fp32 residual updated in place (else bf16 out)
VIT_B = [("qkv", 2304, 768, None, False), ("proj", 768, 768, None, True),
         ("fc1", 3072, 768, "gelu", False), ("fc2", 768, 3072, None, True)]
VIT_B_ROWS = 256 * 197
USAGE = __doc__.split("\n\n")[1]


def make_gemm(M, N, K, act, out_dtype, res, block_n):
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g).to(out_dtype)
    if res:
        return lambda: ops.gemm(a, w, bias=bias, act=act, residual=x, out=x, block_n=block_n)
    return lambda: ops.gemm(a, w, bias=bias, act=act, out=x, block_n=block_n)


def time_launches(fn, reps=20):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def width_that_ran(fn):
    """BLOCK_N of the gemm_wgmma_kernel instance one launch of fn runs (its template argument, from the kernel name)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    for e in prof.events():
        m = re.search(r"gemm_wgmma_kernel(?:<|ILi)(\d+)", e.name)
        if m:
            return int(m.group(1))
    return None


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                        "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def vit(block_ns):
    print(f"card (name, power limit, max / current SM clock): {card()}")
    print(f"{'gemm':5s} {'M':>6s} {'N':>5s} {'K':>5s} {'epilogue':29s} {'block_n':>7s} {'ran':>4s} {'us':>8s} "
          f"{'TFLOP/s':>8s}")
    for name, N, K, act, res in VIT_B:
        epi = "bias" + (", gelu" if act else "") + (", fp32 residual in place" if res else ", bf16 out")
        for bn in block_ns:
            fn = make_gemm(VIT_B_ROWS, N, K, act, torch.float32 if res else torch.bfloat16, res, bn)
            us = time_launches(fn, reps=50)
            ran = width_that_ran(fn)
            tf = 2.0 * VIT_B_ROWS * N * K / us * 1e-6
            print(f"{name:5s} {VIT_B_ROWS:6d} {N:5d} {K:5d} {epi:29s} {bn:7d} {ran!s:>4s} {us:8.1f} {tf:8.0f}")


def main():
    if len(sys.argv) < 2 or (sys.argv[1] != "vit" and len(sys.argv) < 4):
        sys.exit(USAGE)
    if sys.argv[1] == "vit":
        vit([int(v) for v in sys.argv[2:]] or [0, 64, 128, 256])
        return
    M, N, K = (int(v) for v in sys.argv[1:4])
    act = sys.argv[4] if len(sys.argv) > 4 and sys.argv[4] != "none" else None
    out_dtype = torch.float32 if len(sys.argv) > 5 and sys.argv[5] == "f32" else torch.bfloat16
    res = len(sys.argv) > 6 and sys.argv[6] == "1"
    block_n = int(sys.argv[7]) if len(sys.argv) > 7 else 0
    fn = make_gemm(M, N, K, act, out_dtype, res, block_n)
    us = time_launches(fn)
    print(f"gemm M={M} N={N} K={K} act={act} out={str(out_dtype)[6:]} res={int(res)} block_n={block_n} "
          f"(ran {width_that_ran(fn)}): {us:.1f} us  {2.0 * M * N * K / us * 1e-6:.0f} TFLOP/s")


if __name__ == "__main__":
    main()
