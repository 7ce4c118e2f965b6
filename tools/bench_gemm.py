"""GEMM micro-benchmark.

    python tools/bench_gemm.py M N K [act] [out=bf16|f32] [res=0|1] [block_n]
    python tools/bench_gemm.py vit|convnext|swin [block_n ...]

The first form times one shape.  The second times the GEMMs of one block of a model at the benchmark's batch (256
images at 224 px) with their epilogues, once per listed block_n (default: 0 = the library's choice, 64, 128, 256, and
1 = the persistent 128 x 256 kernel), and prints the card, its power limit and its SM clock first.
  vit       the four GEMMs of a vit_base_patch16_224 block (M = 256 x 197 rows), with their real epilogues
  convnext  fc1 / fc2 of convnext_base's stage 3 (C = 512, 14 x 14) and stage 4 (C = 1024, 7 x 7): GELU, and
            layer scale + fp32 residual in place
  swin      qkv / proj of swin_base_patch4_window7_224's four stages (its fc1 / fc2 have convnext's shapes in stages 3
            and 4, and run in the fused MLP kernel in stages 1 and 2), with ViT's epilogues
Times are device time per launch (CUDA events around back-to-back launches after warm-up).  TFLOP/s counts 2 M N K;
GB/s counts the bytes the GEMM must move at least once: A, W, the output, and the residual when there is one.  The two
floors are those counts over the H100 SXM data-sheet rates (989 TFLOP/s dense bf16, 3.35 TB/s HBM3): bounds, not
measurements.  The "ran" column is the tile width of the kernel that actually ran, read from its name in a separate
profiled launch ("p256": the persistent 128 x 256 kernel, block_n 1).  "L2->SM" is the operand traffic that kernel pulls
into shared memory: every 128 x BN tile loads (128 + BN) x K bf16 elements of A and W, counted over all tiles and divided
by the time."""
import re
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tensorflow-image-models_b200"))

from tfimm.backend import ops  # noqa: E402

PEAK_BF16_FLOPS = 989e12
PEAK_HBM_BYTES = 3.35e12

# name, M, N, K, act, layer scale (gamma), fp32 residual updated in place (else bf16 out)
_VIT_M = 256 * 197
_S1, _S2, _S3, _S4 = 256 * 56 * 56, 256 * 28 * 28, 256 * 14 * 14, 256 * 7 * 7
SHAPES = {
    "vit": [("qkv", _VIT_M, 2304, 768, None, False, False), ("proj", _VIT_M, 768, 768, None, False, True),
            ("fc1", _VIT_M, 3072, 768, "gelu", False, False), ("fc2", _VIT_M, 768, 3072, None, False, True)],
    "convnext": [("s3.fc1", _S3, 2048, 512, "gelu", False, False), ("s3.fc2", _S3, 512, 2048, None, True, True),
                 ("s4.fc1", _S4, 4096, 1024, "gelu", False, False), ("s4.fc2", _S4, 1024, 4096, None, True, True)],
    "swin": [("s1.qkv", _S1, 384, 128, None, False, False), ("s1.proj", _S1, 128, 128, None, False, True),
             ("s2.qkv", _S2, 768, 256, None, False, False), ("s2.proj", _S2, 256, 256, None, False, True),
             ("s3.qkv", _S3, 1536, 512, None, False, False), ("s3.proj", _S3, 512, 512, None, False, True),
             ("s4.qkv", _S4, 3072, 1024, None, False, False), ("s4.proj", _S4, 1024, 1024, None, False, True)],
}
USAGE = __doc__.split("\n\n")[1]


def make_gemm(M, N, K, act, out_dtype, res, block_n, with_gamma=False):
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g) if with_gamma else None
    x = torch.randn(M, N, device="cuda", generator=g).to(out_dtype)
    if res:
        return lambda: ops.gemm(a, w, bias=bias, act=act, gamma=gamma, residual=x, out=x, block_n=block_n)
    return lambda: ops.gemm(a, w, bias=bias, act=act, gamma=gamma, out=x, block_n=block_n)


def min_bytes(M, N, K, out_bytes, res):
    return 2 * (M * K + N * K) + M * N * out_bytes * (2 if res else 1)


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
    """BLOCK_N of the GEMM kernel one launch of fn runs, from the kernel name: the template argument of a
    gemm_wgmma_kernel instance, or "p256" for gemm_persistent_kernel."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    for e in prof.events():
        if "gemm_persistent_kernel" in e.name:
            return "p256"
        m = re.search(r"gemm_wgmma_kernel(?:<|ILi)(\d+)", e.name)
        if m:
            return int(m.group(1))
    return None


def l2_to_sm(M, N, K, ran, us):
    """Operand bytes the kernel that ran loads from L2 into shared memory, over its time, in TB/s ("-" if unknown)."""
    if ran is None:
        return "-"
    bn = 256 if ran == "p256" else ran
    tiles = -(-M // 128) * -(-N // bn)
    return f"{tiles * (128 + bn) * K * 2 / us * 1e-6:.1f}"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                        "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def table(family, block_ns):
    print(f"card (name, power limit, max / current SM clock): {card()}")
    print(f"{'gemm':7s} {'M':>6s} {'N':>5s} {'K':>5s} {'epilogue':37s} {'block_n':>7s} {'ran':>4s} {'us':>8s} "
          f"{'TFLOP/s':>8s} {'GB/s':>6s} {'L2->SM TB/s':>11s} {'floor flop us':>13s} {'floor HBM us':>12s}")
    for name, M, N, K, act, with_gamma, res in SHAPES[family]:
        epi = ("bias" + (", gelu" if act else "") + (", gamma" if with_gamma else "")
               + (", fp32 residual in place" if res else ", bf16 out"))
        flops, nbytes = 2.0 * M * N * K, min_bytes(M, N, K, 4 if res else 2, res)
        for bn in block_ns:
            fn = make_gemm(M, N, K, act, torch.float32 if res else torch.bfloat16, res, bn, with_gamma)
            us = time_launches(fn, reps=50)
            ran = width_that_ran(fn)
            print(f"{name:7s} {M:6d} {N:5d} {K:5d} {epi:37s} {bn:7d} {ran!s:>4s} {us:8.1f} {flops / us * 1e-6:8.0f} "
                  f"{nbytes / us * 1e-3:6.0f} {l2_to_sm(M, N, K, ran, us):>11s} {flops / PEAK_BF16_FLOPS * 1e6:13.0f} "
                  f"{nbytes / PEAK_HBM_BYTES * 1e6:12.0f}")


def main():
    if len(sys.argv) < 2 or (sys.argv[1] not in SHAPES and len(sys.argv) < 4):
        sys.exit(USAGE)
    if sys.argv[1] in SHAPES:
        table(sys.argv[1], [int(v) for v in sys.argv[2:]] or [0, 64, 128, 256, 1])
        return
    M, N, K = (int(v) for v in sys.argv[1:4])
    act = sys.argv[4] if len(sys.argv) > 4 and sys.argv[4] != "none" else None
    out_dtype = torch.float32 if len(sys.argv) > 5 and sys.argv[5] == "f32" else torch.bfloat16
    res = len(sys.argv) > 6 and sys.argv[6] == "1"
    block_n = int(sys.argv[7]) if len(sys.argv) > 7 else 0
    fn = make_gemm(M, N, K, act, out_dtype, res, block_n)
    us = time_launches(fn)
    nbytes = min_bytes(M, N, K, out_dtype.itemsize, res)
    ran = width_that_ran(fn)
    print(f"gemm M={M} N={N} K={K} act={act} out={str(out_dtype)[6:]} res={int(res)} block_n={block_n} "
          f"(ran {ran}): {us:.1f} us  {2.0 * M * N * K / us * 1e-6:.0f} TFLOP/s  "
          f"{nbytes / us * 1e-3:.0f} GB/s  L2->SM {l2_to_sm(M, N, K, ran, us)} TB/s")


if __name__ == "__main__":
    main()
