"""PVT throughput, its spatial-reduction attention against the byte floor and SDPA, and one forward's kernel families.

    python tools/bench_pvt.py [--models pvt_tiny,...] [--batch 256] [--warmup 3] [--iters 10] [--skip-models]
                              [--attention-only] [--out DIR]

Models (bf16, 224 x 224, random weights): one forward captured with ``cuda_graph`` per model, ``--warmup`` replays,
``--iters`` replays timed with CUDA events -> images / s.

Attention, at batch --batch, at the four stage shapes of the family at 224 px (N queries, N' keys, H heads, dh 64),
each timed with CUDA events over ``--iters`` launches in the same run:
  pvt_sr_attention_bf16  the new kernel on the q GEMM's and the kv GEMM's bf16 outputs
  pvt_sr_attention_f32   the fp32 kernel of the fp32 / tf32 models (on the same values in fp32)
  sdpa                   torch.nn.functional.scaled_dot_product_attention, bf16, on q, k, v already in (B, H, N, dh)
                         layout (the backend torch picks): the comparison only
Each row gives the byte floor: the bytes the kernel must move (pvt_ops.sr_attention_nbytes: q read, out written, k and v
read once) over the 3.35 TB/s HBM3 figure of the H100 SXM data sheet -- a bound, not a rate reached.

Families: one eager bf16 pvt_small forward at --batch with ``ops.trace`` on: the time of each kernel family (CUDA
events around every launch; the launches of a family summed) and its share of the forward.

The card's name and power limit are read in the same run.  Prints one JSON line and writes it to --out.
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
import tfimm.architectures.pvt  # noqa: E402,F401
from tfimm.backend import ops, pvt_ops  # noqa: E402

HBM_TBPS = 3.35        # H100 SXM data sheet
NAMES = ["pvt_tiny", "pvt_small", "pvt_medium", "pvt_large"]
# (label, N, N', H) at 224 px
ATTN_SHAPES = [("stage0", 3136, 49, 1), ("stage1", 784, 49, 2), ("stage2", 196, 49, 5), ("stage3", 50, 50, 8)]
DH = 64


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


def bench_models(names, batch, warmup, iters):
    res = {}
    for name in names:
        m = tfimm.create_model(name, precision="bf16", device="cuda")
        x = torch.rand((batch, 224, 224, 3), device="cuda")
        run = m.cuda_graph(batch)
        ms = timed(lambda: run(x), warmup, iters)
        res[name] = {"img_per_s": round(batch / ms * 1e3, 1), "step_ms": round(ms, 3)}
        print(name, res[name], flush=True)
        del m, run
        torch.cuda.empty_cache()
    return res


def bench_attention(batch, warmup, iters):
    res = {}
    for label, N, Nk, H in ATTN_SHAPES:
        B, scale = batch, DH ** -0.5
        q = torch.randn((B * N, H * DH), device="cuda").to(torch.bfloat16)
        kv = torch.randn((B * Nk, 2 * H * DH), device="cuda").to(torch.bfloat16)
        q32, kv32 = q.float(), kv.float()
        qh = q.view(B, N, H, DH).transpose(1, 2).contiguous()
        k, v = (t.transpose(1, 2).contiguous() for t in kv.view(B, Nk, 2, H, DH).unbind(2))
        t_bf16 = timed(lambda: pvt_ops.pvt_sr_attention_bf16(q, kv, B, N, Nk, H, DH, scale), warmup, iters)
        t_f32 = timed(lambda: pvt_ops.pvt_sr_attention_f32(q32, kv32, B, N, Nk, H, DH, scale), 1, max(1, iters // 2))
        t_sdpa = timed(lambda: F.scaled_dot_product_attention(qh, k, v, scale=scale), warmup, iters)
        nbytes = pvt_ops.sr_attention_nbytes(B, N, Nk, H, DH, 2)
        floor_us = nbytes / (HBM_TBPS * 1e12) * 1e6
        row = {"B": B, "N": N, "Nk": Nk, "H": H, "pvt_sr_attention_bf16_us": round(t_bf16 * 1e3, 1),
               "pvt_sr_attention_f32_us": round(t_f32 * 1e3, 1), "sdpa_us": round(t_sdpa * 1e3, 1),
               "mbytes": round(nbytes / 1e6, 1), "byte_floor_us": round(floor_us, 1),
               "of_floor": round(floor_us / (t_bf16 * 1e3), 3), "vs_sdpa": round(t_sdpa / t_bf16, 2)}
        res[label] = row
        print(label, row, flush=True)
        del q, kv, q32, kv32, qh, k, v
        torch.cuda.empty_cache()
    return res


def bench_families(batch):
    m = tfimm.create_model("pvt_small", precision="bf16", device="cuda")
    x = torch.rand((batch, 224, 224, 3), device="cuda")
    m(x)
    torch.cuda.synchronize()
    ops.trace = []
    try:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m(x)
        e1.record()
        torch.cuda.synchronize()
        fam = {}
        for name, a, b, _, _ in ops.trace:
            t, n = fam.get(name, (0.0, 0))
            fam[name] = (t + a.elapsed_time(b), n + 1)
    finally:
        ops.trace = None
    total = e0.elapsed_time(e1)
    rows = {k: {"ms": round(t, 3), "launches": n, "share": round(t / total, 3)}
            for k, (t, n) in sorted(fam.items(), key=lambda kv: -kv[1][0])}
    for k, r in rows.items():
        print(k, r, flush=True)
    return {"forward_ms": round(total, 3), "families": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(NAMES))
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--skip-models", action="store_true")
    ap.add_argument("--attention-only", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pvt needs a CUDA device")
    res = {"card": smi("name,power.limit"), "batch": args.batch}
    res["attention"] = bench_attention(args.batch, args.warmup, args.iters)
    if not args.attention_only:
        res["families"] = bench_families(args.batch)
        if not args.skip_models:
            res["models"] = bench_models(args.models.split(","), args.batch, args.warmup, args.iters)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_pvt.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
