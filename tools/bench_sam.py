"""Segment Anything image-encoder throughput and the relative-position attention kernel's tensor-core throughput.

    python tools/bench_sam.py [--models sam_vit_b,sam_vit_l,sam_vit_h] [--batches 1,8] [--warmup 3] [--iters 10]
                              [--out DIR]

For each model (bf16, 1024 x 1024 input) and batch: one encoder forward captured with ``cuda_graph``, ``--warmup``
replays, ``--iters`` replays timed with CUDA events -> images / s.  Then one eager forward with every launch bracketed by
CUDA events (``ops.trace``) -> time per kernel family, and the relpos attention kernel's achieved TFLOP/s in its global
and windowed form, with FLOPs computed here from the shapes (4 N^2 dh per sequence and head: q k^T and P V; the padded
windows' positions count, the kernel computes them) against the 989 TFLOP/s dense bf16 peak of the H100 SXM data sheet.
The card's name, power limit and SM clocks (sampled right after the timed loops) are read in the same run and printed
with the numbers.  Prints one JSON line at the end and writes it to ``--out`` if given.
"""
import argparse
import json
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tensorflow-image-models_b200"))

import tfimm  # noqa: E402
import tfimm.architectures.segment_anything  # noqa: E402,F401
from tfimm.backend import ops  # noqa: E402

BF16_PEAK_TFLOPS = 989.0   # H100 SXM data sheet, dense


def smi(fields):
    idx = torch.cuda.current_device()
    try:
        out = subprocess.run(["nvidia-smi", f"--id={idx}", f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return [v.strip() for v in out.split(",")]
    except (OSError, subprocess.SubprocessError):
        return None


def relpos_flops(cfg, batch):
    """(global, windowed) FLOPs of the relpos attention launches of one forward, from the shapes."""
    gh, gw = cfg.input_size[0] // cfg.encoder_patch_size, cfg.input_size[1] // cfg.encoder_patch_size
    H, dh, ws = cfg.encoder_nb_heads, cfg.encoder_embed_dim // cfg.encoder_nb_heads, cfg.encoder_window_size
    nglob = len(cfg.encoder_global_attn_indices)
    nwin = cfg.encoder_nb_blocks - nglob
    glob = nglob * 4.0 * batch * H * (gh * gw) ** 2 * dh
    win = nwin * 4.0 * batch * (-(-gh // ws)) * (-(-gw // ws)) * H * (ws * ws) ** 2 * dh
    return glob, win


def run(name, batches, warmup, iters):
    model = tfimm.create_model(name, precision="bf16", device="cuda")
    enc = model.image_encoder
    h, w = model.cfg.input_size
    res = {}
    for batch in batches:
        x = torch.rand(batch, h, w, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
        fwd = enc.cuda_graph(batch)
        for _ in range(warmup):
            fwd(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fwd(x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        clocks = smi("clocks.sm")
        del fwd
        # per-family time of one eager forward (events around every launch; a separate pass, not the timed one)
        enc(x)
        torch.cuda.synchronize()
        ops.trace = []
        try:
            enc(x)
            torch.cuda.synchronize()
            fam = defaultdict(float)
            for fname, a, b, _, _ in ops.trace:
                fam[fname] += a.elapsed_time(b)
            # the relpos launches alternate by block kind: split them by the block's window setting
            rel = [a.elapsed_time(b) for fname, a, b, _, _ in ops.trace if fname.startswith("relpos_attention")]
        finally:
            ops.trace = None
        kinds = [0 if j in model.cfg.encoder_global_attn_indices else 1 for j in range(model.cfg.encoder_nb_blocks)]
        t_glob = sum(t for t, k in zip(rel, kinds) if k == 0)
        t_win = sum(t for t, k in zip(rel, kinds) if k == 1)
        f_glob, f_win = relpos_flops(model.cfg, batch)
        row = {"ms": ms, "img_per_s": batch / (ms * 1e-3), "sm_clock_mhz": clocks[0] if clocks else None,
               "family_ms": dict(sorted(fam.items(), key=lambda kv: -kv[1])),
               "relpos_global": {"ms": t_glob, "tflops": f_glob / (t_glob * 1e-3) * 1e-12},
               "relpos_window": {"ms": t_win, "tflops": f_win / (t_win * 1e-3) * 1e-12}}
        for k in ("relpos_global", "relpos_window"):
            row[k]["share_of_peak"] = row[k]["tflops"] / BF16_PEAK_TFLOPS
        res[batch] = row
        print(f"{name} batch {batch}: {row['img_per_s']:7.2f} img/s ({ms:8.2f} ms / forward, graph), SM clock "
              f"{row['sm_clock_mhz']} MHz")
        for k in ("relpos_global", "relpos_window"):
            r = row[k]
            print(f"   {k:15s} {r['ms']:8.2f} ms  {r['tflops']:6.1f} TFLOP/s = {100 * r['share_of_peak']:.1f} % of "
                  f"{BF16_PEAK_TFLOPS:.0f}")
        tot = sum(fam.values())
        for k, v in row["family_ms"].items():
            print(f"   {k:26s} {v:8.2f} ms  {100 * v / tot:5.1f} %  (eager pass, events per launch)")
        torch.cuda.empty_cache()
    del enc, model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="sam_vit_b,sam_vit_l,sam_vit_h")
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sam.py measures on the GPU; no CUDA device found")
    lim = smi("power.limit,clocks.max.sm")
    dev = {"name": torch.cuda.get_device_name(), "power_limit_w": lim[0] if lim else None,
           "max_sm_clock_mhz": lim[1] if lim else None}
    print(f"card: {dev['name']}, power limit {dev['power_limit_w']} W, max SM clock {dev['max_sm_clock_mhz']} MHz")
    res = {"card": dev, "input": [1024, 1024], "precision": "bf16", "models": {}}
    for name in args.models.split(","):
        res["models"][name] = run(name, [int(b) for b in args.batches.split(",")], args.warmup, args.iters)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_sam.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
