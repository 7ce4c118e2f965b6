"""Swin window attention: kernel time at Swin-B's stage shapes, and outputs of two builds of the library compared.

    python tools/bench_window_attention.py [--libs A.so,B.so] [--batch 256] [--iters 50] [--rounds 5] [--out DIR]

Timing: swin_base_patch4_window7_224's four stages at batch --batch (56 x 56 / 28 x 28 / 14 x 14 tokens in shifted 7 x 7
windows with 4 / 8 / 16 heads, then 7 x 7 tokens in one unshifted window with 32 heads), through the padded-table entry
the model runs, on random bf16 qkv and bias.  Each library given by --libs (default: the in-tree build) is timed with
CUDA events over --iters launches per shape, the libraries alternating, --rounds times; the median is reported.

Outputs (with two libraries): the window outputs at N = 49 (stage 1 above, batch 8) and N = 144 (12 x 12 windows,
96 x 96 tokens, 4 heads, batch 8, labels entry), and the logits of swin_base_patch4_window7_224 (bf16, random weights,
batch 8), each as the number of elements that differ between the libraries.

The card's name and power limit are read in the same run.  Prints one JSON line and writes it to --out.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tensorflow-image-models_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tfimm.architectures.swin import window_tables  # noqa: E402
from tfimm.backend import lib, ops  # noqa: E402

DH = 32
# (label, tokens per side, heads, shift) of swin_base_patch4_window7_224 at 224 x 224
STAGES = [("stage1", 56, 4, 3), ("stage2", 28, 8, 3), ("stage3", 14, 16, 3), ("stage4", 7, 32, 0)]


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", f"--query-gpu={fields}",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        return [v.strip() for v in out.strip().split(",")]
    except (OSError, subprocess.SubprocessError):
        return None


def open_libs(paths):
    """One ctypes handle per library (``lib.load`` with TFIMM_B200_LIB pointing at it); ``use(h)`` makes the ops
    launchers call ``h``."""
    handles = []
    for p in paths:
        lib._lib = None
        os.environ["TFIMM_B200_LIB"] = str(p)
        handles.append(lib.load())
    return handles


def use(handle):
    lib._lib = handle


def window_inputs(side, ws, H, shift, B, seed, padded):
    g = torch.Generator(device="cuda").manual_seed(seed)
    N, nw = ws * ws, (side // ws) ** 2
    qkv = torch.randn(B * nw * N, 3 * H * DH, device="cuda", generator=g).to(torch.bfloat16)
    bias = torch.randn(H, N, N, device="cuda", generator=g)
    row_map, labels = window_tables(side, side, ws, shift)
    rm = torch.from_numpy(row_map).cuda()
    lab = torch.from_numpy(labels).view(nw, N) if labels is not None else None
    if not padded:
        return lambda: ops.window_attention(qkv, bias, rm, lab.reshape(-1).cuda() if lab is not None else None, B,
                                            nw, N, H, DH, DH ** -0.5)
    bias_pad = torch.zeros(H, 64, 64, device="cuda")
    bias_pad[:, :N, :N] = bias
    bits = None
    if lab is not None:
        diff = (lab[:, :, None] != lab[:, None, :]).to(torch.int64)
        bits = torch.zeros(nw, 64, dtype=torch.int64)
        bits[:, :N] = (diff << torch.arange(N)[None, None, :]).sum(-1)
        bits = bits.cuda()
    return lambda: ops.window_attention_tc(qkv, bias_pad, rm, bits, B, nw, N, H, DH, DH ** -0.5)


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters      # us


def differing(a, b):
    return int((a.view(torch.int16) != b.view(torch.int16)).sum().item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", default=str(lib.LIB_PATH), help="comma-separated library paths")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    paths = args.libs.split(",")
    handles = open_libs(paths)
    name, power = (smi("name,power.limit") or ["?", "?"])[:2]
    res = {"gpu": name, "power_limit_w": power, "batch": args.batch, "libs": paths, "kernel_us": {}}

    fns = {label: window_inputs(side, 7, H, shift, args.batch, seed=i, padded=True)
           for i, (label, side, H, shift) in enumerate(STAGES)}
    times = {(label, j): [] for label in fns for j in range(len(handles))}
    for j, h in enumerate(handles):                      # warm every shape with every library
        use(h)
        for fn in fns.values():
            timed(fn, 3)
    for _ in range(args.rounds):
        for j, h in enumerate(handles):
            use(h)
            for label, fn in fns.items():
                times[(label, j)].append(timed(fn, args.iters))
    for label in fns:
        med = [statistics.median(times[(label, j)]) for j in range(len(handles))]
        res["kernel_us"][label] = {"median": [round(t, 2) for t in med],
                                   "spread": [round(max(times[(label, j)]) - min(times[(label, j)]), 2)
                                              for j in range(len(handles))]}
        if len(handles) == 2:
            res["kernel_us"][label]["ratio"] = round(med[1] / med[0], 4)

    if len(handles) == 2:
        import tfimm
        from oracle import params
        from oracle import swin as oswin

        diffs = {}
        for label, fn in (("window_N49", window_inputs(56, 7, 4, 3, 8, seed=7, padded=True)),
                          ("window_N144", window_inputs(96, 12, 4, 6, 8, seed=8, padded=False))):
            outs = []
            for h in handles:
                use(h)
                outs.append(fn())
            diffs[label] = {"differ": differing(*outs), "of": outs[0].numel()}
        model = tfimm.create_model("swin_base_patch4_window7_224", precision="bf16", device="cuda")
        model.load_weights_dict(params.random_params(oswin.param_shapes(model.cfg), seed=3))
        x = params.test_images(8, 224, 224).cuda()
        logits = []
        for h in handles:
            use(h)
            logits.append(model(x).float())
        diffs["swin_b_logits"] = {"differ": int((logits[0] != logits[1]).sum().item()), "of": logits[0].numel(),
                                  "max_abs": (logits[0] - logits[1]).abs().max().item()}
        res["outputs"] = diffs

    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "bench_window_attention.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
