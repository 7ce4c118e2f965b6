"""Measured DRAM traffic per kernel family (the `roofline.traffic` field of bench.py).

    # on the GPU, one model per ncu run (metrics-only pass, no clock control):
    ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none \
        --profile-from-start off --csv --log-file traffic_<model>.csv \
        python tools/ncu_traffic.py run <model> [batch]
    # anywhere: fold the CSVs into profiles/dram_traffic.json (read by bench.py) + a readable summary
    python tools/ncu_traffic.py parse traffic_*.csv

`run` executes one eager forward of the model at the bench batch between cudaProfilerStart/Stop (after a warm-up
forward), so ncu sees exactly the launches of one step.  Kernel names are mapped to the families bench.py's
instrumented pass reports (the C-ABI entry point that launched them).
"""
import csv
import json
import re
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

# kernel-name substring -> family name used by tfimm.backend.ops._call / bench.py
FAMILIES = [
    ("mlp_fused", "mlp_bf16"),
    # the TF32 instances of the wgmma GEMM (template argument A-transform = 2, fp32 out) before the bf16 ones
    ("gemm_wgmma_kernelILi64EfLi2E", "gemm_tf32"), ("gemm_wgmma_kernelILi128EfLi2E", "gemm_tf32"),
    ("gemm_wgmma", "gemm_bf16"), ("gemm_persistent", "gemm_bf16"), ("gemm_bf16_skinny", "gemm_bf16"),
    # before "gemm_f32": the MLP-Mixer fp32 token-mixing kernel's name contains it
    ("token_gemm_f32", "token_gemm_f32"), ("affine_kernel", "affine"),
    ("gn1_partials", "gn1_partials"), ("poolformer_mixer", "poolformer_mixer"), ("gn1_apply", "gn1_apply"),
    ("gemm_f32", "gemm_f32"),
    ("pit_attention_bf16", "pit_attention_bf16"), ("pit_pool", "pit_pool"),
    ("cait_talking_heads_bf16", "cait_talking_heads_bf16"), ("cait_talking_heads_f32", "cait_talking_heads_f32"),
    ("cait_class_attn", "cait_class_attention"), ("cait_add_pos", "cait_add_pos"),
    # before "dwconv_*": the ConvMixer kernel's name contains "dwconv"
    ("convmixer_dwconv", "convmixer_dwconv"),
    # PVT v2's head-dim-32 instances (template argument 32) before the PVT head-dim-64 ones
    ("pvt_sr_attention_bf16_kernelILi32E", "pvt_v2_sr_attention_bf16"),
    ("pvt_sr_attention_f32_kernelILi32E", "pvt_v2_sr_attention_f32"), ("pvt_v2_conv_mlp", "pvt_v2_conv_mlp_bf16"),
    ("pvt_sr_attention_bf16", "pvt_sr_attention_bf16"), ("pvt_embed_norm", "pvt_embed_norm"),
    # before "attention_f32": the PVT and Segment Anything kernels' names contain it
    ("pvt_sr_attention_f32", "pvt_sr_attention_f32"),
    ("relpos_attention_bf16", "relpos_attention_bf16"), ("relpos_attention_f32", "relpos_attention_f32"),
    ("vit_attention_tf32", "attention_tf32"), ("vit_attention", "attention_bf16"), ("attention_cls", "attention_cls_bf16"), ("attention_f32", "attention_f32"),
    ("window_attention", "window_attention_bf16"),
    ("layernorm_patch2x2", "layernorm_patch2x2"), ("patch_merge_ln", "patch_merge_ln"), ("layernorm", "layernorm"),
    ("dwconv7_ln", "dwconv_ln"), ("dwconv_ln", "dwconv_ln"), ("dwconv_act", "dwconv_bias_act"),
    ("dwconv_bias_act", "dwconv_bias_act"),
    ("patchify", "patchify"), ("assemble_tokens", "assemble_tokens"), ("cast", "cast"),
    ("global_avg_pool", "global_avg_pool"), ("im2col", "im2col"), ("stem", "im2col"), ("group_norm", "group_norm"),
    ("blur_pool", "blur_pool"), ("se_gate", "se_gate"), ("scale_channels", "scale_channels"), ("pool2d", "pool2d"),
    ("grouped_conv", "grouped_conv"), ("eca_gate", "eca_gate"), ("scale_add_act", "scale_add_act"),
]


def family_of(kernel):
    for key, fam in FAMILIES:
        if key in kernel:
            return fam
    return "other:" + kernel.split("(")[0][:40]


def run(model_name, batch):
    sys.path.insert(0, str(ROOT / "tensorflow-image-models_b200"))
    import torch

    import tfimm

    model = tfimm.create_model(model_name, precision="bf16", device="cuda")
    h, w = model.cfg.input_size
    x = torch.rand(batch, h, w, model.cfg.in_channels, device="cuda")
    model(x)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStart()
    model(x)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStop()
    print(f"TRAFFIC_RUN model={model_name} batch={batch}")


def parse(paths):
    out_path = ROOT / "profiles" / "dram_traffic.json"
    table = json.loads(out_path.read_text()) if out_path.exists() else {}
    for path in paths:
        text = Path(path).read_text()
        m = re.search(r"TRAFFIC_RUN model=(\S+) batch=(\d+)", text)
        lines = [ln for ln in text.splitlines() if ln.startswith('"')]
        rows = list(csv.DictReader(lines))
        if not rows:
            print(f"{path}: no rows")
            continue
        name = m.group(1) if m else Path(path).stem.replace("traffic_", "")
        batch = int(m.group(2)) if m else 256
        per = {}
        for r in rows:
            metric, val = r["Metric Name"], float(r["Metric Value"].replace(",", ""))
            unit = r.get("Metric Unit", "")
            scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1.0, "us": 1e3, "ms": 1e6,
                     "usecond": 1e3, "nsecond": 1.0, "msecond": 1e6}.get(unit, 1.0)
            d = per.setdefault(r["ID"], {"kernel": r["Kernel Name"], "bytes": 0.0, "ns": 0.0})
            if metric.startswith("dram__bytes"):
                d["bytes"] += val * scale
            elif metric.startswith("gpu__time_duration"):
                d["ns"] += val * scale
        fam = {}
        for d in per.values():
            f = fam.setdefault(family_of(d["kernel"]), {"bytes": 0.0, "ns": 0.0, "launches": 0})
            f["bytes"] += d["bytes"]
            f["ns"] += d["ns"]
            f["launches"] += 1
        table[name] = {"batch": batch, "families": {k: v["bytes"] for k, v in fam.items()},
                       "launches": {k: v["launches"] for k, v in fam.items()},
                       "ncu_ms": {k: round(v["ns"] / 1e6, 4) for k, v in fam.items()},
                       "how": "ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum --clock-control none, one eager "
                              "forward (cold-cache, serialised launches)"}
        # per-kernel launch list of the same pass (cold-cache, serialised: compare SHARES with the bench line, not times)
        kern = {}
        for d in per.values():
            k = kern.setdefault(re.sub(r"\(.*", "", d["kernel"])[-72:], {"n": 0, "ns": 0.0, "bytes": 0.0})
            k["n"] += 1
            k["ns"] += d["ns"]
            k["bytes"] += d["bytes"]
        tot_ns = sum(k["ns"] for k in kern.values()) or 1.0
        lines_out = [f"# {name}, batch {batch}: ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,"
                     "gpu__time_duration.sum --clock-control none, one eager forward",
                     "# kernel | launches | avg us | share of the pass | DRAM MB per launch"]
        for kname, k in sorted(kern.items(), key=lambda kv: -kv[1]["ns"]):
            lines_out.append(f"{kname:74s} {k['n']:4d} {k['ns'] / k['n'] / 1e3:9.1f} {100 * k['ns'] / tot_ns:6.1f}% "
                             f"{k['bytes'] / k['n'] / 1e6:9.1f}")
        (ROOT / "profiles" / f"r02_launches_{name}.txt").write_text("\n".join(lines_out) + "\n")
        tot = sum(v["bytes"] for v in fam.values())
        print(f"{name} (batch {batch}): {tot / 1e9:.2f} GB DRAM traffic per forward = {tot / batch / 1e6:.1f} MB/image")
        for k, v in sorted(fam.items(), key=lambda kv: -kv[1]["bytes"]):
            print(f"   {k:26s} {v['launches']:4d} launches {v['bytes'] / 1e9:8.3f} GB {v['ns'] / 1e6:8.3f} ms")
    out_path.write_text(json.dumps(table, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    if sys.argv[1] == "run":
        run(sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else 256)
    else:
        parse(sys.argv[2:])
