"""Builds libtfimm_b200.so (sm_90a, H100) in-tree with nvcc.

    python tensorflow-image-models_b200/build.py [--force] [--verbose]

The shared object lands next to the ctypes binding
(``tensorflow-image-models_b200/tfimm/backend/libtfimm_b200.so``) so that it travels to
wherever the repository tree goes.  nvcc cross-compiles without a GPU.
"""
import argparse
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
OUT_DIR = ROOT / "tfimm" / "backend"
OBJ_DIR = ROOT / "build"
LIB = OUT_DIR / "libtfimm_b200.so"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
    "-I", str(ROOT.parent / "include"),
]


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, defines=(), out: Path = None) -> Path:
    """defines / out: build a variant of the library (e.g. -DTFIMM_FAST_ACT for an A/B measurement) into another
    file; load it with TFIMM_B200_LIB=<path>.  The default build is the product."""
    if defines or out is not None:
        return _build_variant(list(defines), Path(out or (OBJ_DIR / "libtfimm_b200_variant.so")))
    sources = sorted(CSRC.glob("*.cu"))
    headers = sorted(CSRC.glob("*.cuh")) + sorted((ROOT.parent / "include").glob("*.h"))
    stamp = OBJ_DIR / "stamp.txt"
    digest = _digest(sources + headers)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    OBJ_DIR.mkdir(exist_ok=True)
    OUT_DIR.mkdir(parents=True, exist_ok=True)

    def compile_one(src: Path):
        obj = OBJ_DIR / (src.stem + ".o")
        cmd = [NVCC, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, res

    with ThreadPoolExecutor(max_workers=min(8, len(sources))) as pool:
        results = list(pool.map(compile_one, sources))
    log = []
    for src, obj, res in results:
        log.append(f"==== {src.name}\n{res.stdout}\n{res.stderr}")
        if res.returncode != 0:
            sys.stderr.write(log[-1])
            raise RuntimeError(f"nvcc failed on {src.name}")
    (OBJ_DIR / "ptxas.log").write_text("\n".join(log))
    if verbose:
        print("\n".join(log))
    link = [NVCC, "-shared", "-o", str(LIB), *[str(o) for _, o, _ in results],
            "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    res = subprocess.run(link, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("link failed")
    stamp.write_text(digest)
    return LIB


def _build_variant(defines, out: Path) -> Path:
    obj_dir = OBJ_DIR / ("variant_" + hashlib.sha256(" ".join(defines).encode()).hexdigest()[:8])
    obj_dir.mkdir(parents=True, exist_ok=True)
    flags = NVCC_FLAGS + [f"-D{d}" for d in defines]

    def compile_one(src: Path):
        obj = obj_dir / (src.stem + ".o")
        return obj, subprocess.run([NVCC, *flags, "-c", str(src), "-o", str(obj)], capture_output=True, text=True)

    with ThreadPoolExecutor(max_workers=8) as pool:
        results = list(pool.map(compile_one, sorted(CSRC.glob("*.cu"))))
    for obj, res in results:
        if res.returncode != 0:
            sys.stderr.write(res.stderr)
            raise RuntimeError(f"nvcc failed on {obj.stem}")
    res = subprocess.run([NVCC, "-shared", "-o", str(out), *[str(o) for o, _ in results],
                          "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"], capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("link failed")
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--define", action="append", default=[], help="extra -D macro: builds a VARIANT library")
    ap.add_argument("--out", default=None, help="output path of the variant library")
    args = ap.parse_args()
    print(build(force=args.force, verbose=args.verbose, defines=args.define, out=args.out))
