"""Build libfrosting_b200.so (the C-ABI library) in-tree with nvcc for sm_90a (H100).

    python -m frosting_b200.build [-v] [--force]

The .so and the object files are build products and stay out of git.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libfrosting_b200.so")
SOURCES = ["api.cu", "preprocess.cu", "binning.cu", "render_fwd.cu", "render_bwd.cu", "geom_bwd.cu", "mesh_vis.cu",
           "frosting_attr.cu", "frosting_edit.cu", "frosting_skin.cu", "texture.cu", "loss.cu", "optim.cu", "sugar_reg.cu",
           "sugar_dn.cu", "knn.cu", "frosting_init.cu"]
ARCH = "arch=compute_90a,code=sm_90a"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", ARCH, "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr",
]


def _deps_mtime():
    m = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            m = max(m, os.path.getmtime(os.path.join(root, f)))
    return m


def build(verbose: bool = False, force: bool = False) -> str:
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _deps_mtime():
        return LIB
    os.makedirs(OBJ, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, r

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        results = list(ex.map(compile_one, SOURCES))
    log = []
    for src, obj, r in results:
        log.append(f"== {src}\n{r.stderr}")
        if r.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed for {src}")
    with open(os.path.join(OBJ, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    objs = [o for _, o, _ in results]
    cmd = [NVCC, "-shared", "-gencode", ARCH, "-cudart", "shared", "-o", LIB, *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stderr)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="--force" in sys.argv))
