"""Builds lib/libh3dgs.so from csrc/*.cu with nvcc for sm_90a (H100), in-tree, so that the package
imports from the repository tree.  No torch dependency."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "lib")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr",
          "-ccbin", "/usr/bin/g++"]
# files whose results feed integer artefacts, or whose arithmetic is pinned bit for bit (knn.cu, the Morton keys of
# hier_build.cu and hier_merge.cu, the merger's ownership rule), are compiled without FMA contraction
NO_FMAD = {"preprocess.cu", "binning.cu", "hierarchy.cu", "knn.cu", "hier_build.cu", "hier_merge.cu"}
SOURCES = ["api.cu", "preprocess.cu", "binning.cu", "render_forward.cu", "render_backward.cu",
           "preprocess_backward.cu", "hierarchy.cu", "loss.cu", "l1_loss.cu", "optim.cu", "peer.cu", "metrics.cu",
           "knn.cu", "hier_build.cu", "hier_merge.cu"]


def _needs_build(src, obj, deps):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.getmtime(d) > t for d in [src] + deps)


def build(verbose=False, force=False, variant=None, defs=()):
    """variant / defs: an A/B build with extra -D switches -> lib/libh3dgs_<variant>.so (objects under build_<variant>/);
    h3dgs/_lib.py loads it when H3DGS_LIBRARY names it."""
    os.makedirs(OUT, exist_ok=True)
    objdir = os.path.join(HERE, "build" + (f"_{variant}" if variant else ""))
    os.makedirs(objdir, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    deps.append(os.path.join(HERE, "..", "include", "h3dgs.h"))
    deps.append(os.path.abspath(__file__))

    def compile_one(name):
        src = os.path.join(CSRC, name)
        obj = os.path.join(objdir, name.replace(".cu", ".o"))
        if not force and not _needs_build(src, obj, deps):
            return obj, ""
        cmd = [NVCC] + ARCH + COMMON + (["-fmad=false"] if name in NO_FMAD else []) + \
            [f"-D{d}" for d in defs] + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {name}:\n{r.stdout}\n{r.stderr}")
        return obj, r.stderr

    with ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(compile_one, SOURCES))
    objs = [o for o, _ in results]
    log = "\n".join(f"== {n} ==\n{l}" for n, (_, l) in zip(SOURCES, results) if l)
    with open(os.path.join(objdir, "ptxas.log"), "a") as f:
        f.write(log)
    if verbose and log:
        print(log)
    so = os.path.join(OUT, f"libh3dgs_{variant}.so" if variant else "libh3dgs.so")
    if force or not os.path.exists(so) or any(os.path.getmtime(o) > os.path.getmtime(so) for o in objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", so] + objs + ["-ccbin", "/usr/bin/g++"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return so


if __name__ == "__main__":
    # python build.py [-v] [-f] [--variant NAME -DSWITCH ...]
    var = sys.argv[sys.argv.index("--variant") + 1] if "--variant" in sys.argv else None
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv, variant=var,
                defs=[a[2:] for a in sys.argv if a.startswith("-D")]))
