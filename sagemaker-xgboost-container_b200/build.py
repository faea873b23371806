"""Build libb200xgb.so (CUDA kernels + C-ABI) in-tree with nvcc for the H100 (sm_90a).

    python sagemaker-xgboost-container_b200/build.py [--force]

nvcc cross-compiles without a GPU.  Objects go to build/ (git-ignored), the library to
sagemaker-xgboost-container_b200/lib/libb200xgb.so (git-ignored).
"""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "lib", "libb200xgb.so")
SOURCES = ["hist.cu", "tree.cu", "misc.cu", "predict_bins.cu", "quantile.cu", "auc.cu", "curve.cu", "container_metrics.cu", "shap.cu", "dart.cu", "survival.cu", "rank.cu", "adaptive.cu", "multi_target.cu", "custom_grad.cu", "sampling.cu", "refresh.cu", "csv.cu", "recordio.cu", "ingest.cu", "nvlink.cu", "grow.cu", "booster.cu", "model_io.cc", "legacy_io.cc", "comm.cc", "capi.cc"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden",
         "-diag-suppress", "177", "-I", os.path.join(HERE, "..", "include")]
# survival.cu and rank.cu compute their objectives, curve.cu its aucpr / auc terms, in double: no fused multiply-adds, so they
# round like a host restatement of the formulas.  container_metrics.cu and multi_target.cu keep the default flags of misc.cu:
# they inline predict()'s transform (csrc/transform.h) or the per-element formulas (csrc/elementwise.h), and --fmad=false
# would split the multiply-add inside expf
EXTRA_FLAGS = {"survival.cu": ["--fmad=false"], "rank.cu": ["--fmad=false"], "curve.cu": ["--fmad=false"]}


def _newest_header():
    t = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            if f.endswith((".h", ".cuh")):
                t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def _compile(src, force):
    obj = os.path.join(OBJ, src.rsplit(".", 1)[0] + ".o")
    sp = os.path.join(CSRC, src)
    if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(sp), _newest_header()):
        return obj, False
    cmd = [NVCC] + FLAGS + EXTRA_FLAGS.get(src, []) + (["-x", "cu"] if src.endswith(".cc") else []) + ["-c", sp, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, True


def build(force=False, verbose=True):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        res = list(ex.map(lambda s: _compile(s, force), SOURCES))
    objs = [o for o, _ in res]
    if force or any(c for _, c in res) or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        if verbose:
            print("built", LIB)
    elif verbose:
        print("up to date:", LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
