"""Build libhgt_b200.so (sm_90a, H100) in-tree with nvcc.  No torch headers are involved: the library is
plain CUDA C++ behind the C ABI in include/hgt_b200.h."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")
LIB_PATH = os.path.join(HERE, "libhgt_b200.so")
SOURCES = ["common.cu", "plan.cu", "linear.cu", "linear_tc.cu", "edge.cu", "edge_bwd.cu", "update.cu", "layer.cu", "linear_bwd.cu", "update_bwd.cu", "sampler.cu", "gsample.cu", "merge.cu", "ingest.cu", "features.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(ROOT, "include", "hgt_b200.h"))
    nvcc = _nvcc()
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + headers):
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r.stderr

    with ThreadPoolExecutor(max_workers=min(6, max(1, len(jobs)))) as ex:
        logs = list(ex.map(run, jobs))
    if verbose:
        for l in logs:
            sys.stderr.write(l)
    objs = [os.path.join(BUILD, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(LIB_PATH, objs):
        run([nvcc, "-shared", "-o", LIB_PATH] + objs + ["-lcudart"])
    return LIB_PATH


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
