"""Build libigmc_b200.so (sm_90a, H100) in-tree with nvcc.  No torch headers: the library is a plain C-ABI."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libigmc_b200.so")
SOURCES = ["extract.cu", "batch.cu", "rgcn.cu", "rgcn_rs.cu", "rgcn_l2.cu", "optim.cu", "sortpool.cu",
           "recommend.cu", "retrieve.cu", "graph_update.cu", "explain.cu", "influence.cu", "session.cu",
           "online.cu", "draws.cu", "counterfactual.cu", "elicit.cu", "recommend_cache.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "-shared", "-DIGMC_SM_ARCH=90"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "igmc_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    flags = list(FLAGS)
    cmd = [NVCC] + flags + (["-Xptxas", "-v"] if verbose else []) + \
          [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed")
    if verbose:
        print(r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    build(force=True, verbose="-v" in sys.argv)
    print(LIB)
