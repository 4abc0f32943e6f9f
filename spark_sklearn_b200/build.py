"""Build libb200gs.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200gs.so")
SOURCES = ["api.cu", "kernel_svm.cu", "gram.cu", "smo.cu", "smo_lean.cu", "smo_colown.cu", "score.cu", "svr.cu", "linear.cu", "logreg.cu", "gemm_tc.cu", "gemm_f64.cu", "linsvc.cu", "knn.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-cudart", "static"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "b200gs.h")]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library (separate objects, parallel)."""
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for s in SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, o, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for s, o, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed on %s" % s)
        objs.append(o)
    cmd = [_nvcc()] + NVCC_FLAGS + ["-shared", "-o", LIB] + objs
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
