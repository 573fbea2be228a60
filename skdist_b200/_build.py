"""Build libskdist_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBPATH = os.path.join(LIBDIR, "libskdist_b200.so")
SOURCES = ["api.cu", "logreg_simt.cu", "lbfgs_dev.cu", "logreg_multi.cu", "auc.cu", "logreg_tc.cu", "ridge.cu", "predict.cu", "sgd.cu", "sgd_tc.cu", "forest.cu", "forest_fast.cu", "bootstrap.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libskdist_b200.so")


def needs_build():
    if not os.path.exists(LIBPATH):
        return True
    t = os.path.getmtime(LIBPATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "include", "skdist_b200.h"))
    return any(os.path.getmtime(p) > t for p in deps if os.path.exists(p))


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into lib/libskdist_b200.so."""
    if not force and not needs_build():
        return LIBPATH
    os.makedirs(LIBDIR, exist_ok=True)
    # one builder at a time (torchrun starts N ranks that may all find the sources newer than the
    # library): the others wait on the lock and then see an up-to-date file
    import fcntl
    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not needs_build():
            return LIBPATH
        srcs = [os.path.join(CSRC, s) for s in SOURCES]
        tmp = "%s.%d.tmp" % (LIBPATH, os.getpid())
        cmd = [_nvcc()] + NVCC_FLAGS + srcs + ["-o", tmp]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            if os.path.exists(tmp):
                os.remove(tmp)
            raise RuntimeError("nvcc failed building libskdist_b200.so")
        os.replace(tmp, LIBPATH)
    log = os.path.join(LIBDIR, "build.log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return LIBPATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
