"""Build the CUDA extension in-tree: dsrg_b200/csrc/*.cu -> dsrg_b200/lib/libdsrg_b200.so.

sm_90a (H100) only; nvcc cross-compiles without a GPU.  The .so is a build product (git-ignored).
`python -m dsrg_b200.build` rebuilds when a source is newer.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdsrg_b200.so")
SOURCES = ["api.cu", "graph.cu", "lattice.cu", "tiles.cu", "meanfield.cu", "meanfield_wide.cu", "srg.cu", "loss.cu", "sec_loss.cu", "wire.cu", "numa.cu", "prep.cu", "post.cu", "annot.cu", "segdata.cu", "eval.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-fopenmp", "--fmad=true"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "dsrg_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defines=(), out=None):
    """defines/out: build an experimental variant (extra -D flags) next to the main library.
    Serialised with a file lock: under torchrun every rank may find the library stale at once."""
    import fcntl
    os.makedirs(LIBDIR, exist_ok=True)
    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose, defines, out)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose, defines, out):
    if out is None and not force and not needs_build():   # re-checked under the lock
        return LIB
    lib = out or LIB
    objdir = os.path.join(LIBDIR, "obj" if out is None else "obj_" + os.path.basename(out))
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + \
              ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", lib] + objs + ARCH + ["-Xcompiler", "-fopenmp", "-lgomp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
