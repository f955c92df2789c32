"""Build libprisma_b200.so in-tree with nvcc for sm_90a (no torch extension machinery, no JIT cache).

    python -m prisma_b200.build          # or prisma_b200.build.build()

Objects are rebuilt only when a source or header is newer.  The resulting
prisma_b200/libprisma_b200.so is a build product (git-ignored).
"""
import concurrent.futures
import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libprisma_b200.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found; prisma_b200 has no non-CUDA path")


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    hdrs = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    newest_hdr = max(os.path.getmtime(h) for h in hdrs)
    nvcc = _nvcc()
    extra = os.environ.get("PRISMA_NVCC_EXTRA", "").split()  # extra nvcc flags, e.g. -Xptxas -v
    jobs = []
    objs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), newest_hdr):
            jobs.append([nvcc] + NVCC_FLAGS + extra + ["-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout + r.stderr)

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    if jobs or not os.path.exists(LIB):
        run([nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart", "-ldl"])
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
