"""Build libg2pc.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m g2pc.build            (from 3dgs-to-pc_b200/)   or   g2pc.build.build()

Replaces the reference's setup.py / CMakeLists.txt (gaussian-pointcloud-rasterization/setup.py:17-33,
CMakeLists.txt:37) which build a pybind11 torch extension for sm_70/75/86; here a plain shared library is
produced (no torch headers) so the boundary stays a C ABI.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG_ROOT = os.path.dirname(HERE)
CSRC = os.path.join(PKG_ROOT, "csrc")
LIB_PATH = os.path.join(HERE, "libg2pc.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(os.path.dirname(PKG_ROOT), "include", "g2pc.h"))
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False, extra_flags=()):
    """Compile every .cu under csrc/ into one shared library.  Returns the library path.
    Safe to call from several processes at once (torchrun ranks): an exclusive file lock serialises the build and the
    staleness check is repeated under the lock."""
    if not force and not _stale():
        return LIB_PATH
    import fcntl
    os.makedirs(os.path.join(PKG_ROOT, "build"), exist_ok=True)
    with open(os.path.join(PKG_ROOT, "build", ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not _stale():
                return LIB_PATH
            return _build_locked(verbose, extra_flags)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose, extra_flags):
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    procs = []
    build_dir = os.path.join(PKG_ROOT, "build")
    os.makedirs(build_dir, exist_ok=True)
    for src in sources():
        obj = os.path.join(build_dir, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *extra_flags, "-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out.decode()}")
        if verbose and out:
            print(out.decode())
    tmp = LIB_PATH + ".tmp"
    cmd = [nvcc, "-shared", "-o", tmp, *objs, "-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout.decode()}")
    os.replace(tmp, LIB_PATH)  # atomic: a concurrent loader never sees a half-written library
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True,
                extra_flags=("-Xptxas", "-v") if "--ptxas" in sys.argv else ()))
