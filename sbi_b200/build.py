"""Build the C-ABI CUDA library in-tree: sbi_b200/lib/libsbi_b200.so (sm_90a, H100).

nvcc cross-compiles without a GPU; everything under sbi_b200/lib/ is a git-ignored build product.
"""
import concurrent.futures
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libsbi_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _fingerprint():
    h = hashlib.sha256()
    for root in (CSRC, INCLUDE):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(f.encode())
                    h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build_variant(name, defines):
    """Tuning helper: compile a variant library sbi_b200/lib/libsbi_b200_<name>.so with extra -D flags."""
    os.makedirs(LIBDIR, exist_ok=True)
    out = os.path.join(LIBDIR, f"libsbi_b200_{name}.so")
    objs = []
    for src in sources():
        obj = os.path.join(LIBDIR, f"{name}_" + os.path.basename(src)[:-3] + ".o")
        cmd = [_nvcc(), *[f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")], *[f"-D{d}" for d in defines],
               "-I", INCLUDE, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(obj)
    subprocess.check_call([_nvcc(), "-shared", "-o", out, *objs, "-gencode", "arch=compute_90a,code=sm_90a"])
    return out


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    fp = _fingerprint()
    if not force and os.path.exists(LIB) and os.path.exists(stamp):
        if open(stamp).read().strip() == fp:
            return LIB
    def compile_one(src):
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [_nvcc(), *NVCC_FLAGS, "-I", INCLUDE, "-c", src, "-o", obj]
        return src, obj, subprocess.run(cmd, capture_output=True, text=True)

    objs = []
    log = []
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        for src, obj, r in pool.map(compile_one, sources()):
            log.append(r.stderr)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError(f"nvcc failed on {src}")
            objs.append(obj)
    cmd = [_nvcc(), "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    with open(os.path.join(LIBDIR, "ptxas.log"), "w") as fh:
        fh.write("\n".join(log))
    with open(stamp, "w") as fh:
        fh.write(fp)
    if verbose:
        sys.stderr.write("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
