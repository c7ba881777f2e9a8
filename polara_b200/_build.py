"""Builds ``libpolara_b200.so`` in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import glob
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libpolara_b200.so")

ARCH = "arch=compute_90a,code=sm_90a"
NVCC_FLAGS = [
    "-gencode", ARCH, "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "--expt-relaxed-constexpr",
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build the polara_b200 CUDA library")
    return exe


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + \
        [os.path.join(os.path.dirname(PKG_DIR), "include", "polara_b200.h")]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False, extra_flags=()):
    if not force and not needs_build():
        return LIB_PATH
    objs = []
    obj_dir = os.path.join(PKG_DIR, "csrc", "build")
    os.makedirs(obj_dir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(src)
                and all(os.path.getmtime(obj) > os.path.getmtime(h)
                        for h in glob.glob(os.path.join(CSRC, "*.cuh")) +
                        [os.path.join(os.path.dirname(PKG_DIR), "include", "polara_b200.h")])):
            continue
        cmd = [_nvcc()] + [f for f in NVCC_FLAGS if f != "-shared"] + list(extra_flags) + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, out))
        if verbose and out.strip():
            print(out)
    cmd = [_nvcc(), "-gencode", ARCH, "-shared", "-Xcompiler", "-fPIC",
           "-o", LIB_PATH] + objs
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stdout)
    return LIB_PATH


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose=True, extra_flags=["-Xptxas", "-v"] if "-v" in sys.argv else ()))
