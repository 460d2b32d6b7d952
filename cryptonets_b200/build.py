"""Builds cryptonets_b200/libcnhe.so (sm_90a only: H100) with nvcc, in the package directory, so that the package imports from the source tree."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["ntt.cu", "poly_ops.cu", "mac_imma.cu", "mac_umma.cu", "behz.cu", "behz_fp.cu", "runtime.cu", "vec.cu", "wire.cu", "compact.cu", "diag.cu"]
OUT = os.path.join(HERE, "libcnhe.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2"]


def _stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "cnhe.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return OUT
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for s in SOURCES:
        o = os.path.join(HERE, "build", s.replace(".cu", ".o"))
        objs.append(o)
        cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, s), "-o", o]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError("nvcc failed on " + s)
        if verbose:
            sys.stderr.write(out.decode())
    tmp = OUT + ".tmp"  # link beside the target and rename: a snapshot of the tree never sees a half-written library
    subprocess.check_call([NVCC, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
