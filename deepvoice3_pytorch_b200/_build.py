"""In-tree nvcc build of the C-ABI library (sm_90a only).  Used by ``__graft_entry__.build()``.

    python -m deepvoice3_pytorch_b200._build
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libdv3b200.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(os.path.dirname(HERE), "include", "dv3b200.h")]
    return any(os.path.getmtime(f) > t for f in deps)


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into csrc/libdv3b200.so (separate objects, parallel nvcc)."""
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]
    if verbose:
        flags = flags + ["-Xptxas", "-v"]
    objs, procs = [], []
    for src in sources():
        obj = src[:-3] + ".o"
        objs.append(obj)
        procs.append((src, subprocess.Popen([nvcc] + flags + ["-c", src, "-o", obj],
                                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, out))
        if verbose and out.strip():
            print(out)
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB] + objs)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
