"""Build libpsalm_b200.so (hand-written sm_90a kernels for H100 + C ABI) in-tree with nvcc.

The .so and the objects under build/ are git-ignored build products.  No torch headers are involved: the
library is a plain C-ABI shared object loaded with ctypes (psalm_b200/_lib.py).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpsalm_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
         "--use_fast_math" if os.environ.get("PSALM_FAST_MATH") else "-DPSALM_PRECISE",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-O3", "--expt-relaxed-constexpr"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _hash(paths, extra=""):
    h = hashlib.sha256()
    for p in paths:
        h.update(os.path.basename(p).encode())
        h.update(open(p, "rb").read())
    h.update(extra.encode())
    return h.hexdigest()


def _shared_headers():
    hdrs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    return hdrs + [os.path.join(HERE, "..", "include", "psalm_b200.h")]


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library (incrementally: an object is rebuilt only when its
    source, a shared header or the flags changed).  Returns the library path."""
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    hdrs = _shared_headers()
    objs, procs, stamps = [], [], {}
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        stamp = _hash([src] + hdrs, " ".join(FLAGS))
        stamps[obj] = stamp
        objs.append(obj)
        sf = obj + ".stamp"
        if not force and os.path.exists(obj) and os.path.exists(sf) and open(sf).read() == stamp:
            continue
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, out))
        else:
            with open(obj + ".stamp", "w") as f:
                f.write(stamps[obj])
            if verbose or out.strip():
                sys.stderr.write(out)
    if failed:
        raise RuntimeError("psalm_b200: CUDA build failed")
    lib_stamp = hashlib.sha256("".join(stamps[o] for o in objs).encode()).hexdigest()
    stamp_file = LIB + ".stamp"
    if not procs and os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == lib_stamp:
        return LIB
    subprocess.check_call([NVCC, "-shared"] + FLAGS[:2] + ["-o", LIB] + objs + ["-lcudart"])
    with open(stamp_file, "w") as f:
        f.write(lib_stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
