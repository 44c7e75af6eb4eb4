"""In-tree build of the sm_90a kernels into deep_gcns_torch_b200/lib/libdgcn.so.

nvcc cross-compiles without a GPU; the .so is a build product (git-ignored).  `python -m deep_gcns_torch_b200.build` rebuilds.
"""
import hashlib
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libdgcn.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    root = os.path.dirname(PKG)
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(root, "include", "dgcn.h")]
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode() + b"\0" + fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "libdgcn.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out = p.communicate()[0].decode()
        if verbose:
            print(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s" % (" ".join(cmd), out))
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH
    subprocess.run(cmd, check=True)
    for o in objs:
        os.remove(o)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
