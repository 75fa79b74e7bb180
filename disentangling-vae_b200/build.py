"""Builds libdisvae_b200.so in-tree with nvcc for sm_90a (H100) (no JIT cache, no torch extension:
the library is a plain C-ABI shared object, see include/disvae_b200.h).

    python disentangling-vae_b200/build.py [--force] [--verbose]
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(ROOT, "include")
LIB = os.path.join(HERE, "libdisvae_b200.so")
STAMP = os.path.join(HERE, ".libdisvae_b200.stamp")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
                     "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v",
                     "-I", INCLUDE, "-I", CSRC]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    files = sources() + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh"))
    files.append(os.path.join(INCLUDE, "disvae_b200.h"))
    for f in files:
        h.update(f.encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library.  Returns the library path."""
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == digest:
                return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    procs = []
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    flags = [f for f in NVCC_FLAGS if f != "-shared"]
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [nvcc] + flags + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append("==== %s\n%s" % (os.path.basename(src), out))
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError("nvcc failed on %s" % src)
    link = [nvcc, "-shared"] + ARCH + ["-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log.append("==== link\n" + r.stdout)
    if r.returncode != 0:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("link failed")
    with open(os.path.join(objdir, "ptxas.log"), "w") as fh:
        fh.write("\n".join(log))
    with open(STAMP, "w") as fh:
        fh.write(digest)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
