"""Build libmmssl_b200.so in-tree with nvcc for sm_90a (no torch extension machinery: the library
is a plain C-ABI shared object, loaded with ctypes).

    python -m mmssl_b200.build [--force] [--verbose]
"""
import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libmmssl_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function",
         "--expt-relaxed-constexpr", "--expt-extended-lambda", "-Xptxas", "-warn-spills"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    deps = [path] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "mmssl_b200.h"))
    for p in sorted(deps):
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(FLAGS + ARCH).encode())
    return h.hexdigest()


def _compile(src, force, verbose):
    os.makedirs(OBJ, exist_ok=True)
    spath = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src[:-3] + ".o")
    stamp = obj + ".sha1"
    dig = _digest(spath)
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False, ""
    cmd = [NVCC, *ARCH, *FLAGS, "-c", spath, "-o", obj]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return obj, True, r.stderr


def build(force=False, verbose=False):
    srcs = _sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, force, verbose), srcs))
    objs = [r[0] for r in res]
    rebuilt = any(r[1] for r in res)
    if verbose:
        for r in res:
            if r[2]:
                print(r[2])
    if rebuilt or not os.path.exists(LIB):
        cmd = [NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-lcudart_static", "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    lib = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(lib, os.path.getsize(lib) // 1024, "KiB")
