"""Build tests/cuemu/_build/libmmssl_emu.so: the library's plain-CUDA kernels compiled for the HOST under the cuemu
fiber emulator (include/cuemu.h).  TEST INFRASTRUCTURE ONLY -- nothing under mmssl_b200/ imports this.

The sources are mmssl_b200/csrc/*.cu, untouched except for three pieces of syntax g++ cannot parse, rewritten textually:
  kernel<<<grid, block, smem, stream>>>(args)   ->  cuemu::launch(kernel, cuemu::cfg(grid, block, smem, stream), "kernel")(args)
  extern __shared__ [__align__(n)] T name[];    ->  T* name = (T*)cuemu::dyn_smem();
  asm volatile("ptx" : outs : ins : ...);       ->  cuemu::ptx_op("ptx", &outs, sizes, n, ins, n)   (cuemu_ptx.cpp: a functional model of
                                                    the mbarrier / TMA / wgmma subset the library uses; anything else fails the launch)
CUB's SortPairs / ExclusiveSum are host shims (include/cub/cub.cuh).  Every .cu of the library is compiled.

    python -m tests.cuemu.build [--force]
"""
import concurrent.futures as cf
import hashlib
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "mmssl_b200", "csrc")
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libmmssl_emu.so")
SOURCES = ["core.cu", "gan.cu", "eval.cu", "sgemm.cu", "adamw.cu", "rowops.cu", "loss.cu", "idfuse.cu", "sampler.cu", "spmm.cu", "graph.cu", "proj_common.cu", "regraph.cu", "shard.cu", "proj_tc.cu", "gemm_wide.cu", "spmm_hot.cu", "spmm_bulk.cu", "loss_tc.cu"]
HEADERS = ["common.cuh", "spmm_common.cuh", "tc_common.cuh"]
CXX = os.environ.get("CXX", "g++")
FLAGS = ["-O1", "-g", "-std=c++17", "-fPIC", "-fno-strict-aliasing", "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas",
         "-Wno-unused-variable", "-Wno-sign-compare", "-Wno-unused-but-set-variable"]

_LAUNCH = re.compile(r"([A-Za-z_][\w:]*(?:\s*<[^;{}()<>]*>)?)\s*<<<(.+?)>>>\s*\(", re.S)
_EXT_SH = re.compile(r"extern\s+__shared__\s+(?:__align__\(\s*\d+\s*\)\s+)?([\w:\s]+?)\s+(\w+)\s*\[\s*\]\s*;")
_ASM = re.compile(r"\basm\s+volatile\s*\(")


def _split_top(text: str, sep: str):
    """Split at `sep` outside parentheses / brackets / string literals."""
    parts, depth, in_str, cur = [], 0, False, []
    i = 0
    while i < len(text):
        ch = text[i]
        if in_str:
            cur.append(ch)
            if ch == "\\":
                i += 1
                cur.append(text[i])
            elif ch == '"':
                in_str = False
        elif ch == '"':
            in_str = True
            cur.append(ch)
        elif ch in "([{":
            depth += 1
            cur.append(ch)
        elif ch in ")]}":
            depth -= 1
            cur.append(ch)
        elif ch == sep and depth == 0:          # C++ scope operators only occur inside the operands' parentheses
            parts.append("".join(cur))
            cur = []
        else:
            cur.append(ch)
        i += 1
    parts.append("".join(cur))
    return parts


_OPERAND = re.compile(r'^\s*"([^"]*)"\s*\((.*)\)\s*$', re.S)
_STRLIT = re.compile(r'"((?:[^"\\]|\\.)*)"')


def _strip_asm(src: str) -> str:
    """asm volatile("template" : outputs : inputs : clobbers);  ->  a call of cuemu::ptx_op with the template text, pointers to
    the output operands and the input operands as 64-bit values (floats by bit pattern).  include/cuemu_ptx.h interprets the
    subset of PTX the library uses (mbarrier, TMA tensor copies, wgmma, griddepcontrol) and fails the launch on the rest."""
    out, pos = [], 0
    while True:
        m = _ASM.search(src, pos)
        if not m:
            out.append(src[pos:])
            return "".join(out)
        out.append(src[pos:m.start()])
        i, depth, in_str = m.end(), 1, False
        while depth:
            ch = src[i]
            if in_str:
                if ch == "\\":
                    i += 1
                elif ch == '"':
                    in_str = False
            elif ch == '"':
                in_str = True
            elif ch == "(":
                depth += 1
            elif ch == ")":
                depth -= 1
            i += 1
        body = src[m.end():i - 1]
        while src[i] in " \t\n":
            i += 1
        assert src[i] == ";", "asm statement without ';'"
        secs = _split_top(body, ":")
        template = "".join(x.group(1) for x in _STRLIT.finditer(secs[0]))
        outs = [o for o in _split_top(secs[1], ",") if o.strip()] if len(secs) > 1 else []
        ins = [o for o in _split_top(secs[2], ",") if o.strip()] if len(secs) > 2 else []
        o_expr = [_OPERAND.match(o).group(2) for o in outs]
        i_expr = [_OPERAND.match(o).group(2) for o in ins]
        code = "{ void* cuemu_o[] = {%s nullptr}; int cuemu_os[] = {%s 0}; uint64_t cuemu_i[] = {%s 0}; cuemu::ptx_op(\"%s\", cuemu_o, cuemu_os, %d, cuemu_i, %d); }" % (
            "".join("(void*)&(%s)," % e for e in o_expr), "".join("(int)sizeof(%s)," % e for e in o_expr),
            "".join("cuemu::as_u64(%s)," % e for e in i_expr), template.replace("\\", "\\\\").replace('"', '\\"'), len(o_expr), len(i_expr))
        out.append(code)
        pos = i + 1


def transform(src: str) -> str:
    src = _strip_asm(src)
    src = _EXT_SH.sub(lambda m: "%s* %s = (%s*)cuemu::dyn_smem();" % (m.group(1), m.group(2), m.group(1)), src)
    src = _LAUNCH.sub(lambda m: 'cuemu::launch(%s, cuemu::cfg(%s), "%s")(' % (m.group(1), m.group(2), re.sub(r"\s+", "", m.group(1))), src)
    assert "<<<" not in src, "unconverted launch"
    return src


def _digest() -> str:
    h = hashlib.sha1()
    files = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.join(HERE, "cuemu.cpp"), os.path.join(HERE, "selftest.cu"), os.path.join(HERE, "cuemu_ptx.cpp"), os.path.join(HERE, "include", "cuda.h"), os.path.join(HERE, "include", "cuemu.h"),
                                                                   os.path.join(ROOT, "include", "mmssl_b200.h"), __file__]
    for p in files:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(path_in: str, path_obj: str):
    cmd = [CXX, *FLAGS, "-I", os.path.join(HERE, "include"), "-I", OUT, "-I", CSRC, "-c", path_in, "-o", path_obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("cuemu: g++ failed for %s:\n%s" % (path_in, r.stderr[-6000:]))
    return r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT, exist_ok=True)
    stamp = os.path.join(OUT, "stamp.sha1")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    jobs = []
    for h in HEADERS:                      # transformed headers shadow the originals (-I OUT comes before -I CSRC)
        with open(os.path.join(CSRC, h)) as f, open(os.path.join(OUT, h), "w") as g:
            g.write(transform(f.read()))
    for s in SOURCES:
        dst = os.path.join(OUT, s[:-3] + ".emu.cpp")
        with open(os.path.join(CSRC, s)) as f, open(dst, "w") as g:
            g.write('#line 1 "%s"\n' % os.path.join(CSRC, s))
            g.write(transform(f.read()))
        jobs.append((dst, dst[:-4] + ".o"))
    dst = os.path.join(OUT, "selftest.emu.cpp")
    with open(os.path.join(HERE, "selftest.cu")) as f, open(dst, "w") as g:
        g.write(transform(f.read()))
    jobs.append((dst, dst[:-4] + ".o"))
    jobs.append((os.path.join(HERE, "cuemu_ptx.cpp"), os.path.join(OUT, "cuemu_ptx.o")))
    jobs.append((os.path.join(HERE, "cuemu.cpp"), os.path.join(OUT, "cuemu.o")))
    with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        warns = list(ex.map(lambda j: _compile(*j), jobs))
    if verbose:
        print("\n".join(w for w in warns if w))
    r = subprocess.run([CXX, "-shared", "-o", LIB, *[j[1] for j in jobs]], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("cuemu: link failed:\n" + r.stderr[-4000:])
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
