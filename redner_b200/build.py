"""In-tree build of libredner_b200.so (hand-written CUDA for sm_90a, H100 + the C ABI) with nvcc.

    python -m redner_b200.build            # build if sources are newer than the library
    python -m redner_b200.build --force

The library is placed next to this file (redner_b200/libredner_b200.so), so the package runs from the source tree.  No JIT cache, no torch extension machinery: the product is a plain C-ABI shared object.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
DATA = os.path.join(HERE, "data")
LIB = os.path.join(HERE, "libredner_b200.so")
LIB_F64 = os.path.join(HERE, "libredner_b200_f64.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(lib):
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    srcs = glob.glob(os.path.join(CSRC, "*")) + glob.glob(os.path.join(HERE, "..", "include", "*.h")) + [__file__]
    return any(os.path.getmtime(s) > t for s in srcs)


def build(force=False, double=False, verbose=False, defines=(), out=None, nvcc_flags=()):
    lib = out or (LIB_F64 if double else LIB)
    if not force and not _stale(lib):
        return lib
    objdir = os.path.join(HERE, "_build_f64" if double else ("_build_" + os.path.basename(out) if out else "_build"))
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    # -prec-div=false / -prec-sqrt=false: the path tracer is full of normalisations and quotients; the IEEE-exact
    # division / square-root sequences (FCHK + slow path) are a large share of the backward kernel's instructions, while the
    # 2-ulp approximations move the image by < 1e-6 relative L2.  sin/cos/pow/log stay accurate (no --use_fast_math).
    common = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-I", os.path.join(HERE, "..", "include")]
    fast = ["-fmad=true", "-prec-div=false", "-prec-sqrt=false"]
    if double:
        common += ["-DRB_REAL_DOUBLE"]
    common += ["-D" + d for d in defines]
    extra = list(nvcc_flags)  # (command-line overrides come last: nvcc keeps the last value of a repeated option)
    if verbose:
        common += ["-Xptxas", "-v"]
    # rb_edge_tree.cu builds the secondary-edge trees and must round like the host builder it is tested against (no FMA contraction,
    # IEEE division / square root); its bottom-up passes hand data between thread blocks, so its global loads bypass the L1.  The
    # steps it shares with the host builder are header-only (rb_edge_tree.cuh) so that they are compiled inside this translation unit,
    # under these flags, rather than in an object built with the fast ones.
    # rb_edge_list.cu drops coplanar edges by a threshold on a dot product of unit normals: same rounding rule.
    # rb_light_build.cu computes the light tables in double with the steps of the host builder (rb_light_build.cuh): same rounding rule.
    per_file = {"rb_edge_tree.cu": ["-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-Xptxas", "-dlcm=cg"],
                "rb_edge_list.cu": ["-fmad=false", "-prec-div=true", "-prec-sqrt=true"],
                "rb_light_build.cu": ["-fmad=false", "-prec-div=true", "-prec-sqrt=true"]}
    objs = []
    procs = []
    for src in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        objs.append(obj)
        procs.append((src, subprocess.Popen([nvcc] + ARCH + common + per_file.get(os.path.basename(src), fast) + extra + ["-c", src, "-o", obj], stdout=subprocess.PIPE,
                                            stderr=subprocess.STDOUT)))
    tab = os.path.join(objdir, "rb_tables.o")
    objs.append(tab)
    procs.append(("rb_tables.cpp", subprocess.Popen(["g++", "-O2", "-fPIC", "-DRB_DATA_DIR=" + DATA, "-c", os.path.join(CSRC, "rb_tables.cpp"), "-o", tab],
                                                   stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("[redner_b200.build] FAILED %s\n%s\n" % (src, out))
        elif verbose or out.strip():
            sys.stderr.write("[redner_b200.build] %s\n%s\n" % (src, out))
    if failed:
        raise RuntimeError("redner_b200: nvcc compilation failed")
    cmd = [nvcc] + ARCH + ["-shared", "-o", lib] + objs + ["-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        sys.stderr.write(r.stdout.decode())
        raise RuntimeError("redner_b200: link failed")
    return lib


if __name__ == "__main__":
    defs = [a[2:] for a in sys.argv[1:] if a.startswith("-D")]
    outs = [a[6:] for a in sys.argv[1:] if a.startswith("--out=")]
    extra = [a[7:] for a in sys.argv[1:] if a.startswith("--nvcc=")]
    path = build(force="--force" in sys.argv or bool(outs), double="--f64" in sys.argv, verbose="-v" in sys.argv, defines=defs, out=outs[0] if outs else None,
                 nvcc_flags=extra)
    print(path)
