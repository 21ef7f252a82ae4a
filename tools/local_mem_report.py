#!/usr/bin/env python
"""Local-memory report of the render kernels: registers, stack frame, spills and the static LDL / STL instructions of every hot
kernel, with the source lines they come from.  Needs nvcc and nvdisasm, no GPU.

    python tools/local_mem_report.py                     # the lean instantiation (the one C3 and C4 run)
    python tools/local_mem_report.py --tu diffuse        # its diffuse-only refinement (the one C2 runs)
    python tools/local_mem_report.py --tu lean diffuse general det --top 8
    python tools/local_mem_report.py --root OTHER_CHECKOUT   # the same report for another tree (before / after)

Each translation unit is compiled to a cubin with the flags of redner_b200/build.py plus -Xptxas -v, and the cubin is disassembled
with --print-line-info-inline.  Every LDL / STL is attributed to its innermost source line and to the chain of call sites it was
inlined through.  "tex" counts the LDL / STL whose chain passes through a texture lookup of rb_material.cuh (tex_eval, the
trilinear fetch and the mat_* helpers).  Out-of-line device functions (tex_eval_mip, bvh_trace_impl) are listed as rows of
their own: their LDL / STL run inside whichever kernel calls them."""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TUS = {"lean": "rb_kernels_lean.cu", "diffuse": "rb_kernels_diffuse.cu", "general": "rb_kernels.cu", "det": "rb_kernels_det.cu"}
HOT = ["k_forward", "k_bwd_trace", "k_bwd_sec_pick", "k_bwd_sec_shade", "k_bwd_sweep", "k_primary_edge", "k_prim_edge_project"]
TEX_FUNCS = ["bilerp_tap", "bilerp_eval", "tex_level", "tex_eval_mip", "tex_eval", "mat_diffuse", "mat_specular", "mat_roughness",
             "mat_normal_tex"]


def tex_line_ranges(csrc):
    """Line ranges of the texture-lookup functions of rb_material.cuh (from the signature to the closing brace at column 0)."""
    lines = open(os.path.join(csrc, "rb_material.cuh")).read().split("\n")
    ranges, start = [], None
    sig = re.compile(r"^(RB_\w+|struct)\s.*?\b(%s)\s*\(" % "|".join(TEX_FUNCS))
    for i, ln in enumerate(lines, 1):
        if start is None and sig.match(ln):
            start = i
        if start is not None and ln.startswith("}"):
            ranges.append((start, i))
            start = None
    return ranges


def compile_tu(root, tu, tmp):
    csrc = os.path.join(root, "redner_b200", "csrc")
    cubin = os.path.join(tmp, tu + ".cubin")
    # the flags of redner_b200/build.py for the render kernels
    cmd = ["/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc", "-gencode", "arch=compute_90a,code=sm_90a",
           "-O3", "-std=c++17", "-lineinfo", "-I", os.path.join(root, "include"), "-fmad=true", "-prec-div=false", "-prec-sqrt=false",
           "-Xptxas", "-v", "-cubin", os.path.join(csrc, TUS[tu]), "-o", cubin]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.exit(r.stdout)
    nvdisasm = os.path.join(os.path.dirname(cmd[0]), "nvdisasm") if os.path.isabs(cmd[0]) else "nvdisasm"
    sass = subprocess.run([nvdisasm, "--print-line-info-inline", "-c", cubin], stdout=subprocess.PIPE, check=True, text=True).stdout
    return r.stdout, sass


def parse_ptxas(text):
    """mangled name -> dict(regs, frame, spill_st, spill_ld)"""
    props, cur = {}, None
    for ln in text.split("\n"):
        m = re.search(r"Function properties for (\S+)", ln)
        if m:
            cur = props.setdefault(m.group(1), dict(regs=None, frame=0, spill_st=0, spill_ld=0))
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur is not None:
            cur.update(frame=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
            continue
        m = re.search(r"Used (\d+) registers", ln)
        if m and cur is not None:
            cur["regs"] = int(m.group(1))
    return props


LOC = re.compile(r'"([^"]+)", line (\d+)')


def parse_sass(sass):
    """mangled name -> list of (opcode, [(file, line) innermost first]) for every LDL / STL"""
    out, fn, chain, newgroup = {}, None, [], True
    for ln in sass.split("\n"):
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", ln)
        if m:
            fn, chain = m.group(1), []
            out.setdefault(fn, [])
            continue
        if fn is None:
            continue
        if ln.lstrip().startswith("//## File"):
            if newgroup:  # the first line of a group carries the whole inline chain
                chain = [(os.path.basename(f), int(l)) for f, l in LOC.findall(ln)]
                newgroup = False
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", ln)
        if m:
            newgroup = True
            op = m.group(1).split(".")[0]
            if op in ("LDL", "STL"):
                out[fn].append((op, list(chain)))
    return out


def demangled_short(name):
    for k in HOT + ["tex_eval_mip", "bvh_trace_impl"]:
        if re.search(r"\d%s(?![a-z_])" % k, name):
            return k + ("<any>" if "ILb1E" in name else "<closest>" if "ILb0E" in name else "")
    return None


def report(root, tu, top):
    csrc = os.path.join(root, "redner_b200", "csrc")
    tex = tex_line_ranges(csrc)
    is_tex = lambda f, l: f == "rb_material.cuh" and any(a <= l <= b for a, b in tex)
    with tempfile.TemporaryDirectory() as tmp:
        ptxas, sass = compile_tu(root, tu, tmp)
    props, locs = parse_ptxas(ptxas), parse_sass(sass)
    rows = []
    for name, p in props.items():
        short = demangled_short(name)
        if short is None:
            continue
        ins = locs.get(name, [])
        if short not in HOT and not ins and p["frame"] == 0:
            continue
        rows.append((HOT.index(short) if short in HOT else len(HOT), short, name, p, ins))
    rows.sort()
    print("== %s (%s)" % (TUS[tu], root))
    print("%-22s %5s %6s %13s %6s %6s %6s" % ("function", "regs", "frame", "spill st/ld B", "LDL", "STL", "tex"))
    for _, short, name, p, ins in rows:
        n_ld = sum(1 for o, _ in ins if o == "LDL")
        n_st = len(ins) - n_ld
        n_tex = sum(1 for _, c in ins if any(is_tex(f, l) for f, l in c))
        print("%-22s %5s %6d %6d / %-6d %6d %6d %6d" % (short, p["regs"] if p["regs"] is not None else "-", p["frame"], p["spill_st"],
                                                         p["spill_ld"], n_ld, n_st, n_tex))
    if top:
        for _, short, name, p, ins in rows:
            if not ins:
                continue
            print("-- %s: top source lines of its %d LDL / STL (innermost line <- call sites)" % (short, len(ins)))
            cnt = collections.Counter(" <- ".join("%s:%d" % fl for fl in c[:3]) if c else "?" for _, c in ins)
            for k, v in cnt.most_common(top):
                print("   %5d  %s" % (v, k))
    print()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--root", default=os.path.dirname(HERE), help="repository tree to compile (default: this one)")
    ap.add_argument("--tu", nargs="+", default=["lean"], choices=sorted(TUS))
    ap.add_argument("--top", type=int, default=0, help="print the N most frequent source lines of the LDL / STL of each function")
    a = ap.parse_args()
    for tu in a.tu:
        report(os.path.abspath(a.root), tu, a.top)


if __name__ == "__main__":
    main()
