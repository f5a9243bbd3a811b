#!/usr/bin/env python3
"""Per-stage SASS budget of the warp-collective LV 2-32-32-2 kernels (csrc/k_lv32_wm.cu), on the CPU.

Compiles k_lv32_wm.cu for sm_90a with the library's flags into a temporary directory (or reads a given object), then for the
default forward and adjoint instantiations at N = 65 536 prints the registers, the spill traffic, and the opcode counts of
the stage loop (the smallest loop that holds a tensor-core instruction; HMMA counted by shape: m16n8k16 fp16, m16n8k8 fp16,
m16n8k8 TF32) and of the step loop around it, and the instructions one step issues: the stage loop times its trip count
plus the rest of the step loop (branches taken once per solve or on rare rescales included).  The forward's stage loop runs
6 times per step; the adjoint's runs stages 1..4, and stage 5 with the next step's stage 0 (the state they share) is step
code.  Also counts the instructions of one tanh_quad_z.

    python tools/sass_budget.py                   # compile the working tree's k_lv32_wm.cu
    python tools/sass_budget.py --obj k_lv32_wm.o # read a compiled object (spills then come from LDL/STL counts only)
    python tools/sass_budget.py --fwd-g 1         # the forward with one group per warp (small ensembles)
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "universal_differential_equations_b200", "csrc")
NVCC = os.environ.get("NVCC", "nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v"]

# one tanh_quad_z on registers: every floating-point and MUFU instruction of this kernel belongs to it
TANH_PROBE = r"""
#include "lv32_packed.cuh"
__global__ void tanh_probe(float4 *p) { float4 v = *p; float2 a = make_float2(v.x, v.y), b = make_float2(v.z, v.w);
  b200ude::lv32::tanh_quad_z<0>(a, b); *p = make_float4(a.x, a.y, b.x, b.y); }
"""

# HMMA by shape: m16n8k16 fp16, m16n8k8 fp16, m16n8k8 TF32 (the two m16n8k8 differ only in the .TF32 suffix)
HMMA_SHAPES = [("16816", "HMMA.16816"), ("1688", "HMMA.1688"), ("1688tf32", "HMMA.1688.F32.TF32")]
COLUMNS = [
    ("16816", ()),
    ("1688", ()),
    ("1688tf32", ()),
    ("MOVM", ("MOVM",)),
    ("MUFU", ("MUFU",)),
    ("FP32", ("FFMA", "FMUL", "FADD", "FMNMX")),
    ("FSEL", ("FSEL",)),
    ("LDS", ("LDS", "LDSM")),
    ("STS", ("STS",)),
    ("SHFL", ("SHFL",)),
    ("LDG", ("LDG",)),
    ("STG", ("STG",)),
    ("BRA/BRX", ("BRA", "BRX")),
    ("MOV", ("MOV", "IMAD.MOV")),
    ("LDL/STL", ("LDL", "STL")),
]
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z0-9_.]+)([^;]*);")
LABEL = re.compile(r"^\s*(\.L_x_\d+):")
TARGET = re.compile(r"BRA\S*\s+(?:`\((\.L_x_\d+)\)|(0x[0-9a-f]+))")  # label or absolute address, by cuobjdump version


def sh(cmd, **kw):
    r = subprocess.run(cmd, capture_output=True, text=True, **kw)
    if r.returncode != 0:
        sys.exit(f"{' '.join(cmd)} failed:\n{r.stdout}\n{r.stderr}")
    return r.stdout + r.stderr


def functions(sass):
    """name -> (instructions [(addr, opcode, text)], labels {label: addr})"""
    out, name, lines = {}, None, []
    for ln in sass.splitlines() + ["Function : <end>"]:
        m = re.search(r"Function : (\S+)", ln)
        if m:
            if name:
                insns, labels, pending = [], {}, []
                for l2 in lines:
                    lm = LABEL.match(l2)
                    if lm:
                        pending.append(lm.group(1))
                        continue
                    im = INSN.search(l2)
                    if im:
                        addr = int(im.group(1), 16)
                        for p in pending:
                            labels[p] = addr
                        pending = []
                        insns.append((addr, im.group(3), l2.strip()))
                out[name] = (insns, labels)
            name, lines = m.group(1), []
        else:
            lines.append(ln)
    return out


def loops(insns, labels):
    """(start, end) address ranges of the backward branches"""
    res = []
    for addr, op, text in insns:
        if op.startswith("BRA"):
            t = TARGET.search(text)
            dst = labels.get(t.group(1)) if t and t.group(1) else (int(t.group(2), 16) if t else None)
            if dst is not None and dst <= addr:
                res.append((dst, addr))
    return sorted(set(res), key=lambda r: r[1] - r[0])


def count(insns, lo, hi):
    c = collections.Counter()
    n = 0
    for addr, op, _ in insns:
        if lo <= addr <= hi:
            n += 1
            base = op.split(".")[0]
            if base == "HMMA":
                c[next(col for col, pre in reversed(HMMA_SHAPES) if op.startswith(pre))] += 1
                continue
            for col, ops in COLUMNS:
                if base in ops or op in ops or (col == "MOV" and op.startswith("IMAD.MOV")):
                    c[col] += 1
                    break
    c["total"] = n
    return c


def row(label, c):
    return f"  {label:34s} {c['total']:6d} " + " ".join(f"{c[col]:>7d}" for col, _ in COLUMNS)


STAGE_TRIPS = {"forward": 6, "adjoint": 4}   # stage-loop iterations per step


def report(fname, funcs, res, spills, trips):
    insns, labels = funcs[fname]
    hm = [a for a, op, _ in insns if op.startswith("HMMA")]
    ls = loops(insns, labels)
    stage = next((l for l in ls if any(l[0] <= a <= l[1] for a in hm)), None)
    print(f"{fname}")
    print(f"  registers {res.get('REG', '?')}, local memory {res.get('LOCAL', '?')} B, {spills}")
    print(f"  {'region':34s} {'insns':>6s} " + " ".join(f"{col:>7s}" for col, _ in COLUMNS))
    if stage is None:
        print("  (no loop holds an HMMA)")
        return
    print(row("stage loop", count(insns, *stage)))
    for l in ls:
        if stage[0] <= l[0] and l[1] <= stage[1] and l != stage:
            print(row(f"  nested loop {l[0]:#x}..{l[1]:#x}", count(insns, *l)))
    outer = next((l for l in ls if l[0] <= stage[0] and stage[1] <= l[1] and l != stage), None)
    if outer:
        cs, co = count(insns, *stage), count(insns, *outer)
        print(row("step loop (stage loop included)", co))
        per_step = collections.Counter({k: trips * cs[k] + co[k] - cs[k] for k in co})
        print(row(f"per step: {trips} x stage loop + rest", per_step))
    print(row("whole kernel", count(insns, 0, 1 << 40)))


def resources(obj):
    res = {}
    cur = None
    for ln in sh(["cuobjdump", "-res-usage", obj]).splitlines():
        m = re.search(r"Function (\S+):", ln)
        if m:
            cur = m.group(1)
            continue
        if cur:
            res[cur] = dict(re.findall(r"(REG|STACK|SHARED|LOCAL):(\d+)", ln))
            cur = None
    return res


def spill_lines(log):
    """mangled name -> 'N bytes spill stores, M bytes spill loads' from ptxas -v"""
    out, cur = {}, None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur:
            out[cur] = f"spill stores {m.group(1)} B, spill loads {m.group(2)} B"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--obj", help="read this compiled k_lv32_wm.o instead of compiling")
    ap.add_argument("--fwd-g", type=int, default=2, help="groups per warp of the forward: 2 at N = 65 536 (B200UDE_WM_G)")
    ap.add_argument("--dump", help="also write the full SASS here")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        spills, tanh = {}, None
        if a.obj:
            obj = a.obj
        else:
            obj = os.path.join(tmp, "k_lv32_wm.o")
            spills = spill_lines(sh([NVCC] + FLAGS + ["-c", "-o", obj, os.path.join(CSRC, "k_lv32_wm.cu")]))
            probe = os.path.join(tmp, "probe.cu")
            with open(probe, "w") as f:
                f.write(TANH_PROBE)
            pobj = os.path.join(tmp, "probe.o")
            sh([NVCC] + FLAGS + ["-I", CSRC, "-c", "-o", pobj, probe])
            pf = functions(sh(["cuobjdump", "-sass", pobj]))
            insns = next(v for k, v in pf.items() if "tanh_probe" in k)[0]
            tanh = count(insns, 0, 1 << 40)
        sass = sh(["cuobjdump", "-sass", obj])
        if a.dump:
            with open(a.dump, "w") as f:
                f.write(sass)
        funcs = functions(sass)
        res = resources(obj)
    want = {
        "forward": f"forward_kernelILi0ELi{a.fwd_g}ELi2ELi2EE",
        "adjoint": "adjoint_kernelILi0ELi2ELi1ELi1EE",
    }
    for what, key in want.items():
        fname = next((k for k in funcs if key in k), None)
        if fname is None:
            sys.exit(f"no {what} instantiation {key} in the object")
        insns = funcs[fname][0]
        sp = spills.get(fname) or f"{sum(1 for _, op, _ in insns if op.startswith(('STL', 'LDL')))} LDL/STL instructions"
        print(f"== {what}: ", end="")
        report(fname, funcs, res.get(fname, {}), sp, STAGE_TRIPS[what])
    if tanh is not None:
        fp = tanh["FP32"] + tanh["MUFU"]
        print(f"== tanh_quad_z<0> (four values): {fp} instructions: {tanh['MUFU']} MUFU, {tanh['FP32']} FFMA/FMUL/FADD/FMNMX")


if __name__ == "__main__":
    main()
