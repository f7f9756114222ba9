"""Instruction census of the backward blend's visit loop, read from the SASS (no GPU needed).

    python scripts/bwd_sass_census.py [--src DIR] [--arm NAME] [--out profiles/h100/bwd_reduce.jsonl]

Compiles DIR/gaussianavatars_b200/csrc/blend.cu (default: this checkout) for sm_90a with the library's flags and
`-Xptxas -v`, disassembles it with source lines (cuobjdump -xelf, nvdisasm -g) and, for blend_backward_kernel<false,
false> and <true, false>, finds the two visit loops (`while (todo)` of backward_task: K = 2 for heavy tiles, K = 4 for
light ones) as the innermost loops that hold the walk's FLO (or UFLO).  Every instruction of a loop is put in one class:

  reduction  RED, the lines of the row-reduction lambda (reduce_step or send_batch) and of the reduction's pipeline
             state, and the STS / address arithmetic of the row stores;
  walk       VOTE, FLO, BREV, POPC, SHFL, BAR, WARPSYNC, BRA, BSSY, BSYNC (and their uniform-datapath forms) and the
             record loads (LDS) elsewhere;
  band       FFMA, FMUL, FADD, FMNMX, MUFU, FSETP, FSEL elsewhere (the band math and the gradient rows' arithmetic);
  other      integer, select and move instructions elsewhere.

`static` counts the whole loop.  `per_visit` counts the instructions one visit with all K bands live issues: the
partial-band blocks (BandLoop, the blocks with fewer MUFU than the largest) are left out, and the lines of a reduction
lambda that runs once per B visits, and the blocks made of them alone, are weighted 1/B (send_batch: B = 3).  Registers, shared memory and spills come
from ptxas.  One JSON line per (kernel, K) goes to stdout and, with --out, is appended there.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from gaussianavatars_b200.build import ARCH, COMMON, _nvcc  # noqa: E402

KERNELS = {"blend_backward_kernel<false, false>": "blend_backward_kernelILb0ELb0E",
           "blend_backward_kernel<true, false>": "blend_backward_kernelILb1ELb0E"}
# reduction lambda -> visits per call
LAMBDAS = {"reduce_step": 1, "send_batch": 3}
# reduction pipeline state updated once per visit (either arm)
STATE = re.compile(r"^\s*(id2 = id1;|id1 = id0;|par \^= 1;|if \(my_slot == fill\)|if \(\+\+fill == 3\)|fill = 0;)")
ROW = re.compile(r"^\s*(float\* row = |if constexpr \(DA\) row\[|row\[\d \* ROWS_STRIDE\])")
WALK = ("VOTE", "FLO", "BREV", "POPC", "SHFL", "BAR", "WARPSYNC", "BRA", "BSSY", "BSYNC")
BAND = ("FFMA", "FMUL", "FADD", "FMNMX", "MUFU", "FSETP", "FSEL")


def source_lines(blend_cu):
    """(lines of the reduction lambda, lines of the reduction's per-visit state, lines of the row stores, visits per
    call of the lambda) of blend.cu."""
    text = open(blend_cu).read().split("\n")
    lam, state, row, per = set(), set(), set(), 1
    for i, line in enumerate(text, 1):
        m = re.match(r"^\s*auto (\w+) = \[&\]", line)
        if m and m.group(1) in LAMBDAS:
            per = LAMBDAS[m.group(1)]
            j = i
            while not text[j - 1].startswith("  };"):
                lam.add(j)
                j += 1
            lam.add(j)
        elif STATE.match(line):
            state.add(i)
        elif ROW.match(line):
            row.add(i)
    return lam, state, row, per


def compile_blend(blend_cu, tmp):
    obj = os.path.join(tmp, "blend.o")
    cmd = [_nvcc(), *ARCH, *COMMON, "-Xptxas", "-v", "-ccbin", "/usr/bin/g++", "-c", blend_cu, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(r.stderr)
    res, cur = {}, None
    for line in r.stderr.split("\n"):
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            res.setdefault(cur, {}).update(stack=int(m.group(1)), spill_stores=int(m.group(2)),
                                           spill_loads=int(m.group(3)))
        m = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", line)
        if m:
            res.setdefault(cur, {}).update(registers=int(m.group(1)), smem=int(m.group(2)))
    cuobjdump = os.path.join(os.path.dirname(_nvcc()), "cuobjdump") if os.path.isabs(_nvcc()) else "cuobjdump"
    subprocess.run([cuobjdump, "-xelf", "all", obj], cwd=tmp, check=True, capture_output=True)
    cubin = [f for f in os.listdir(tmp) if f.endswith(".cubin")][0]
    nvdisasm = os.path.join(os.path.dirname(cuobjdump), "nvdisasm") if os.path.isabs(cuobjdump) else "nvdisasm"
    sass = subprocess.run([nvdisasm, "-g", "-c", os.path.join(tmp, cubin)], check=True, capture_output=True,
                          text=True).stdout
    return res, sass


def functions(sass):
    """{mangled name: (instructions [(opcode, text, source line)], {label: index of the instruction it marks},
    {index: True where a label precedes it})}"""
    out, cur, line = {}, None, None
    pending = []
    for raw in sass.split("\n"):
        m = re.match(r"^\.text\.(\w+):", raw)
        if m:
            cur = out.setdefault(m.group(1), ([], {}, set()))
            pending = []
            continue
        if cur is None:
            continue
        m = re.search(r'//## File ".*blend\.cu", line (\d+)', raw)
        if m:
            line = int(m.group(1))
            continue
        if "//## File" in raw:
            line = None
            continue
        m = re.match(r"^(\.L_x_\d+):", raw)
        if m:
            pending.append(m.group(1))
            continue
        m = re.match(r"^\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", raw)
        if m:
            body = m.group(1)
            op = re.sub(r"^@!?U?P\w+\s+", "", body).split()[0]
            ins, labels, led = cur
            for lab in pending:
                labels[lab] = len(ins)
                led.add(len(ins))
            pending = []
            ins.append((op, body, line))
    return out


def visit_loops(ins, labels):
    """[head, back-edge] index ranges of the innermost loops that hold a FLO (the walk's __ffs)."""
    loops = []
    for i, (op, body, _line) in enumerate(ins):
        m = re.search(r"`\((\.L_x_\d+)\)", body)
        if op.startswith("BRA") and m and labels.get(m.group(1), i + 1) <= i:
            loops.append((labels[m.group(1)], i))
    found = set()
    for i, (op, _b, _l) in enumerate(ins):
        if op.startswith(("FLO", "UFLO")):
            inner = [lp for lp in loops if lp[0] <= i <= lp[1]]
            if inner:
                found.add(min(inner, key=lambda lp: lp[1] - lp[0]))
    return sorted(found)


def classify(op, line, red, row):
    base = op.split(".")[0]
    if base in ("RED", "REDG", "ATOM", "ATOMG") or line in red or (line in row and not base.startswith("F")):
        return "reduction"
    if base in WALK or base[1:] in WALK and base[0] == "U" or base == "LDS":
        return "walk"
    if base in BAND:
        return "band"
    return "other"


def loop_census(ins, led, lo, hi, lam, state, row, per):
    """(K, static counts, per-visit counts, per-visit reduction opcodes) of the loop ins[lo .. hi]."""
    blocks, start = [], lo  # basic blocks: a label or the instruction after a branch starts one
    for i in range(lo + 1, hi + 1):
        if i in led or ins[i - 1][0].startswith(("BRA", "EXIT")):
            blocks.append((start, i - 1))
            start = i
    blocks.append((start, hi))
    mufu = [sum(ins[i][0].startswith("MUFU") for i in range(b0, b1 + 1)) for b0, b1 in blocks]
    full = max(mufu)
    static, visit, ops = collections.Counter(), collections.Counter(), collections.Counter()
    for (b0, b1), mu in zip(blocks, mufu):
        known = [ins[i][2] for i in range(b0, b1 + 1) if ins[i][2] is not None]
        batch = bool(known) and all(line in lam for line in known)  # a block of the lambda alone (the RED's too)
        for i in range(b0, b1 + 1):
            op, _body, line = ins[i]
            c = classify(op, line, lam | state, row)
            static[c] += 1
            if 0 < mu < full:  # a partial-band block
                continue
            w = 1.0 / per if batch or line in lam else 1.0
            visit[c] += w
            if c == "reduction":
                ops[op if op.startswith("LDS") else op.split(".")[0]] += w
    return full // 2, static, visit, ops  # one ex2 and one rcp per band


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--src", default=ROOT, help="checkout whose blend.cu is counted")
    ap.add_argument("--arm", default="branch", help="label of the lines written")
    ap.add_argument("--out", default=None, help="JSONL file the lines are appended to")
    a = ap.parse_args()
    blend_cu = os.path.join(a.src, "gaussianavatars_b200", "csrc", "blend.cu")
    lam, state, row, per = source_lines(blend_cu)
    with tempfile.TemporaryDirectory() as tmp:
        res, sass = compile_blend(blend_cu, tmp)
    funcs = functions(sass)
    lines = []
    for name, key in KERNELS.items():
        mangled = [f for f in funcs if key in f][0]
        ins, labels, led = funcs[mangled]
        loops = visit_loops(ins, labels)
        if len(loops) != 2:
            raise RuntimeError(f"{name}: expected two visit loops, found {len(loops)}")
        for lo, hi in loops:
            k, static, visit, ops = loop_census(ins, led, lo, hi, lam, state, row, per)
            lines.append({
                "kind": "sass_census", "arm": a.arm, "kernel": name, "K": k,
                "tile": "heavy" if k == 2 else "light", "visits_per_reduction": per,
                "static": dict(sorted(static.items()), total=sum(static.values())),
                "per_visit": {c: round(v, 2) for c, v in sorted(visit.items())} | {
                    "total": round(sum(visit.values()), 2)},
                "per_visit_reduction_ops": {o: round(v, 2) for o, v in sorted(ops.items())},
                **res[mangled]})
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        with open(a.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
