#!/usr/bin/env python3
"""Instruction budget of K1's loops, read from the SASS of a built library:
python tools/k1_sass_budget.py [libbftq.so] [--json]

Every backward branch of `rsa_verify_r32_kernel` closes a loop [target, branch].  For each loop it prints the modelled
FMA-pipe cycles per warp (4 per IMAD.WIDE*, 2 per other IMAD*: the 64-bit-result forms issue at half the IMAD rate,
DESIGN.md §4), the other IMADs by kind, the ALU-pipe instruction counts and the SHFLs.  The squaring loop (mont_sqr's
owner loop, rsa_square_r32.cuh) is the innermost loop whose body holds 2 x 337 IMAD.WIDE.U32.X; an outer loop counts
the bodies of the loops it holds once."""
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "rsa_verify_r32_kernel"
SQR_WIDEX = 2 * 337
ALU = ("IADD3", "LOP3", "SEL", "SHF", "ISETP", "PLOP3", "MOV", "LEA", "FLO", "POPC", "BMSK", "IABS", "IMNMX", "P2R", "R2P")


def kernel_sass(so, kernel=KERNEL):
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    blk = [b for b in sass.split("Function :") if kernel in b.split("\n")[0]]
    assert len(blk) == 1, (kernel, len(blk))
    # (address, opcode with modifiers, operands) without the guard predicate
    ins = []
    for m in re.finditer(r"/\*([0-9a-f]{4,5})\*/\s+([^;]+);", blk[0]):
        text = m.group(2).strip()
        if text.startswith("@"):
            text = text.split(None, 1)[1]
        op, _, args = text.partition(" ")
        ins.append((int(m.group(1), 16), op, args.strip()))
    return ins


def imad_kind(op, args):
    """the job a non-wide IMAD does: a carry limb, a copy or a product"""
    a = [x.strip() for x in args.split(",")]
    if op.startswith("IMAD.X") and len(a) >= 4 and a[1] == "RZ" and a[2] == "RZ":
        return "carry_to_value" if a[3] == "RZ" else "carry_add"
    if op.startswith("IMAD.MOV"):
        return "copy"
    return "other"


def classify(body):
    wide = sum(op.startswith("IMAD.WIDE") for _, op, _ in body)
    widex = sum(op.startswith("IMAD.WIDE.U32.X") for _, op, _ in body)
    kinds = {"carry_add": 0, "carry_to_value": 0, "copy": 0, "other": 0}
    for _, op, args in body:
        if op.startswith("IMAD") and not op.startswith("IMAD.WIDE"):
            kinds[imad_kind(op, args)] += 1
    other = sum(kinds.values())
    alu = {}
    for _, op, _ in body:
        base = op.split(".")[0]
        if base in ALU:
            alu[base] = alu.get(base, 0) + 1
    shfl = sum(op.startswith("SHFL") for _, op, _ in body)
    return {"instructions": len(body), "imad_wide": wide, "imad_wide_x": widex, "imad_other": other, "imad_other_by_kind": kinds,
            "fma_cycles": 4 * wide + 2 * other, "alu": dict(sorted(alu.items())), "alu_total": sum(alu.values()), "shfl": shfl}


def loops(ins):
    out = []
    for addr, op, args in ins:
        if op.startswith("BRA"):
            t = re.search(r"0x([0-9a-f]+)", args)
            if t and int(t.group(1), 16) < addr:
                start = int(t.group(1), 16)
                out.append((start, addr))
    res = []
    for start, end in sorted(out):
        body = [i for i in ins if start <= i[0] <= end]
        res.append({"start": hex(start), "end": hex(end), **classify(body)})
    return res


def budget(so):
    """{"loops": [...], "squaring": the squaring loop's entry}"""
    ls = loops(kernel_sass(so))
    sq = [l for l in ls if l["imad_wide_x"] == SQR_WIDEX]
    assert sq, [(l["start"], l["imad_wide_x"]) for l in ls]
    return {"loops": ls, "squaring": min(sq, key=lambda l: l["instructions"])}     # the innermost one


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    so = args[0] if args else os.path.join(ROOT, "bftkv_b200", "libbftq.so")
    b = budget(so)
    if "--json" in sys.argv:
        print(json.dumps(b, indent=1))
        return
    print("loops of %s (FMA cycles per warp: 4 per IMAD.WIDE*, 2 per other IMAD*)" % KERNEL)
    print("%-17s %6s %6s %6s %6s %7s %6s %5s" % ("range", "instr", "wide", "imad", "fma_cy", "alu", "shfl", "sqr"))
    for l in b["loops"]:
        print("%-17s %6d %6d %6d %6d %7d %6d %5s" % (l["start"] + "-" + l["end"], l["instructions"], l["imad_wide"], l["imad_other"],
                                                     l["fma_cycles"], l["alu_total"], l["shfl"], "<-" if l is b["squaring"] else ""))
    s = b["squaring"]
    print("\nsquaring loop %s-%s, one trip = two owner steps:" % (s["start"], s["end"]))
    print("  IMAD.WIDE* %d (IMAD.WIDE.U32.X %d)  ->  %d FMA cycles" % (s["imad_wide"], s["imad_wide_x"], 4 * s["imad_wide"]))
    k = s["imad_other_by_kind"]
    print("  other IMAD* %d  ->  %d FMA cycles: carry limb adds (IMAD.X R, RZ, RZ, R) %d, carries to values (IMAD.X R, RZ, RZ, RZ) %d, "
          "copies (IMAD.MOV) %d, other %d" % (s["imad_other"], 2 * s["imad_other"], k["carry_add"], k["carry_to_value"], k["copy"], k["other"]))
    print("  FMA cycles %d, of which not multiplies %.1f %%" % (s["fma_cycles"], 100.0 * 2 * s["imad_other"] / s["fma_cycles"]))
    print("  ALU %d: %s" % (s["alu_total"], ", ".join("%s %d" % kv for kv in s["alu"].items())))
    print("  SHFL %d, instructions %d" % (s["shfl"], s["instructions"]))


if __name__ == "__main__":
    main()
