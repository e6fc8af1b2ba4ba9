"""Per-evaluation instruction mix of K1q's Form W full-tile path, read from the SASS (needs nvcc and cuobjdump, no GPU).

    python examples/kw_sass.py [--src senweaver-ide_b200/csrc/apo_compact.cu] [--recip] [--dump FILE]

Compiles apo_compact.cu with the Makefile's nvcc flags into a temporary cubin, takes the Form W instantiation of
k_reward9q, and walks its full-tile path (n == TILE): from the end of the short-tile loop, which branches past it, to that
branch's target.  Without --recip the generic-division blocks (the ones holding MUFU.RCP64H, taken only for masks whose
reciprocal is flagged negative) are left out.  Counts are divided by the evaluations one pass covers (EPT)."""
import argparse
import collections
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "senweaver-ide_b200", "csrc")

CLASSES = (
    ("integer", ("IMAD", "IADD3", "IADD", "VIADD", "LOP3", "LOP", "SHF", "SHL", "SHR", "LEA", "PRMT", "SEL", "IMNMX", "VIMNMX",
                 "ISETP", "BFE", "BFI", "FLO", "POPC", "MOV", "IABS")),
    ("LDS", ("LDS",)),
    ("FP64", ("DADD", "DMUL", "DFMA", "DSETP")),
    ("conversion", ("F2F", "F2I", "I2F", "I2I", "F2FP")),
)


def nvflags():
    with open(os.path.join(CSRC, "Makefile")) as f:
        text = f.read()
    arch = re.search(r"^ARCH\s*=\s*(.*)$", text, re.M).group(1).split()
    flags = re.search(r"^NVFLAGS\s*=\s*(.*)$", text, re.M).group(1).replace("$(ARCH)", " ".join(arch)).split()
    return [f for f in flags if f not in ("-lineinfo", "-Xptxas", "-v")]


def sass_of(src):
    with tempfile.TemporaryDirectory() as d:
        cubin = os.path.join(d, "k.cubin")
        subprocess.run(["nvcc", *nvflags(), "-cubin", "-o", cubin, os.path.basename(src)], cwd=os.path.dirname(src), check=True)
        return subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout


def kernels(sass):
    out, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and name:
            out[name].append((int(m.group(1), 16), m.group(2).strip()))
    return out


def opcode(text):
    t = re.sub(r"^@!?U?P\w+\s+", "", text)
    return t.split()[0]


def branch_target(text):
    m = re.search(r"\bBRA\b(?:\s+!?U?P\w+,)?\s+(0x[0-9a-f]+)", text)
    return int(m.group(1), 16) if m else None


def full_tile_path(ins, skip_generic):
    """instructions of the n == TILE path; the short-tile loop ends in `BRA <join>` just before it"""
    addr = [a for a, _ in ins]
    ops = [opcode(t) for _, t in ins]
    f2i = [i for i, o in enumerate(ops) if o.startswith("F2I.S64")]
    # the first run of four conversions within 40 instructions belongs to the full-tile path's first group
    first = next(i for i in range(len(f2i) - 3) if f2i[i + 3] - f2i[i] < 40)
    bra = max(i for i in range(f2i[first]) if ops[i] == "BRA" and not ins[i][1].startswith("@")
              and branch_target(ins[i][1]) > addr[f2i[first]])
    start, end = bra + 1, addr.index(branch_target(ins[bra][1]))
    keep = [True] * len(ins)
    if skip_generic:
        for i in range(start, end):
            t = branch_target(ins[i][1])
            if ops[i] == "BRA" and ins[i][1].startswith("@") and t and t > addr[i]:
                j = addr.index(t)
                if any(ops[k].startswith("MUFU.RCP64H") for k in range(i + 1, j)):
                    for k in range(i + 1, j):
                        keep[k] = False
    return [ins[i] for i in range(start, end) if keep[i]]


def classify(op):
    base = op.split(".")[0]
    for cls, names in CLASSES:
        if base in names:
            return cls
    return "rest"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=os.path.join(CSRC, "apo_compact.cu"))
    ap.add_argument("--recip", action="store_true", help="the recip instantiation (no generic division)")
    ap.add_argument("--dump", help="write the path's SASS to this file")
    a = ap.parse_args()
    ks = kernels(sass_of(os.path.abspath(a.src)))
    pat = re.compile(r"_ZN3apo10k_reward9qILi(\d+)ELi(\d+)ELi(\d+)ELb%dELi0ELb1EEEvNS_8KqParamsE" % (1 if a.recip else 0))
    (name, ins), = [(n, i) for n, i in ks.items() if pat.fullmatch(n)]
    cw, ept, stages = (int(x) for x in pat.fullmatch(name).groups())
    path = full_tile_path(ins, not a.recip)
    if a.dump:
        with open(a.dump, "w") as f:
            f.writelines(f"/*{ad:05x}*/ {t}\n" for ad, t in path)
    by_cls, by_op = collections.Counter(), collections.Counter()
    for _, t in path:
        op = opcode(t)
        by_cls[classify(op)] += 1
        by_op[op.split(".")[0]] += 1
    print(f"{name}: CW={cw} EPT={ept} STAGES={stages}, full-tile path {len(path)} instructions for {ept} evaluations")
    print(f"{'class':<12}{'per evaluation':>16}")
    for cls in [c for c, _ in CLASSES] + ["rest"]:
        print(f"{cls:<12}{by_cls[cls] / ept:>16.2f}")
    print(f"{'total':<12}{len(path) / ept:>16.2f}")
    print("by opcode:", ", ".join(f"{k} {v / ept:.2f}" for k, v in sorted(by_op.items(), key=lambda kv: -kv[1])))


if __name__ == "__main__":
    main()
