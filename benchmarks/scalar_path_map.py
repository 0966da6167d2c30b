"""Where the calls and the local-memory accesses of a NUTS kernel sit: every CALL, LDL and STL of the SASS of one or more
k_nuts instantiations, sorted by how often it runs, from the line information that csrc/Makefile compiles in (-lineinfo).

    python benchmarks/scalar_path_map.py BUILD_DIR [--kernel UNIT:MANGLED_NAME ...] [--csrc DIR] > map.md

BUILD_DIR holds the family objects of one build (csrc/build/fam_*.o).  For each instruction the script reads the chain of
source locations it was inlined through (nvdisasm -gi) and puts it into one of these groups:
- leaf loop: a frame lies in the body of the leaf loop of NutsMachine::transition (`for (unsigned k = 1; …)`), i.e. it
  can run once per leaf of the tree;
- transition level: otherwise a frame lies in NutsMachine::transition or in the loop over transitions of
  NutsMachine::run — it runs once per transition (the momentum draw, the doubling-level merge, the draw output);
- once per call: everything else in the kernel body (chain load and store, the step-size search, set-up);
- inside an out-of-line body: the instruction belongs to a subroutine (a noinline math body or a CUDA division / square
  root slow path) and runs whenever that subroutine is called.
The source ranges come from csrc/nuts_machine.cuh (--csrc; the tree the objects were built from)."""
import argparse
import collections
import glob
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynamichmc.jl_b200", "csrc")
# C2 (1000-dim standard normal) and C5 (1000-dim diagonal normal): EPL 8, four warps, diagonal metric, one chain per CTA
DEFAULT_KERNELS = ["fam_0_0:_ZN4dhmc6k_nutsILi8ELi0ELi4ELb0ELi1ELb0EEEvNS_5KArgsE",
                   "fam_1_0:_ZN4dhmc6k_nutsILi8ELi1ELi4ELb0ELi1ELb0EEEvNS_5KArgsE"]
GROUPS = ["leaf loop", "transition level", "once per call", "inside an out-of-line body"]


def block_range(lines, pattern):
    """1-based first and last line of the brace block that opens on the first line matching `pattern`."""
    start = next(i for i, l in enumerate(lines) if re.search(pattern, l))
    depth = 0
    for i in range(start, len(lines)):
        depth += lines[i].count("{") - lines[i].count("}")
        if depth == 0 and i > start:
            return start + 1, i + 1
    raise ValueError(pattern)


def source_ranges(csrc):
    lines = open(os.path.join(csrc, "nuts_machine.cuh")).read().splitlines()
    return dict(leaf=block_range(lines, r"for \(unsigned k = 1; k <= nleaves; \+\+k\)"),
                transition=block_range(lines, r"DHMC_M void transition\("),
                run_loop=block_range(lines, r"for \(int n = 0; n < N; \+\+n\)"))


def disassemble(obj, tmp):
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(obj)], cwd=tmp, check=True, capture_output=True)
    cubin = glob.glob(os.path.join(tmp, "*.cubin"))
    assert len(cubin) == 1, cubin
    out = subprocess.run(["nvdisasm", "-gi", cubin[0]], check=True, capture_output=True, text=True).stdout
    os.remove(cubin[0])
    return out


FRAME = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def short_callee(s):
    m = re.search(r"\$_ZN\w*?\d+(dm_\w+?)E", s) or re.search(r"\$__cuda_sm20_(\w+)", s) or re.search(r"(dm_\w+)", s)
    return m.group(1) if m else s


def scan(text, kernel, ranges):
    """Yield (address, instruction, group, where) for every CALL / LDL / STL of the kernel's text section."""
    lines = text.splitlines()
    start = next(i for i, l in enumerate(lines) if l.startswith("\t.section\t.text." + kernel + ","))
    sub = None                                     # the subroutine being read (None: the kernel body)
    chain = []                                     # (file, line) frames of the current location, innermost first
    fresh = False
    for l in lines[start + 1:]:
        if l.startswith("\t.section\t"):
            break
        if l.startswith("$") and l.rstrip().endswith(":"):
            sub = short_callee(l.rstrip()[:-1])
            continue
        m = FRAME.search(l)
        if m:
            if not fresh:
                chain, fresh = [], True
            chain.append((os.path.basename(m.group(1)), int(m.group(2))))
            continue
        m = INSN.match(l)
        if not m:
            continue
        fresh = False
        insn = m.group(2)
        op = insn.split()[0] if not insn.startswith("@") else insn.split()[1]
        if not (op.startswith("CALL") or op.startswith("LDL") or op.startswith("STL")):
            continue
        inner = f"{chain[0][0]}:{chain[0][1]}" if chain else "?"
        if sub is not None:
            yield m.group(1), insn, GROUPS[3], f"{sub} ({inner})"
            continue
        nm = [ln for f, ln in chain if f == "nuts_machine.cuh"]
        inside = lambda r: any(r[0] <= ln <= r[1] for ln in nm)
        if inside(ranges["leaf"]):
            g = GROUPS[0]
        elif inside(ranges["transition"]) or inside(ranges["run_loop"]):
            g = GROUPS[1]
        else:
            g = GROUPS[2]
        where = inner + (f" ← nuts_machine.cuh:{nm[0]}" if nm and not inner.startswith("nuts_machine.cuh") else "")
        yield m.group(1), insn, g, where


def kind(insn):
    op = insn.split()[1] if insn.startswith("@") else insn.split()[0]
    if op.startswith("CALL"):
        return "CALL"
    return "LDL" if op.startswith("LDL") else "STL"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("build_dir")
    ap.add_argument("--kernel", action="append", help="UNIT:MANGLED_NAME (default: the C2 and C5 kernels)")
    ap.add_argument("--csrc", default=CSRC)
    args = ap.parse_args()
    ranges = source_ranges(args.csrc)
    kernels = args.kernel or DEFAULT_KERNELS
    cache = {}
    with tempfile.TemporaryDirectory() as tmp:
        for spec in kernels:
            unit, name = spec.split(":", 1)
            if unit not in cache:
                cache[unit] = disassemble(os.path.join(args.build_dir, unit + ".o"), tmp)
            rows = list(scan(cache[unit], name, ranges))
            dem = subprocess.run(["c++filt"], input=name, capture_output=True, text=True).stdout.strip() or name
            print(f"## `{dem.replace('(dhmc::KArgs)', '')}` ({unit})\n")
            cnt = collections.Counter((g, kind(i)) for _, i, g, _ in rows)
            print("| group | CALL | LDL | STL |")
            print("|---|---|---|---|")
            for g in GROUPS:
                print(f"| {g} | {cnt[(g, 'CALL')]} | {cnt[(g, 'LDL')]} | {cnt[(g, 'STL')]} |")
            print(f"| total | {sum(v for (g, k), v in cnt.items() if k == 'CALL')} | "
                  f"{sum(v for (g, k), v in cnt.items() if k == 'LDL')} | {sum(v for (g, k), v in cnt.items() if k == 'STL')} |\n")
            for g in GROUPS:
                sel = [r for r in rows if r[2] == g]
                if not sel:
                    continue
                print(f"<details><summary>{g}: {len(sel)} sites</summary>\n")
                print("| address | instruction | source (innermost ← machine line) |")
                print("|---|---|---|")
                for a, i, _, w in sel:
                    i = re.sub(r"`\(\$\S+?\$(\S+?)\)", lambda mm: "`" + short_callee("$" + mm.group(1)) + "`", i)
                    i = re.sub(r"`\((\$__internal_\d+_)?\$__cuda_sm20_(\w+)\)", r"`\2`", i)
                    print(f"| {a} | `{i.replace('`', '').replace('|', '/')}` | {w} |")
                print("\n</details>\n")


if __name__ == "__main__":
    sys.exit(main())
