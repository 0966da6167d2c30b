"""Registers and spills of every kernel instantiation, from the `ptxas -v` logs of two builds (csrc/Makefile writes one
`build/*.ptxas.log` per translation unit; a user-model build keeps its own under csrc/user_models/<name>/build/).

    python benchmarks/ptxas_diff.py OLD_LOG_DIR NEW_LOG_DIR [...more OLD NEW pairs] > table.md

Prints a markdown table with one row per entry function: registers, spill stores / loads (bytes) before and after.
Spill figures are those of the kernel's own "Function properties" block (noinline device functions have their own)."""
import glob
import os
import re
import subprocess
import sys


def parse(log_dir):
    out = {}
    for f in sorted(glob.glob(os.path.join(log_dir, "*.ptxas.log"))):
        unit = os.path.basename(f)[: -len(".ptxas.log")]
        entry, props = None, None
        for line in open(f):
            m = re.search(r"Compiling entry function '(\w+)'", line)
            if m:
                entry = m.group(1)
                out[(unit, entry)] = {}
                continue
            m = re.search(r"Function properties for (\w+)", line)
            if m:
                props = m.group(1)
                continue
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and props is not None and (unit, props) in out:
                out[(unit, props)].update(st=int(m.group(2)), ld=int(m.group(3)))
                continue
            m = re.search(r"Used (\d+) registers", line)
            if m and entry is not None:
                out[(unit, entry)]["reg"] = int(m.group(1))
    return out


def demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return r.stdout.splitlines() if r.returncode == 0 else names


def main():
    pairs = sys.argv[1:]
    if not pairs or len(pairs) % 2:
        sys.exit(__doc__)
    rows = []
    for old_dir, new_dir in zip(pairs[::2], pairs[1::2]):
        a, b = parse(old_dir), parse(new_dir)
        for key in sorted(set(a) | set(b)):
            rows.append((key, a.get(key), b.get(key)))
    names = demangle([k[1] for k, _, _ in rows])
    fmt = lambda d: "—" if d is None else f"{d.get('reg', '?')} | {d.get('st', 0)} / {d.get('ld', 0)}"
    changed = sum(1 for _, x, y in rows if x != y)
    print(f"{len(rows)} entry functions, {changed} changed.\n")
    print("| unit | kernel | before: registers \\| spill st / ld (B) | after: registers \\| spill st / ld (B) | changed |")
    print("|---|---|---|---|---|")
    for ((unit, _), x, y), name in zip(rows, names):
        print(f"| {unit} | `{name.replace('(dhmc::KArgs)', '')}` | {fmt(x).replace('|', chr(92) + '|')} | "
              f"{fmt(y).replace('|', chr(92) + '|')} | {'**yes**' if x != y else ''} |")


if __name__ == "__main__":
    main()
