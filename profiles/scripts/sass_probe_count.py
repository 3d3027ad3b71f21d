"""Instruction counts of the PCG-II link kernel's pass-1 tile loops, by opcode, from `cuobjdump -sass`.

usage: python sass_probe_count.py OLD.{so,o} [NEW.{so,o}] [--kernel MANGLED_NAME]

A pass-1 tile loop is a loop of the kernel (a backward branch and its target) that holds exactly one mbarrier wait
(`SYNCS.PHASECHK`, the ring's full barrier) and the `DMUL`s of the scoring: the TE / 32 = 4 unrolled warp-steps of a
tile, the ring wait, the chunk close and the arrive on the empty barrier.  The wait's retry path lies outside the loop
and is not counted.  The branch-free loop (records without a missing non-constant value) has no global load; the
missing-value loop gathers 1/n(y) with `LDG`.  Default kernel: k_link_pcg2<10, 6, 32, PK, ID16, SC>, the benchmark's.
"""
import argparse
import collections
import re
import subprocess

KERNEL = "_Z11k_link_pcg2ILi10ELi6ELi32ELb1ELb1ELb1EEv10LinkParams"
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);")


def instructions(path, kernel):
    out = subprocess.run(["cuobjdump", "-sass", "-fun", kernel, path], capture_output=True, text=True, check=True).stdout
    ins = []
    for m in INSN.finditer(out):
        ins.append((int(m.group(1), 16), m.group(3), m.group(4)))
    if not ins:
        raise SystemExit(f"{path}: no SASS for {kernel}")
    return ins


def tile_loops(ins):
    """(kind, instructions) of every pass-1 tile loop, in address order"""
    loops = []
    for i, (addr, op, args) in enumerate(ins):
        if not op.startswith("BRA") or op.startswith("BRA.DIV"):
            continue
        m = re.search(r"(0x[0-9a-f]+)\s*$", args.strip())
        if not m or int(m.group(1), 16) >= addr:
            continue
        body = [x for x in ins if int(m.group(1), 16) <= x[0] <= addr]
        ops = [x[1] for x in body]
        if sum(o.startswith("SYNCS.PHASECHK") for o in ops) != 1 or not any(o.startswith("DMUL") for o in ops):
            continue
        loops.append(body)
    # the loop with the fewest DMULs is the branch-free one; the missing-value loop adds the 1/n(y) multiplies
    dmul = [sum(x[1].startswith("DMUL") for x in body) for body in loops]
    return [("branch-free" if d == min(dmul) else "missing-value", body) for d, body in zip(dmul, loops)]


def histogram(body):
    return collections.Counter(op.split(".")[0] for _, op, _ in body if op != "NOP")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("binaries", nargs="+")
    ap.add_argument("--kernel", default=KERNEL)
    a = ap.parse_args()
    counts = {}
    for path in a.binaries:
        for kind, body in tile_loops(instructions(path, a.kernel)):
            counts.setdefault(kind, []).append((path, histogram(body)))
    for i, path in enumerate(a.binaries):
        print(f"[{i}] {path}")
    for kind, rows in counts.items():
        ops = sorted(set().union(*(h for _, h in rows)), key=lambda o: -max(h[o] for _, h in rows))
        print(f"{kind} pass-1 tile loop (4 warp-steps)")
        print(f"  {'opcode':<10}" + "".join(f"{f'[{a.binaries.index(p)}]':>8}" for p, _ in rows))
        print(f"  {'total':<10}" + "".join(f"{sum(h.values()):>8}" for _, h in rows))
        for o in ops:
            print(f"  {o:<10}" + "".join(f"{h[o]:>8}" for _, h in rows))


if __name__ == "__main__":
    main()
