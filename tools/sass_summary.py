"""SASS evidence for the TMA / mbarrier pipelines: per kernel the opcode histogram and every bulk-copy (UBLKCP),
mbarrier (SYNCS.*), shared-memory atomic (ATOMS) and bulk-fence instruction with two lines of context.

    python tools/sass_summary.py quickwit_b200/libqwgpu.so k_union k_aggscan > sass_summary.txt

Needs cuobjdump (CUDA toolkit); runs on the build box, no GPU."""
import collections
import re
import subprocess
import sys


def main():
    lib, wanted = sys.argv[1], sys.argv[2:]
    names = subprocess.run(["cuobjdump", "-elf", lib], capture_output=True, text=True).stdout
    funcs = sorted(set(re.findall(r"\.text\.(_Z\w+)", names)))
    for fn in funcs:
        if not any(w in fn for w in wanted):
            continue
        demangled = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip()
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", fn, lib], capture_output=True, text=True).stdout.splitlines()
        ins = [l for l in sass if re.match(r"\s+/\*[0-9a-f]{4}\*/", l)]
        ops = collections.Counter()
        for l in ins:
            m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", l)
            if m:
                ops[m.group(1).split(".")[0]] += 1
        print("=" * 110)
        print(demangled)
        print(f"{len(ins)} SASS instructions; opcode histogram (top 40):")
        print("  " + ", ".join(f"{k} {v}" for k, v in ops.most_common(40)))
        keys = ("UBLKCP", "SYNCS", "ATOMS", "FENCE", "NANOSLEEP", "REDUX", "UTMA")
        print("counts: " + ", ".join(f"{k} {sum(1 for l in ins if k in l)}" for k in keys))
        print("-- bulk copies, mbarrier operations (first 3 of each distinct form, with context) --")
        seen = collections.Counter()
        for i, l in enumerate(ins):
            m = re.search(r"(UBLKCP[.\w]*|SYNCS[.\w]*|FENCE[.\w]*)", l)
            if not m:
                continue
            seen[m.group(1)] += 1
            if seen[m.group(1)] > 3:
                continue
            for c in ins[max(0, i - 2): i + 3]:
                print("   " + re.sub(r"\s+/\* 0x[0-9a-f]+ \*/\s*$", "", c.rstrip()))
            print("   ...")


if __name__ == "__main__":
    main()
