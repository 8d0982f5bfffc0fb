"""Per-kernel SASS mnemonic histogram of the built library.

    python tools/sass_histogram.py

Runs `cuobjdump -sass` on yolov3_b200/libyolov3_b200.so (no GPU needed) and counts, for every kernel, the instructions that
prove which hardware path it takes: HGMMA (wgmma), WARPGROUP (wgmma fences / waits), UTMALDG / UTMASTG (TMA load / store),
SYNCS (mbarrier), ACQBULK / PREEXIT (griddepcontrol.wait / launch_dependents: programmatic
dependent launch), HMMA / IMMA (legacy mma.sync: only the 3-channel stem conv and the fallback wgrad), MUFU, REDUX, ATOM/ATOMS/RED,
LDGSTS (cp.async: the shared-memory ring of the BatchNorm backward passes).
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "yolov3_b200" / "libyolov3_b200.so"
KEYS = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "SYNCS", "ACQBULK", "PREEXIT", "HMMA", "IMMA", "MUFU", "REDUX", "ATOM", "ATOMS", "RED", "LDG", "STG", "LDGSTS"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    sass = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True).stdout
    per = collections.OrderedDict()
    cur = None
    total = collections.Counter()
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per[cur] = collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if not (m and cur):
            continue
        op = m.group(1)
        per[cur]["_insts"] += 1
        base = op.split(".")[0]
        if base in KEYS:
            per[cur][base] += 1
    names = demangle(list(per))
    print(f"# cuobjdump -sass {LIB.relative_to(ROOT)}  ({len(per)} kernels; sm_90a)")
    print("# columns: " + " ".join(KEYS) + " | total instructions | kernel")
    for k, c in per.items():
        total.update(c)
        short = names.get(k, k).replace("(anonymous namespace)::", "").replace("void ", "")
        short = re.sub(r"\((?!anonymous).*$", "", short)
        print(" ".join(f"{c[x]:5d}" for x in KEYS) + f" | {c['_insts']:6d} | {short}")
    print("# total")
    print(" ".join(f"{total[x]:5d}" for x in KEYS) + f" | {total['_insts']:6d} | all kernels")
    legacy = [re.sub(r"\(.*$", "", names.get(k, k).replace("(anonymous namespace)::", "")) for k, c in per.items() if c["HMMA"] or c["IMMA"]]
    print("# kernels with legacy mma.sync (HMMA): " + (", ".join(sorted(set(x.split("::")[-1].split("<")[0] for x in legacy))) or "none"))


if __name__ == "__main__":
    main()
