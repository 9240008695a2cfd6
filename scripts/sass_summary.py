"""Per-kernel SASS evidence of the in-tree library (runs without a GPU):

    python scripts/sass_summary.py > sass_summary.txt

Counts, for every kernel in libvoxtral_b200.so (sm_90a only), the mnemonics that are proof of a
Hopper-native path: HGMMA (wgmma), UBLKCP (cp.async.bulk), UTMALDG/UTMASTG
(cp.async.bulk.tensor), HMMA (legacy mma.sync), plus registers per thread from the ELF.
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "voxtral_mini_realtime_rs_b200", "libvoxtral_b200.so")
KEYS = ["HGMMA", "UBLKCP", "UTMALDG", "UTMASTG", "HMMA", "IMMA", "SYNCS", "LDGSTS", "REDG", "ATOMG"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    regs = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"REG:(\d+)", line)
        if m and cur:
            regs[cur] = int(m.group(1))
    counts = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m:
            op = m.group(1)
            counts[cur]["_total"] += 1
            for k in KEYS:
                if op.startswith(k):
                    counts[cur][k] += 1
    dm = demangle(list(counts))
    arch = re.findall(r"arch = (sm_\w+)", sass)
    print(f"# {os.path.relpath(LIB, ROOT)}: {len(counts)} kernels, architectures {sorted(set(arch))}")
    print(f"# columns: instructions, registers, then counts of {' '.join(KEYS)} (zeros omitted)")
    for k, c in counts.items():
        name = dm.get(k, k).replace("vox::(anonymous namespace)::", "").replace("(anonymous namespace)::", "").replace("vox::", "")
        name = re.sub(r"^void ", "", name)
        # strip the parameter list (the last top-level parenthesis group), keep template arguments
        depth, cut = 0, len(name)
        for i in range(len(name) - 1, -1, -1):
            if name[i] == ")":
                depth += 1
            elif name[i] == "(":
                depth -= 1
                if depth == 0:
                    cut = i
                    break
        name = name[:cut]
        hits = " ".join(f"{key}={c[key]}" for key in KEYS if c[key])
        print(f"{name:70s} instr={c['_total']:6d} regs={regs.get(k, 0):3d}  {hits}")


if __name__ == "__main__":
    main()
