"""Per-kernel SASS audit of lib/libacr_b200.so: which kernels carry warpgroup MMA (HGMMA), TMA (UTMALDG / UTMASTG),
mbarrier (SYNCS), warp-level MMA (HMMA), system-scope stores, or local-memory (spill) traffic (LDL / STL).  Needs no GPU:
cuobjdump -sass.
    python tools/sass_audit.py [lib.so]  ->  markdown table on stdout"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LIB = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
MNEMONICS = ["HGMMA", "UTMALDG", "UTMASTG", "SYNCS", "HMMA", "STG.E.128.STRONG.SYS", "LDGSTS", "LDL", "STL", "USETMAXREG"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.split("\n")
    return dict(zip(names, out))


def audit(lib=LIB):
    sass = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    per, cur = collections.OrderedDict(), None
    for line in sass.split("\n"):
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = per.setdefault(m.group(1), collections.Counter())
            continue
        if cur is None:
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m:
            cur["_n"] += 1
            for k in MNEMONICS:
                if m.group(1).startswith(k):
                    cur[k] += 1
    names = demangle(list(per))
    rows = collections.OrderedDict()
    for f, c in per.items():
        n = names[f]
        n = re.sub(r"\(anonymous namespace\)::|acr::", "", n).split("(")[0]
        n = re.sub(r"^void ", "", n)
        r = rows.setdefault(n, collections.Counter())
        r.update(c)
    return rows


if __name__ == "__main__":
    rows = audit()
    cols = [k for k in MNEMONICS if any(r[k] for r in rows.values())]
    print("| kernel | SASS instructions | " + " | ".join(f"`{c}`" for c in cols) + " |")
    print("|---|---:|" + "---:|" * len(cols))
    for n, r in sorted(rows.items(), key=lambda kv: (-kv[1]["HGMMA"], kv[0])):
        print(f"| `{n}` | {r['_n']} | " + " | ".join(str(r[c]) if r[c] else "" for c in cols) + " |")
