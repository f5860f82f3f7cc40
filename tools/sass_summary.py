"""SASS evidence of a kernel: resource usage, opcode histogram and the instructions that prove the Hopper-native paths
(UBLKCP = cp.async.bulk / TMA, SYNCS = mbarrier, ATOMS / REDUX / VOTE / MATCH = warp-level protocol).
usage: python tools/sass_summary.py <object or .so> <mangled kernel name>"""
import re
import subprocess
import sys

obj, kname = sys.argv[1], sys.argv[2]
res = subprocess.run(["cuobjdump", "-res-usage", obj], capture_output=True, text=True).stdout
sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout.splitlines()
start = next(i for i, l in enumerate(sass) if "Function : " + kname in l)
end = next((i for i in range(start + 1, len(sass)) if "Function : " in sass[i]), len(sass))
body = [l for l in sass[start:end] if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l)]
ins = [re.sub(r"^\s+/\*[0-9a-f]+\*/\s+", "", l).split(";")[0].strip() for l in body]
print(f"# SASS summary of {kname} in {obj} (cuobjdump -sass, sm_90a)")
for i, l in enumerate(res.splitlines()):
    if kname in l:
        print("# " + l.strip())
        print("# " + res.splitlines()[i + 1].strip())
print(f"# {len(ins)} instructions")
hist = {}
for x in ins:
    t = x.split()
    op = t[1] if t[0].startswith("@") and len(t) > 1 else t[0]
    hist[op] = hist.get(op, 0) + 1
print("\n## opcode histogram (top 40)")
for op, n in sorted(hist.items(), key=lambda kv: -kv[1])[:40]:
    print(f"{n:7d}  {op}")
print("\n## TMA / mbarrier / warp-protocol instructions")
pat = re.compile(r"UBLKCP|UTMA|SYNCS|ATOMS|REDUX|VOTE|MATCH|LDGSTS|FENCE|MEMBAR|ERRBAR|CCTL")
for l in body:
    if pat.search(l):
        print(re.sub(r"\s+", " ", l.split(";")[0]).strip())
