"""Attribute ncu SASS-level counters to CUDA source lines via nvdisasm line info.
usage: python tools/ncu_lines.py rep.ncu-rep cubin mangled_kernel_name [top]"""
import csv, io, re, subprocess, sys
rep, cubin, kname = sys.argv[1:4]
top = int(sys.argv[4]) if len(sys.argv) > 4 else 40
raw = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"] + (["-k", "regex:" + sys.argv[5]] if len(sys.argv) > 5 else []), capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr = rows[1]; c = {h: i for i, h in enumerate(hdr)}
sass = [(r[c["Source"]].strip(), float(r[c["Instructions Executed"]] or 0), float(r[c["# Samples"]] or 0)) for r in rows[2:] if len(r) > 5]
dis = subprocess.run(["nvdisasm", "-g", "-c", cubin], capture_output=True, text=True).stdout.splitlines()
# walk the function's section
start = next(i for i, l in enumerate(dis) if l.strip().startswith(".section") and kname in l)
cur = None; seq = []
for l in dis[start + 1:]:
    if l.strip().startswith(".section") or l.startswith("//-----"):
        if seq: break
        continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m:
        inl = "inlined" in l
        cur = (m.group(1).split("/")[-1], int(m.group(2)))
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
    if m:
        seq.append((cur, m.group(2).strip()))
print(len(sass), len(seq))
n = min(len(sass), len(seq))
agg = {}
for i in range(n):
    k = seq[i][0]
    a = agg.setdefault(k, [0.0, 0.0]); a[0] += sass[i][1]; a[1] += sass[i][2]
ti = sum(v[0] for v in agg.values()); ts = sum(v[1] for v in agg.values())
src = {}
import os
key_ix = 1 if os.environ.get("BY_SAMPLES") else 0
for k, v in sorted(agg.items(), key=lambda kv: -kv[1][key_ix])[:top]:
    f, ln = k if k else ("?", 0)
    if f not in src:
        try: src[f] = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vello_b200", "csrc", f)).read().splitlines()
        except Exception: src[f] = []
    text = src[f][ln - 1].strip()[:90] if 0 < ln <= len(src[f]) else ""
    print(f"{100*v[0]/ti:5.1f}% inst {100*v[1]/max(ts,1):5.1f}% smp  {f}:{ln:<5d} {text}")
