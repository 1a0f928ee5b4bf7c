"""Per-source-line profile of one kernel: joins `ncu -i X.ncu-rep --page source --csv --kernel-name regex:K` (SASS rows in address
order, with executed-instruction and stall-sample counts) with the line table of the same kernel in the cubin
(`nvdisasm -g -c`).  Inlined device functions are attributed to the innermost line.
   python tools/ncu_lines.py <source.csv> <cubin> <mangled-name-substring> [min_pct]"""
import csv, os, re, subprocess, sys, collections
src_csv, cubin, kname = sys.argv[1:4]
minpct = float(sys.argv[4]) if len(sys.argv) > 4 else 0.8
rows = list(csv.reader(open(src_csv)))
hi = [i for i, r in enumerate(rows) if r and r[0] == 'Address'][0]
hdr = rows[hi]; idx = {h: i for i, h in enumerate(hdr)}
data, seen = [], set()
for r in rows[hi + 1:]:
    if len(r) < len(hdr) - 2 or not r[idx['Instructions Executed']].isdigit() or r[0] in seen: continue
    seen.add(r[0]); data.append(r)
dis = subprocess.run(['nvdisasm', '-g', '-c', cubin], capture_output=True, text=True).stdout.splitlines()
start = [i for i, l in enumerate(dis) if l.startswith('.text.') and kname in l][0]
lines, cur = [], None
for l in dis[start + 1:]:
    if l.startswith('//-----') or l.startswith('.text.'): break
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m: cur = (m.group(1).split('/')[-1], int(m.group(2))); continue
    if re.match(r'\s+/\*[0-9a-f]{4,}\*/', l): lines.append(cur)
assert len(lines) == len(data), (len(lines), len(data))
ins, smp = collections.Counter(), collections.Counter()
for ln, r in zip(lines, data):
    ins[ln] += int(r[idx['Instructions Executed']]); smp[ln] += int(r[idx['# Samples']] or 0)
ti, ts = sum(ins.values()), sum(smp.values())
srcs = {}
print(f"warp instructions {ti}, samples {ts}")
for ln in sorted(ins, key=lambda k: (k[0], k[1]) if k else ('', 0)):
    if 100 * ins[ln] / ti < minpct and 100 * smp[ln] / max(ts, 1) < minpct: continue
    f, n = ln if ln else ('?', 0)
    if f not in srcs:
        try: srcs[f] = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'zstd_b200', 'csrc', f)).read().splitlines()
        except Exception: srcs[f] = []
    text = srcs[f][n - 1].strip()[:110] if 0 < n <= len(srcs[f]) else ''
    print(f"{f}:{n:4d} {100*ins[ln]/ti:5.1f}% ins {100*smp[ln]/max(ts,1):5.1f}% smp | {text}")
