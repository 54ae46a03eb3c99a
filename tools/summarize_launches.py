"""ncu launch list (CSV of `--metrics gpu__time_duration.sum`) -> per-kernel table (markdown).

    python tools/summarize_launches.py gpurun_out/launches.csv [skip_first_n_launches_per_kernel]
"""
import csv
import re
import sys
from collections import OrderedDict

path = sys.argv[1]
skip = int(sys.argv[2]) if len(sys.argv) > 2 else 10
rows = []
with open(path) as f:
    lines = [l for l in f if l.startswith('"')]
for r in csv.DictReader(lines):
    if r.get('Metric Name') == 'gpu__time_duration.sum':
        name = re.sub(r'\(.*', '', r['Kernel Name'])
        rows.append((name, float(r['Metric Value']) / 1e3, r['Grid Size'], r['Block Size']))
per = OrderedDict()
for name, us, grid, block in rows:
    per.setdefault(name, []).append((us, grid, block))
tot = 0.0
out = []
for name, v in per.items():
    vals = [x[0] for x in v[skip:]] or [x[0] for x in v]
    mean = sum(vals) / len(vals)
    out.append((name, len(v), mean, v[-1][1], v[-1][2]))
    tot += mean
print('| kernel | launches | grid | block | mean us | share |')
print('|---|---|---|---|---|---|')
for name, n, mean, grid, block in sorted(out, key=lambda x: -x[2]):
    print(f'| {name} | {n} | {grid} | {block} | {mean:.2f} | {mean / tot:.3f} |')
print(f'\nSum of per-kernel means = {tot:.1f} us')
