"""Summarise an `ncu --csv --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum` launch list per
kernel (template arguments and parameter lists stripped): launches, DRAM MB read/written, total time.

    python profiles/summarise_ncu.py launches.csv [--skip-kernel lm_gemm_kernel<8] > summary.json

`--skip-kernel` drops kernels whose full name contains the given text (e.g. the once-per-generate cross-K/V prefill,
which is not part of a decode step)."""
import argparse
import collections
import csv
import json
import re

ap = argparse.ArgumentParser()
ap.add_argument('csv')
ap.add_argument('--skip-kernel', action='append', default=[])
a = ap.parse_args()

units = {'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9, 'ns': 1e-3, 'us': 1.0, 'ms': 1e3, 'nsecond': 1e-3,
         'usecond': 1.0, 'msecond': 1e3}
agg = collections.OrderedDict()
ids = collections.defaultdict(set)
hdr = None
for row in csv.reader(open(a.csv, errors='replace')):
    if 'Kernel Name' in row and 'Metric Name' in row:
        hdr = row
        continue
    if hdr is None or len(row) != len(hdr):
        continue
    d = dict(zip(hdr, row))
    full = d['Kernel Name']
    if any(s in full for s in a.skip_kernel):
        continue
    name = re.sub(r'^void ', '', full)
    name = re.split(r'[<(]', name)[0]
    e = agg.setdefault(name, dict(launches=0, dram_read_MB=0.0, dram_write_MB=0.0, time_us=0.0))
    ids[name].add(d['ID'])
    try:
        v = float(d['Metric Value'].replace(',', '')) * units.get(d['Metric Unit'], 1.0)
    except ValueError:
        continue
    m = d['Metric Name']
    if m == 'dram__bytes_read.sum':
        e['dram_read_MB'] += v / 1e6
    elif m == 'dram__bytes_write.sum':
        e['dram_write_MB'] += v / 1e6
    elif m == 'gpu__time_duration.sum':
        e['time_us'] += v
for name, e in agg.items():
    e['launches'] = len(ids[name])
    for k in ('dram_read_MB', 'dram_write_MB', 'time_us'):
        e[k] = round(e[k], 2)
print(json.dumps(agg, indent=1))
