#!/usr/bin/env python
"""Warp-instruction share per SOURCE line of a kernel in an .ncu-rep captured with --import-source on (-lineinfo build):
    python profiles/ncu_hot_lines.py out/r02_cov.ncu-rep k_covariance [top]"""
import csv
import subprocess
import sys

rep, kern = sys.argv[1], sys.argv[2]
top = int(sys.argv[3]) if len(sys.argv) > 3 else 30
out = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--csv', '--print-source', 'cuda,sass', '--kernel-name', 'regex:' + kern],
                     capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
fpath, hdr, data = None, None, []
def f(x):
    try:
        return float(x.replace(',', ''))
    except Exception:
        return 0.0
for r in rows:
    if len(r) >= 2 and r[0] == 'File Path':
        fpath = r[1].split('/')[-1]
    elif r and r[0] == 'Line No':
        hdr = r
    elif hdr and len(r) == len(hdr) and r[0].isdigit():
        ia, it, ist = hdr.index('Instructions Executed'), hdr.index('Thread Instructions Executed'), hdr.index('Warp Stall Sampling (All Samples)')
        if f(r[ia]) > 0:
            data.append((fpath, int(r[0]), r[1].strip(), f(r[ia]), f(r[it]), f(r[ist])))
tot = sum(d[3] for d in data)
stot = sum(d[5] for d in data)
print('total warp instructions %.4g, stall samples %.4g' % (tot, stot))
for d in sorted(data, key=lambda d: -d[3])[:top]:
    print('%5.1f%% instr %5.1f%% stall  lanes %4.1f  %s:%d  %s' % (100 * d[3] / tot, 100 * d[5] / max(stot, 1), d[4] / d[3], d[0], d[1], d[2][:90]))
