#!/usr/bin/env python3
"""Developer tool: attribute `Instructions Executed` / stall samples of an ncu report to CUDA source
lines (ncu's CSV source page is SASS-only; nvdisasm -g supplies the SASS offset -> file:line map).

  python tools/ncu_by_line.py <report>.ncu-rep [kernel-substring] [top-N] [--sectors]

--sectors ranks the lines by L2 sectors instead ("L2 Theoretical Sectors Local" + "... Global", 32 B each): which
source lines generate the memory traffic (local = per-thread scratch of the throughput mode, global = task lists,
rows, records).
"""
import collections
import csv
import os
import re
import subprocess
import sys
import tempfile

sectors = '--sectors' in sys.argv
if sectors:
    sys.argv.remove('--sectors')
rep = sys.argv[1]
kern = sys.argv[2] if len(sys.argv) > 2 else 'het_search_kernelILi64'
top = int(sys.argv[3]) if len(sys.argv) > 3 else 45
repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.environ.get('NCU_BY_LINE_LIB') or os.path.join(repo, 'metis_b200', 'libmetis_b200.so')
tmp = tempfile.mkdtemp()
subprocess.run(['cuobjdump', '-xelf', 'all', lib], cwd=tmp, capture_output=True)
cubin = [f for f in os.listdir(tmp) if f.startswith('metis_search.') and f.endswith('.cubin')][0]
dis = subprocess.run(['nvdisasm', '-g', '-c', os.path.join(tmp, cubin)], capture_output=True, text=True).stdout
line_of = {}
cur = None
inside = False
for ln in dis.splitlines():
    if ln.startswith('//---') and '.text.' in ln:
        inside = kern in ln
        continue
    if not inside:
        continue
    m = re.match(r'\s*//## File "(.*)", line (\d+)', ln)
    if m:
        cur = (os.path.basename(m.group(1)), int(m.group(2)))
        continue
    m = re.match(r'\s*/\*([0-9a-f]{4,})\*/', ln)
    if m:
        line_of[int(m.group(1), 16)] = cur
csvtxt = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--csv', '--print-source', 'sass'],
                        capture_output=True, text=True).stdout
allrows = list(csv.reader(csvtxt.splitlines()))
# the report may hold several kernels: sections start with a "Kernel Name" row followed by the column header
want = kern.replace('ILi', '<(int)').split('<')[0] if False else kern
sections, cur_rows = [], None
for r in allrows:
    if r and r[0] == 'Kernel Name':
        cur_rows = [r]
        sections.append(cur_rows)
    elif cur_rows is not None:
        cur_rows.append(r)
def _matches(name):
    plain = re.sub(r'[^A-Za-z0-9_]', '', name)
    return re.sub(r'[^A-Za-z0-9_]', '', kern.split('ILi')[0]) in plain and \
        (('ILi' not in kern) or re.sub(r'\D', '', kern.split('ILi', 1)[1])[:2] in re.sub(r'\D', '', name)[:4])
rows = next((sec for sec in sections if _matches(sec[0][1])), sections[0] if sections else allrows)
hdr = rows[1]
ia, iex, ith, ism = hdr.index('Address'), hdr.index('Instructions Executed'), hdr.index('Thread Instructions Executed'), hdr.index('# Samples')
base = int(rows[2][ia], 16)
agg = collections.defaultdict(lambda: [0, 0, 0])
tot = [0, 0, 0]
for r in rows[2:]:
    off = int(r[ia], 16) - base
    key = line_of.get(off, ('?', 0))
    for k, idx in enumerate((iex, ith, ism)):
        agg[key][k] += int(r[idx]); tot[k] += int(r[idx])
src = {}
def text(key):
    f, n = key
    path = os.path.join(repo, 'metis_b200', 'csrc', f)
    if f not in src and os.path.exists(path):
        src[f] = open(path).read().splitlines()
    return src[f][n - 1].strip()[:90] if f in src and 0 < n <= len(src[f]) else ''
if sectors:
    il, ig = hdr.index('L2 Theoretical Sectors Local'), hdr.index('L2 Theoretical Sectors Global')
    iop = hdr.index('Access Operation')
    mem = collections.defaultdict(lambda: [0, 0, set()])
    mt = [0, 0]
    for r in rows[2:]:
        key = line_of.get(int(r[ia], 16) - base, ('?', 0))
        loc, glo = int(r[il] or 0), int(r[ig] or 0)
        if loc or glo:
            mem[key][0] += loc; mem[key][1] += glo; mem[key][2].add(r[iop])
            mt[0] += loc; mt[1] += glo
    print(f'L2 theoretical sectors: local {mt[0]/1e6:.1f} M ({mt[0]*32/1e9:.2f} GB), global {mt[1]/1e6:.1f} M ({mt[1]*32/1e9:.2f} GB)')
    for key, (loc, glo, ops) in sorted(mem.items(), key=lambda kv: -(kv[1][0] + kv[1][1]))[:top]:
        print(f'{100*(loc+glo)/max(mt[0]+mt[1],1):5.1f}%  local {loc*32/1e6:8.1f} MB  global {glo*32/1e6:8.1f} MB  {"/".join(sorted(o for o in ops if o and o != "-")):12s} {key[0]}:{key[1]:<5d} {text(key)}')
    sys.exit(0)
print(f'total warp-inst {tot[0]/1e9:.3f}e9, thread/inst {tot[1]/max(tot[0],1):.2f}, samples {tot[2]}')
for key, (ex, th, sm) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:top]:
    print(f'{100*ex/tot[0]:5.1f}% inst {100*sm/max(tot[2],1):5.1f}% smp  {key[0]}:{key[1]:<5d} {text(key)}')

# ---- the same, summed per enclosing function (crude: the nearest preceding function header in the source file) ----
if '--functions' in os.environ.get('NCU_BY_LINE', ''):
    heads = {}
    for f, lines in src.items():
        hs = []
        for i, l in enumerate(lines, 1):
            m = re.match(r'\s*(?:template.*)?\s*(?:MB_HD(?:_NOINLINE)?|static __device__ \w+|__device__(?: __\w+__)?|__global__)\s+.*?(\w+)\(', l)
            if m and not l.strip().startswith('//'):
                hs.append((i, m.group(1)))
        heads[f] = hs
    fagg = collections.defaultdict(lambda: [0, 0])
    for (f, n), (ex, th, sm) in agg.items():
        name = '?'
        for i, nm in heads.get(f, []):
            if i <= n:
                name = nm
        fagg[(f, name)][0] += ex; fagg[(f, name)][1] += sm
    print('--- by function ---')
    for key, (ex, sm) in sorted(fagg.items(), key=lambda kv: -kv[1][0])[:30]:
        print(f'{100*ex/tot[0]:5.1f}% inst {100*sm/max(tot[2],1):5.1f}% smp  {key[0]}:{key[1]}')
