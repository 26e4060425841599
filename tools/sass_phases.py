#!/usr/bin/env python3
"""Developer tool: static count of the local-memory instructions (LDL / STL) and generic loads (LD) of a search
kernel, by phase of the bulk round.

  python tools/sass_phases.py [kernel-substring] [--lib PATH | --cubin PATH]

The library is built with -lineinfo, so `nvdisasm -gi` gives every SASS instruction its source line and the chain of
inlined calls that led there.  An instruction belongs to the innermost frame that lies in one of the evaluator's
drivers in metis_eval.cuh (PlanEvaluator::begin / compute_performance / memory_phase / adjust_performance / get_cost,
balance_run cut at its x.mark() hooks); the out-of-line helpers count for the phase that calls them.  Printed per
phase: instructions, LDL, STL and LD.  Together with the phase clock (tools/phase_profile.py --bulk) this says which
phase's scratch traffic is worth cutting; it counts code, not executions.  In the instantiations that read the tables
from shared memory (template flag SMEM) a generic LD is never a table read on a common path: a table or descriptor
read that shows up here lost its shared-memory hint (metis_eval.cuh, assume_shared_tables).
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EVAL = 'metis_eval.cuh'
MARKS = {10: 'R forward', 11: 'R backward', 12: 'R leftovers', 13: 'R vote', 14: 'R capacities', 15: 'R adjust',
         16: 'R part'}
DRIVERS = {'begin': 'P begin', 'compute_performance': 'P performance', 'balance_run': 'R init',
           'memory_phase': 'M memory', 'adjust_performance': 'M reweight', 'get_cost': 'C cost',
           'first_task': 'first_task'}
HELPERS = {'hetero_performance': 'P performance', 'hetero_memory_demand': 'M memory',
           'memory_demand_own_type': 'M memory', 'hetero_exec_cost': 'C cost'}
ORDER = ['P begin', 'P performance', 'R init', 'R forward', 'R backward', 'R leftovers', 'R vote', 'R capacities',
         'R adjust', 'R part', 'M memory', 'M reweight', 'C cost', 'first_task', 'other']


def regions(path):
    """[(first line, last line, phase)] of the drivers in metis_eval.cuh, balance_run split at its marks."""
    lines = open(path).read().splitlines()
    heads = []
    for i, l in enumerate(lines, 1):
        m = re.match(r'\s*(?:MB_HD|MB_HD_NOINLINE)\s+[\w:<>,\s\*&]*?\b(\w+)\(', l)
        if m and not l.lstrip().startswith('//'):
            heads.append((i, m.group(1)))
    out = []
    for k, (i, name) in enumerate(heads):
        end = heads[k + 1][0] - 1 if k + 1 < len(heads) else len(lines)
        phase = DRIVERS.get(name) or HELPERS.get(name)
        if not phase:
            continue
        if name != 'balance_run':
            out.append((i, end, phase))
            continue
        cuts = [(i, 'R init')]
        for j in range(i, end + 1):
            m = re.search(r'x\.mark\((\d+)\)', lines[j - 1])
            if m and int(m.group(1)) in MARKS:
                cuts.append((j, MARKS[int(m.group(1))]))
        for c, (a, ph) in enumerate(cuts):
            out.append((a, cuts[c + 1][0] - 1 if c + 1 < len(cuts) else end, ph))
    return out


def phase_of(chain, regs):
    for f, n in chain:                                        # innermost first
        if f != EVAL:
            continue
        for a, b, ph in regs:
            if a <= n <= b:
                return ph
    return 'other'


def cubin_of(ns, tmp):
    if ns.cubin:
        return ns.cubin
    lib = ns.lib or os.path.join(REPO, 'metis_b200', 'libmetis_b200.so')
    subprocess.run(['cuobjdump', '-xelf', 'all', os.path.abspath(lib)], cwd=tmp, capture_output=True, check=True)
    return os.path.join(tmp, [f for f in os.listdir(tmp) if f.startswith('metis_search.') and f.endswith('.cubin')][0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('kernel', nargs='?', default='het_first_kernel')
    ap.add_argument('--lib', default=None, help='library to read (default: metis_b200/libmetis_b200.so)')
    ap.add_argument('--cubin', default=None, help='read this cubin instead of a library')
    ap.add_argument('--src', default=os.path.join(REPO, 'metis_b200', 'csrc'),
                    help='directory of the metis_eval.cuh the binary was compiled from')
    ns = ap.parse_args()
    regs = regions(os.path.join(ns.src, EVAL))
    with tempfile.TemporaryDirectory() as tmp:
        dis = subprocess.run(['nvdisasm', '-gi', '-c', cubin_of(ns, tmp)], capture_output=True, text=True,
                             check=True).stdout
    per = {}
    name, chain, fresh = None, [], True
    for ln in dis.splitlines():
        if ln.startswith('//---') and '.text.' in ln:
            name = ln.split('.text.', 1)[1].split()[0]
            name = name if ns.kernel in name else None
            if name:
                per[name] = collections.defaultdict(lambda: [0, 0, 0, 0])
            continue
        if name is None:
            continue
        m = re.match(r'\s*//## File "(.*?)", line (\d+)', ln)
        if m:
            if fresh:
                chain, fresh = [], False
            chain.append((os.path.basename(m.group(1)), int(m.group(2))))
            continue
        m = re.match(r'\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)', ln)
        if m:
            fresh = True
            op = m.group(1).split('.')[0]
            row = per[name][phase_of(chain, regs)]
            row[0] += 1
            row[1] += op == 'LDL'
            row[2] += op == 'STL'
            row[3] += op == 'LD'
    if not per:
        raise SystemExit(f'no kernel matches {ns.kernel!r}')
    for name, rows in per.items():
        tot = [sum(r[k] for r in rows.values()) for k in range(4)]
        print(f'{name}: {tot[0]} instructions, {tot[1]} LDL, {tot[2]} STL, {tot[3]} LD')
        print(f'  {"phase":<14s} {"instr":>6s} {"LDL":>5s} {"STL":>5s} {"LD":>5s}')
        for ph in ORDER:
            if ph in rows:
                r = rows[ph]
                print(f'  {ph:<14s} {r[0]:6d} {r[1]:5d} {r[2]:5d} {r[3]:5d}')


if __name__ == '__main__':
    sys.exit(main())
