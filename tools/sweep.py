#!/usr/bin/env python3
"""BASELINE.json configs[4]: search-space sweep 8-512 GPUs x 1-4 device types.

For every point: host enumeration time, GPU search time (CUDA events), counters A/B/C, the best plan,
plans/s - and a parity spot check: `--check K` sampled inter-stage plans are re-evaluated with the
CPU oracle (oracle/metis_oracle.py) and compared bit-for-bit with the GPU records of those plans.

  python tools/sweep.py [--check 200] [--out sweep_out/sweep.jsonl] [--points n8t1,n64t2,...]
"""
import argparse
import itertools
import json
import os
import random
import re
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from metis_b200 import flatten, native, search  # noqa: E402
from metis_b200.data_loader import ProfileDataLoader  # noqa: E402
from metis_b200.gpu_cluster import GPUCluster  # noqa: E402
from metis_b200.utils import ModelConfig  # noqa: E402
from metis_b200.workloads import materialize, profile_file_order, sweep_workload  # noqa: E402

DEFAULT_POINTS = [(8, 1, 1, 4), (16, 2, 1, 4), (32, 2, 1, 4), (32, 4, 1, 4), (64, 1, 1, 4), (64, 1, 1, 6), (64, 2, 1, 4),
                  (64, 1, 0, 4), (128, 1, 1, 4), (128, 3, 1, 4), (128, 1, 1, 6), (256, 1, 1, 4), (256, 2, 1, 4),
                  (512, 1, 1, 4), (512, 4, 1, 6),
                  # variance 0 (the variance-1 filter collapses the space at >= 256 GPUs, SURVEY.md 8d)
                  (128, 1, 0, 4), (128, 2, 0, 4), (256, 1, 0, 4)]


def run_point(ndev, ntypes, variance, mpl, check):
    w = sweep_workload(ndev, ntypes, variance, mpl)
    # profiles up to bs 16 so that mixed-type stages do not abort the search (quirk Q8)
    w.bss = (1, 2, 4, 8, 16)
    tmp = tempfile.mkdtemp()
    materialize(w, tmp)
    order = profile_file_order(w)
    cluster = GPUCluster(tmp + '/hostfile', tmp + '/clusterfile.json')
    profile, _ = ProfileDataLoader(tmp + '/profile', order).load_profile_data_all()
    cfg = ModelConfig('SYN', w.num_layers, w.sequence_length, w.vocab_size, w.hidden_size, 32)
    seqs = list(itertools.permutations(w.device_types()))
    t0 = time.perf_counter()
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
    # the host lists the compositions; the GPU writes the rows (SURVEY.md 8(f)-1)
    space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance,
                                     w.max_permute_len, device_rows=True)
    enum_ms = 1e3 * (time.perf_counter() - t0)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    dp = search.DeviceProblem(problem, space, 'cuda:0')
    torch.cuda.synchronize()
    upload_ms = 1e3 * (time.perf_counter() - t1)              # arena allocation + H2D + row kernel (first call)
    searcher = search.HetSearcher(dp, want_records=True, want_detail=False)
    out = searcher.run()
    best_only = search.HetSearcher(dp, want_records=False)
    for _ in range(2):
        best_only.launch()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); best_only.launch(); b.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(b)
    row = {'ndev': ndev, 'types': ntypes, 'variance': variance, 'mpl': mpl, 'layers': w.num_layers, 'gbs': w.gbs,
           'A_plans': space.num_plans, 'row_bytes': int(space.rows_total_bytes), 'upload_rows_ms': upload_ms, 'B_partition_calls': out.summary['num_partition_calls'],
           'runs': out.summary['num_balancer_runs'], 'C_costed': out.summary['num_records'],
           'keyerror': out.summary['num_keyerror'],
           'fatal_ordinal': None if out.summary['fatal_ordinal'] == 2 ** 64 - 1 else out.summary['fatal_ordinal'],
           'host_enumeration_ms': enum_ms, 'gpu_search_ms': ms, 'plans_per_s': space.num_plans / (ms * 1e-3),
           'best': out.best[:3] if out.best else None}
    if check > 0 and space.num_plans:
        from oracle import metis_oracle as orc
        ocl = orc.OracleCluster(tmp + '/hostfile', tmp + '/clusterfile.json')
        oprof, _ = orc.load_profile_dir(tmp + '/profile', order)
        omodel = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size, oprof['model']['parameters'])
        norm = orc.norm_layer_duration(oprof)
        rng = random.Random(ndev * 131 + ntypes)
        limit = out.summary['fatal_ordinal'] if out.summary['fatal_ordinal'] != 2 ** 64 - 1 else space.num_plans
        picks = sorted(rng.sample(range(limit), min(check, limit))) if limit else []
        sub = out.records[np.isin(out.records['ordinal'].astype(np.int64), np.asarray(picks, dtype=np.int64))]
        got = search.materialize(sub, searcher.detail_for(sub), space, seqs) if len(sub) else []
        by_ord = {}
        for rec, tup in zip(sub, got):
            by_ord.setdefault(int(rec['ordinal']), []).append(tup)
        bad = 0
        for o in picks:
            ns, label, rowi, batches, codes = space.locate(o)
            plan = {'ns_idx': ns, 'node_sequence': seqs[ns], 'dg_idx': rowi, 'device_groups': [1 << int(c) for c in codes],
                    'num_stage': label, 'batches': batches, 'gbs': w.gbs}
            want, counters = [], {'A': 0, 'B': 0, 'C': 0, 'runs': 0, 'keyerr': 0}
            orc.het_evaluate_plan(oprof, ocl, omodel, norm, plan, o, w.num_layers, w.max_tp, w.max_bs, counters, want)
            mine = by_ord.get(o, [])
            same = len(mine) == len(want) and all(
                (m[1], m[2], m[3], m[4], m[5]) == (x[3], x[4], x[5], x[6], x[7]) and m[6] == x[8] for m, x in zip(mine, want))
            bad += 0 if same else 1
        row['oracle_checked_plans'] = len(picks)
        row['oracle_mismatches'] = bad
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', type=int, default=100)
    ap.add_argument('--out', default='sweep_out/sweep.jsonl')
    ap.add_argument('--points', default='')
    ns = ap.parse_args()
    points = DEFAULT_POINTS
    if ns.points:
        points = []
        for tok in ns.points.split(','):                      # n128t1 or n128t1v0m4
            m = re.fullmatch(r'n(\d+)t(\d+)(?:v(\d+))?(?:m(\d+))?', tok)
            points.append((int(m.group(1)), int(m.group(2)), int(m.group(3) or 1), int(m.group(4) or 4)))
    os.makedirs(os.path.dirname(ns.out) or '.', exist_ok=True)
    with open(ns.out, 'w') as fh:
        for p in points:
            try:
                row = run_point(*p, ns.check)
            except Exception as exc:   # noqa: BLE001 - the sweep reports what each point did
                row = {'ndev': p[0], 'types': p[1], 'variance': p[2], 'mpl': p[3], 'error': f'{type(exc).__name__}: {exc}'}
            print(json.dumps(row))
            fh.write(json.dumps(row) + '\n')
            fh.flush()


if __name__ == '__main__':
    main()
