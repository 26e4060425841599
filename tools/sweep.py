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
                  (128, 1, 0, 4), (128, 2, 0, 4), (256, 1, 0, 4),
                  # beyond one search (2^32 plans / 4 GiB of rows / the device's memory): searched in windows
                  (256, 1, 0, 6), (512, 1, 0, 4), (256, 4, 0, 4)]


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
    space = flatten.build_device_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers,
                                            w.variance, w.max_permute_len)
    if space is None:                                         # compositions beyond the row kernel: host rows
        space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance,
                                         w.max_permute_len, device_rows=True)
    enum_ms = 1e3 * (time.perf_counter() - t0)
    per_plan, per_row, per_rec, fixed = search.window_cost_model(problem)
    budget = search.window_budget('cuda:0', fixed)
    if not flatten.fits_one_search(space) or flatten.window_bytes(space, per_plan, per_row, per_rec) > budget:
        return run_windows(w, tmp, order, seqs, problem, space, flatten.plan_windows(space, budget, per_plan, per_row,
                                                                                       per_rec), enum_ms, check)
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
        rng = random.Random(ndev * 131 + ntypes)
        limit = out.summary['fatal_ordinal'] if out.summary['fatal_ordinal'] != 2 ** 64 - 1 else space.num_plans
        picks = sorted(rng.sample(range(limit), min(check, limit))) if limit else []
        sub = out.records[np.isin(out.records['ordinal'].astype(np.int64), np.asarray(picks, dtype=np.int64))]
        got = search.materialize(sub, searcher.detail_for(sub), space, seqs) if len(sub) else []
        by_ord = {}
        for rec, tup in zip(sub, got):
            by_ord.setdefault(int(rec['ordinal']), []).append(tup)
        row['oracle_checked_plans'] = len(picks)
        row['oracle_mismatches'] = oracle_mismatches(w, tmp, order, seqs, picks, space.locate,
                                                     lambda o: by_ord.get(o, []))
    return row


def run_windows(w, tmp, order, seqs, problem, space, windows, enum_ms, check):
    """A point beyond one search: the windows of flatten.plan_windows searched in ordinal order (search.search_windows).
    The time is the wall time of search.search_windows (every window's upload, row generation and search, and the host
    merges), host enumeration excluded.  The parity check takes each picked plan from the windows (PlanWindow.plan_at)
    and its device groups from the host enumerator's table of its stage count."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()                                  # the peak below is this point's alone
    torch.cuda.reset_peak_memory_stats()
    t1 = time.perf_counter()
    merged, dp, searcher = search.search_windows(problem, windows, 'cuda:0')
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t1)
    s = merged.summary
    row = {'ndev': w_ndev(w), 'types': len(w.device_types()), 'variance': w.variance, 'mpl': w.max_permute_len,
           'layers': w.num_layers, 'gbs': w.gbs, 'A_plans': space.num_plans, 'row_bytes': int(space.rows_total_bytes),
           'windows': len(windows), 'windows_searched': s['windows_searched'],
           'B_partition_calls': s['num_partition_calls'], 'runs': s['num_balancer_runs'], 'C_costed': s['num_records'],
           'keyerror': s['num_keyerror'], 'fatal_ordinal': None if s['fatal_ordinal'] == 2 ** 64 - 1 else s['fatal_ordinal'],
           'host_enumeration_ms': enum_ms, 'gpu_search_ms': ms, 'plans_per_s': space.num_plans / (ms * 1e-3),
           'peak_device_bytes': int(torch.cuda.max_memory_reserved()), 'best': merged.best[:3] if merged.best else None}
    if check > 0 and space.num_plans:
        cand = search.window_candidates(merged, windows, problem, seqs, searcher)
        rng = random.Random(w_ndev(w) * 131 + len(w.device_types()))
        limit = row['fatal_ordinal'] if row['fatal_ordinal'] is not None else space.num_plans
        picks = sorted(rng.sample(range(limit), min(check, limit))) if limit else []
        picks = sorted(set(picks) | {o for x in windows for o in (x.base, x.base + x.space.num_plans - 1) if o < limit})
        rec = merged.records
        glob = merged.bases[np.searchsorted(merged.firsts, np.arange(len(rec)), side='right') - 1] + \
            rec['ordinal'].astype(np.int64)
        bases = np.asarray([x.base for x in windows], dtype=np.int64)
        table = {}

        def plan_of(o):
            # the device groups from the host enumerator's table of the stage count, not from the windows' rows
            ns, label, dg, batches, S, _at = windows[int(np.searchsorted(bases, o, side='right')) - 1].plan_at(o)
            if S not in table:
                table.clear()
                table[S] = flatten.enumerate_device_groups(S, w_ndev(w), w.variance, w.max_permute_len)
            return ns, label, dg, batches, table[S][dg]

        def mine_of(o):
            idx = np.nonzero(glob == o)[0]
            return cand.tuples(idx) if len(idx) else []
        row['oracle_checked_plans'] = len(picks)
        row['oracle_mismatches'] = oracle_mismatches(w, tmp, order, seqs, picks, plan_of, mine_of)
    return row


def oracle_mismatches(w, tmp, order, seqs, picks, plan_of, mine_of) -> int:
    """Plans of ``picks`` whose candidates (``mine_of(ordinal)``: the GPU's 7-tuples) differ from the pinned oracle's;
    ``plan_of(ordinal)`` -> (ns_idx, label, dg_idx, batches, log2 device groups)."""
    from oracle import metis_oracle as orc
    ocl = orc.OracleCluster(tmp + '/hostfile', tmp + '/clusterfile.json')
    oprof, _ = orc.load_profile_dir(tmp + '/profile', order)
    omodel = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size, oprof['model']['parameters'])
    norm = orc.norm_layer_duration(oprof)
    bad = 0
    for o in picks:
        ns, label, rowi, batches, codes = plan_of(o)
        plan = {'ns_idx': ns, 'node_sequence': seqs[ns], 'dg_idx': rowi, 'device_groups': [1 << int(c) for c in codes],
                'num_stage': label, 'batches': batches, 'gbs': w.gbs}
        want, counters = [], {'A': 0, 'B': 0, 'C': 0, 'runs': 0, 'keyerr': 0}
        orc.het_evaluate_plan(oprof, ocl, omodel, norm, plan, o, w.num_layers, w.max_tp, w.max_bs, counters, want)
        mine = mine_of(o)
        same = len(mine) == len(want) and all(
            (m[1], m[2], m[3], m[4], m[5]) == (x[3], x[4], x[5], x[6], x[7]) and m[6] == x[8] for m, x in zip(mine, want))
        bad += 0 if same else 1
    return bad


def w_ndev(w):
    return sum(n for _, n in w.nodes)


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
