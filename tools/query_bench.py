"""Time the plan queries (HetSearchResult.ranked(where=), count, best_by) against the same answers computed in Python
from list(result), on one GPU.

For c3_homo64_mpl6 and c4_het128 (BASELINE configs[2] mpl 6 and configs[3] mpl 4), on the one-search result of
api.cost_het_cluster and on a windowed result of the same space (cut into about 3 windows by flatten.plan_windows and
searched by search.search_windows, the pieces of cost_het_cluster's windowed path):
  - count and ranked(100, where=...) under a geometry-only filter (max_stages=8, max_repartition=1) and under a
    strategy filter (max_tp=2, uniform_tp=True);
  - best_by(('num_stage',)) and best_by(('node_sequence', 'max_tp')) under no filter;
  - the same answers from list(result) in Python (PlanFilter.admits, the first admitted per key of the sorted list),
    once; the time of list(result) is given apart.
The one-search result is queried before list(result) runs, so its detail rows are still on the device, as they are for
a caller that has not iterated the result; 'one_search_after_list' repeats the queries afterwards, when the result has
fetched its detail rows to the host (more than 4 096 rows asked for) and a strategy query uploads them again.
Each GPU query ends with its answer on the host (host clock around a device synchronisation); best of --reps after one
warm-up.  The run checks that both give the same answers.  Prints one JSON line with the card's name, power limit and
max SM clock beside the times (seconds).
Usage: python tools/query_bench.py [--reps 3]
"""
import argparse
import itertools
import json
import os
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from breakdown_bench import _card  # noqa: E402


def _inputs(name, root):
    """(one-search result, windowed result maker) of workload ``name``, with bench.py's node sequences."""
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    from metis_b200.workloads import WORKLOADS, materialize, profile_file_order
    w = WORKLOADS[name]
    materialize(w, root)
    profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), profile_file_order(w)).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                      vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
    args = parse_args(w.cli_args(root))
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    seqs = list(itertools.permutations(w.device_types()))
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    llb = api.LayerLoadBalancer(cluster, profile, cfg, args.gbs)

    def one():
        return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                    llb, node_sequences=seqs, device='cuda:0')

    def windowed(parts):
        from metis_b200 import flatten, search
        problem, space, names = api.het_problem(args, cluster, profile, cfg, llb, seqs, device_rows=True, unbounded=True)
        slice_plans = int(space.comp_recs['num_rows'].max()) * len(space.batches)
        windows = flatten.plan_windows(space, -(-space.num_plans // parts) + slice_plans)   # budget in plans
        merged, _dp, searcher = search.search_windows(problem, windows, 'cuda:0')
        summary = dict(merged.summary)
        cand = search.window_candidates(merged, windows, problem, names, searcher)
        return api.HetSearchResult(cand, None, summary, ranker=search.make_window_ranker(searcher, merged.records, summary))
    return one, windowed


def _timed(fn, reps):
    fn()                                                      # warm-up
    best, out = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        t = time.perf_counter() - t0
        best = t if best is None else min(best, t)
    return best, out


def _python(tuples, ranked, place, flt, keys=None):
    """The definitions over list(result): (count, first 100 admitted) or the best per key."""
    from metis_b200 import search
    adm = [i for i in ranked if flt.admits(tuples[i], place[tuples[i][0]])]
    if keys is None:
        return len(adm), [tuples[i] for i in adm[:100]]
    out = {}
    for i in adm:
        out.setdefault(search.query_key(tuples[i], keys), i)
    return sorted(out.items(), key=lambda kv: tuple(search._names(x) if k == 'node_sequence' else x
                                                   for k, x in zip(keys, kv[0])))


FILTERS = {'geometry': dict(max_stages=8, max_repartition=1), 'strategy': dict(max_tp=2, uniform_tp=True)}
KEYS = (('num_stage',), ('node_sequence', 'max_tp'))


def _gpu_queries(res, reps):
    """(times, answers) of the GPU queries on ``res``."""
    from metis_b200.search import PlanFilter
    t, got = {}, {}
    for label, kw in FILTERS.items():
        flt = PlanFilter(**kw)
        t[f'count_{label}_s'], c = _timed(lambda: res.count(flt), reps)
        t[f'ranked100_{label}_s'], top = _timed(lambda: res.ranked(100, where=flt), reps)
        got[label] = (c, top)
    for keys in KEYS:
        t[f'best_by_{"_".join(keys)}_s'], g = _timed(lambda: res.best_by(keys), reps)
        got[keys] = [(v, int(p)) for v, p in zip(g.values, g.position)]
    return t, got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    opt = ap.parse_args()
    import torch
    from metis_b200 import api, search
    from metis_b200.search import PlanFilter
    out = dict(_card())
    for name in ('c3_homo64_mpl6', 'c4_het128'):
        one, windowed = _inputs(name, tempfile.mkdtemp())
        res = one()
        row = dict(candidates=len(res))
        times, answers = {}, {}
        times['one_search'], answers['one_search'] = _gpu_queries(res, opt.reps)    # detail rows on the device
        t0 = time.perf_counter()
        tuples = list(res)
        row['list_result_s'] = time.perf_counter() - t0
        times['one_search_after_list'], answers['one_search_after_list'] = _gpu_queries(res, opt.reps)
        ranked = sorted(range(len(tuples)), key=lambda i: tuples[i][6])
        place = {s: search.rank_device_map(res.candidates.problem, i) for i, s in enumerate(res.candidates.node_sequences)}
        py, want = {}, {}
        for label, kw in FILTERS.items():
            t0 = time.perf_counter()
            want[label] = _python(tuples, ranked, place, PlanFilter(**kw))
            py[f'count_ranked100_{label}_s'] = time.perf_counter() - t0
        for keys in KEYS:
            t0 = time.perf_counter()
            want[keys] = _python(tuples, ranked, place, PlanFilter(), keys)
            py[f'best_by_{"_".join(keys)}_s'] = time.perf_counter() - t0
        row['python'] = py
        del tuples
        api.release_engines()
        win = windowed(3)
        times['windows'], answers['windows'] = _gpu_queries(win, opt.reps)
        row['num_windows'] = win.summary['num_windows']
        for label in times:
            row[label] = dict(times[label], same_answers=answers[label] == want)
        out[name] = row
        del res, win
        api.release_engines()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
