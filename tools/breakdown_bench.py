"""Time the cost breakdown of searched candidates on one GPU, against the trace replay it replaces.

Until HetSearchResult.breakdown existed, the only way to read a candidate's cost terms and memory headroom was the
verbose path: metis_het_trace replays whole plans and metis_b200.verbose.format_plan decodes their event streams into
the reference's text.  This tool measures both over the same plans:

  - every candidate of c3_homo64_mpl6, with and without the per-stage arrays;
  - the 1 000 best candidates of c4_het128_mpl6;
  - metis_het_trace + format_plan over the plans of the c4 picks, and over the first --trace-plans plans of the c3
    candidates (the trace of every c3 plan would need tens of GB of stream buffers).

Prints one JSON line with the card name and power limit beside the times (seconds, host clock around calls that end
in a device synchronisation; best of --reps after one warm-up).  Usage: python tools/breakdown_bench.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402


def _card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().split('\n')[0]
        name, power, clock = [x.strip() for x in out.split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as exc:                                  # noqa: BLE001 - reported, not fatal
        return dict(gpu=f'unknown ({exc})')


def _best(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return min(times)


def _run(name, root):
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    from metis_b200.workloads import WORKLOADS, materialize, profile_file_order
    w = WORKLOADS[name]
    materialize(w, root)
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), profile_file_order(w)).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                      vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
    args = parse_args(w.cli_args(root))
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    res = api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                               api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), device='cuda:0')
    return res, args, cluster


def _trace(res, args, cluster, idx):
    """metis_het_trace + format_plan over the plans of the candidates ``idx`` (a one-search result)."""
    from metis_b200 import api, search, verbose
    cand = res.candidates
    if cand.space is None:
        return None, 0                                    # a windowed result: no single space to trace
    ordinals = np.unique(cand.records['ordinal'][idx])
    dp = search.DeviceProblem(cand.problem, cand.space, 'cuda:0')

    def run():
        lines = 0
        for lo in range(0, len(ordinals), 2048):
            part = ordinals[lo:lo + 2048]
            trace = verbose.trace_plans(dp, part)
            for k, o in enumerate(part.tolist()):
                ns, label, row, batches, codes = cand.space.locate(o)
                plan = api.InterStagePlan(ns_idx=ns, node_sequence=cand.node_sequences[ns], dg_idx=row,
                                          device_groups=[1 << int(c) for c in codes], num_stage=label,
                                          batches=batches, gbs=args.gbs)
                lines += sum(1 for _ in verbose.format_plan(trace[k], plan, cluster, args.max_profiled_tp_degree,
                                                            args.max_profiled_batch_size))
        return lines
    return run, len(ordinals)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--trace-plans', type=int, default=4096)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'breakdown_bench needs a CUDA device'
    out = dict(_card())
    with tempfile.TemporaryDirectory() as tmp:
        res, args, cluster = _run('c3_homo64_mpl6', os.path.join(tmp, 'c3'))
        n = len(res)
        out['c3_candidates'] = n
        out['c3_breakdown_all_s'] = _best(lambda: res.breakdown(slice(None)), a.reps)
        out['c3_breakdown_all_terms_only_s'] = _best(lambda: res.breakdown(slice(None), per_stage=False), a.reps)
        first = np.nonzero(np.cumsum(np.r_[1, np.diff(res.candidates.records['ordinal'].astype(np.int64)) != 0])
                           <= a.trace_plans)[0]
        run, plans = _trace(res, args, cluster, first)
        out['c3_subset_candidates'] = int(len(first))
        out['c3_subset_plans'] = plans
        out['c3_subset_breakdown_s'] = _best(lambda: res.breakdown(first), a.reps)
        out['c3_subset_trace_decode_s'] = _best(run, 1)

        res, args, cluster = _run('c4_het128_mpl6', os.path.join(tmp, 'c4'))
        res.ranked(1)
        top = res.rank_order[:1000].astype(np.int64)
        out['c4_mpl6_candidates'] = len(res)
        out['c4_top1000_breakdown_s'] = _best(lambda: res.breakdown(top), a.reps)
        run, plans = _trace(res, args, cluster, top)
        out['c4_top1000_plans'] = plans
        out['c4_top1000_trace_decode_s'] = _best(run, 1) if run is not None else 'not measured (windowed result)'
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
