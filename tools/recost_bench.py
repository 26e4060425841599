"""Time the network what-if (HetSearchResult.recost) against fresh searches, on one GPU.

For c3_homo64_mpl6 and c4_het128 (BASELINE configs[2] mpl 6 and configs[3] mpl 4), K = 1, 4 and 16 scenarios: the
searched cluster with every IP's intra_bandwidth scaled by a seeded factor.  In one process, alternating:
  - result.recost(K clusters) (host clock; the call ends with the costs and regret on the host, so with a device
    synchronisation);
  - K fresh api.cost_het_cluster calls, one per scenario (host clock; each ends in a device synchronisation).
The same run checks that both give the same candidates and the same cost bits.  Prints one JSON line with the card's
name, power limit and max SM clock beside the times (seconds; best of --reps after one warm-up).
Usage: python tools/recost_bench.py [--reps 3]
"""
import argparse
import itertools
import json
import os
import random
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

import numpy as np  # noqa: E402

from breakdown_bench import _card  # noqa: E402


def _inputs(name, root):
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
    # bench.py's node sequences: the order of set(device types) (quirk Q4) would change the space from process to process
    seqs = list(itertools.permutations(w.device_types()))

    def cluster(clusterfile='clusterfile.json'):
        return GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, clusterfile))

    def run(gpu_cluster):
        return api.cost_het_cluster(args, gpu_cluster, profile, cfg,
                                    api.HeteroCostEstimator(profile, cfg, volume, gpu_cluster),
                                    api.LayerLoadBalancer(gpu_cluster, profile, cfg, args.gbs), node_sequences=seqs,
                                    device='cuda:0')
    return cluster, run


def _scenarios(root, k, rng):
    """k clusterfiles beside the searched one, each IP's intra_bandwidth scaled by a seeded factor."""
    base = json.load(open(os.path.join(root, 'clusterfile.json')))
    names = []
    for j in range(k):
        info = {ip: dict(v, intra_bandwidth=v['intra_bandwidth'] * rng.choice([0.125, 0.25, 0.5, 2.0, 4.0]))
                for ip, v in base.items()}
        names.append(f'scenario{j}.json')
        with open(os.path.join(root, names[-1]), 'w') as fh:
            json.dump(info, fh)
    return names


def _timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    opt = ap.parse_args()
    import torch
    from metis_b200 import api
    out = dict(_card())
    rng = random.Random(7)
    for name in ('c3_homo64_mpl6', 'c4_het128'):
        root = tempfile.mkdtemp()
        cluster, run = _inputs(name, root)
        res = run(cluster())
        search_s = min(_timed(lambda: run(cluster()))[0] for _ in range(opt.reps))
        res = run(cluster())                                  # the result re-costed below
        row = dict(candidates=len(res), search_s=search_s)
        for k in (1, 4, 16):
            clusters = [cluster(f) for f in _scenarios(root, k, rng)]
            res.recost(clusters)                              # warm-up
            rec_t, fresh_t = [], []
            for _ in range(opt.reps):                         # alternating
                t, rc = _timed(lambda: res.recost(clusters))
                rec_t.append(t)
                t, fresh = _timed(lambda: [run(c) for c in clusters])
                fresh_t.append(t)
            rc = res.recost(clusters)                         # after the fresh searches: the result keeps its tables
            same = True
            for j, f in enumerate(fresh):
                r = f.candidates.records
                same &= bool(len(f) == len(res)
                             and (r['ordinal'] == res.candidates.records['ordinal']).all()
                             and (r['step'] == res.candidates.records['step']).all()
                             and (f.costs.view(np.uint64) == rc.costs[j].view(np.uint64)).all()
                             and f.best()[:6] == rc.best(j)[:6])
            row[f'k{k}'] = dict(recost_s=min(rec_t), fresh_searches_s=min(fresh_t),
                                speedup=min(fresh_t) / min(rec_t), recost_part_s=rc.timings['recost_s'],
                                regret_s=rc.timings['regret_s'], same_results=same)
            del fresh
        out[name] = row
        api.release_engines()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
