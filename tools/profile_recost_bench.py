"""Time the profile what-if (HetSearchResult.recost_profiles) against fresh searches, on one GPU.

For c3_homo64_mpl6 and c4_het128 (BASELINE configs[2] mpl 6 and configs[3] mpl 4), K = 1, 4 and 16 scenario profiles
made from the searched profile by the tests' seeded transform (tests/oracle_profile.py: per-layer compute, memory,
model-section and noise scenarios).  In one process, alternating:
  - result.recost_profiles(K profiles) (host clock; the call ends with costs, headroom, status and regret on the host,
    so with a device synchronisation);
  - K fresh api.cost_het_cluster calls, one per profile (host clock; each ends in a device synchronisation).  Only
    profiles under which a fresh search completes are used: under some of them the reference aborts the search (a
    balancer loop that never ends); how many were skipped is reported.
The same run checks the identity: under the searched profile, costs and headroom equal the search's bit for bit.  A
fresh search answers another question (it re-runs the strategy chain and the balancer); it is timed here as the
alternative a user has without the what-if.  Prints one JSON line with the card's name, power limit and max SM clock
beside the times (seconds; best of --reps after one warm-up).
Usage: python tools/profile_recost_bench.py [--reps 3]
"""
import argparse
import json
import os
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
sys.path.insert(0, os.path.join(REPO, 'tests'))

import numpy as np  # noqa: E402

from breakdown_bench import _card  # noqa: E402
from recost_bench import _timed  # noqa: E402

KINDS = ('compute', 'memory', 'model', 'noise')          # scenarios every fresh search completes


def _inputs(name, root):
    import itertools
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
    seqs = list(itertools.permutations(w.device_types()))
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))

    def run(prof, headroom=False):
        volume = api.GPTActivationAndParam(cfg, prof['model']['parameters'])
        return api.cost_het_cluster(args, cluster, prof, cfg, api.HeteroCostEstimator(prof, cfg, volume, cluster),
                                    api.LayerLoadBalancer(cluster, prof, cfg, args.gbs), node_sequences=seqs,
                                    device='cuda:0', headroom=headroom)
    return profile, [[str(t) for t in s] for s in seqs], run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    opt = ap.parse_args()
    import torch
    import oracle_profile as op
    from metis_b200 import api
    out = dict(_card())
    for name in ('c3_homo64_mpl6', 'c4_het128'):
        root = tempfile.mkdtemp()
        profile, seqs, run = _inputs(name, root)
        res = run(profile, headroom=True)
        ident = res.recost_profiles([profile])
        row = dict(candidates=len(res),
                   identity=bool((ident.status == 0).all()
                                 and (ident.costs[0].view(np.uint64) == res.costs.view(np.uint64)).all()
                                 and (ident.headroom[0].view(np.uint64) == res.headroom.view(np.uint64)).all()))
        for k in (1, 4, 16):
            profiles, seed = [], 1000
            while len(profiles) < k:                          # warm-up of the fresh searches, and only profiles under
                p = op.scenario(profile, KINDS[seed % len(KINDS)], seed, seqs)   # which a search completes: the
                seed += 1                                     # reference aborts some (a balancer loop that never ends)
                try:
                    run(p)
                except RuntimeError:
                    row['aborting_profiles_skipped'] = row.get('aborting_profiles_skipped', 0) + 1
                    continue
                profiles.append(p)
            res.recost_profiles(profiles)                     # warm-up
            rec_t, fresh_t = [], []
            for _ in range(opt.reps):                         # alternating
                t, rc = _timed(lambda: res.recost_profiles(profiles))
                rec_t.append(t)
                t, fresh = _timed(lambda: [len(run(p)) for p in profiles])
                fresh_t.append(t)
            row[f'k{k}'] = dict(recost_profiles_s=min(rec_t), fresh_searches_s=min(fresh_t),
                                ratio=min(fresh_t) / min(rec_t), recost_part_s=rc.timings['recost_s'],
                                regret_s=rc.timings['regret_s'], usable=[int(u.sum()) for u in rc.usable])
        out[name] = row
        api.release_engines()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
