"""Time the search what-if under profile noise (HetSearchResult.search_noise) on one GPU, against K fresh
cost_het_cluster calls on the same samples' dicts, the route without it.

For c3_homo64_mpl6 and c4_het128 (BASELINE configs[2] mpl 6 and configs[3] mpl 4), in one process:
  - result.search_noise(K, sigma) at K = 16 and 256 (host clock; the call ends with the results on the host, so with a
    device synchronisation);
  - K fresh searches: noisy_profile dicts built, HeteroCostEstimator / LayerLoadBalancer built from each, flattened and
    searched by api.cost_het_cluster, best() taken (dict building and flattening counted);
  - the identity on the same samples: each sample's status (the one cost_het_cluster raises with), candidate count,
    winner and best cost (bits) equal the fresh search's;
  - in which samples profile_noise (every partition held fixed) has the searched best as its best, against `same`.
search_noise is the best of --reps after one warm-up; the fresh searches run once per K (their first call is the
warm-up of the cached engine, which the searched result already made).  Prints one JSON line with the card's name,
power limit and max SM clock beside the times (seconds).
Usage: python tools/search_noise_bench.py [--reps 2]
"""
import argparse
import json
import os
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

import numpy as np  # noqa: E402

from breakdown_bench import _card  # noqa: E402
from profile_recost_bench import _inputs  # noqa: E402
from recost_bench import _timed  # noqa: E402

SIGMA = {'layer-computes': 0.05, 'memory': 0.05, 'fb_sync': 0.1}
SEED = 2024
# the statuses with which cost_het_cluster raises each exception (search.raise_fatal)
EXC_STATUS = {'KeyError': (1, 2), 'IndexError': (3,), 'RuntimeError': (4, 5), 'ZeroDivisionError': (6,)}


def _fresh(profile, run, K):
    """K fresh searches under the samples' dicts: (seconds, [(status, count, best) per sample])."""
    from metis_b200 import search
    t0 = time.perf_counter()
    out = []
    for j in range(K):
        prof = search.noisy_profile(profile, SIGMA, SEED, j)
        try:
            r = run(prof)
            out.append((0, len(r), r.best()))
        except (KeyError, IndexError, RuntimeError, ZeroDivisionError) as exc:
            out.append((type(exc).__name__, 0, None))
    return time.perf_counter() - t0, out


def _same(got, fresh) -> bool:
    for j, (status, count, best) in enumerate(fresh):
        if status != 0:
            if got.status[j] not in EXC_STATUS[status]:
                return False
            continue
        if got.status[j] != 0 or got.num_candidates[j] != count or got.winner(j) != best:
            return False
        if best is not None and np.float64(got.best_cost[j]).view(np.uint64) != np.float64(best[6]).view(np.uint64):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=2)
    opt = ap.parse_args()
    import torch
    from metis_b200 import api
    out = dict(_card(), sigma=SIGMA)
    for name in ('c3_homo64_mpl6', 'c4_het128'):
        root = tempfile.mkdtemp()
        profile, _seqs, run = _inputs(name, root)
        res = run(profile)
        row = dict(candidates=len(res), search_gpu_s=res.timings['gpu_search_s'])
        for k in (16, 256):
            res.search_noise(k, SIGMA, SEED)                  # warm-up
            times = []
            for _ in range(opt.reps):
                t, got = _timed(lambda: res.search_noise(k, SIGMA, SEED))
                times.append(t)
            fresh_s, fresh = _fresh(profile, run, k)
            fixed = res.profile_noise(k, SIGMA, SEED)         # the same samples with every partition held fixed
            fixed_same = fixed.best_pos == res._best_position()
            row[f'k{k}'] = dict(search_noise_s=min(times), per_sample_ms=1e3 * min(times) / k,
                                chunks=got.timings['chunks'], fresh_s=fresh_s, identity=_same(got, fresh),
                                same=int(got.same.sum()), same_plan=int(got.same_plan.sum()),
                                statuses=sorted(set(int(s) for s in got.status)),
                                loss_max=float(np.nanmax(np.where(np.isinf(got.loss), np.nan, got.loss)))
                                if np.isfinite(got.loss).any() else None,
                                kept_unusable=int((~got.kept_usable).sum()), near=int(got.near.sum()),
                                distinct_winners=len(got.winners()), fixed_partition_same=int(fixed_same.sum()),
                                same_samples_as_fixed=bool((fixed_same == got.same).all()))
        out[name] = row
        api.release_engines()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
