"""Time the profile-noise what-if (HetSearchResult.profile_noise) on one GPU, against the profile what-if
(recost_profiles) it replaces for this question.

For c3_homo64_mpl6 and c4_het128 (BASELINE configs[2] mpl 6 and configs[3] mpl 4), in one process:
  - result.profile_noise(K, sigma) at K = 16, 256 and 1024 (host clock; the call ends with the statistics on the host,
    so with a device synchronisation);
  - result.recost_profiles of the K = 16 samples' dicts (noisy_profile), the route without profile_noise: the dicts
    built on the host, flattened, uploaded and evaluated, K x N arrays copied back;
  - the host's peak RSS after each K (ru_maxrss, taken before recost_profiles runs: it must not grow with K * N,
    since only O(N + K) bytes come back).
Each time is the best of --reps after one warm-up.  The same run checks the identity at K = 16: every statistic of
profile_noise equals the numpy definitions over the recost_profiles arrays, bit for bit.  Prints one JSON line with the
card's name, power limit and max SM clock beside the times (seconds).
Usage: python tools/profile_noise_bench.py [--reps 3]
"""
import argparse
import json
import os
import resource
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
sys.path.insert(0, os.path.join(REPO, 'tests'))

import numpy as np  # noqa: E402

from breakdown_bench import _card  # noqa: E402
from profile_recost_bench import _inputs  # noqa: E402
from recost_bench import _timed  # noqa: E402

SIGMA = {'layer-computes': 0.05, 'memory': 0.05, 'fb_sync': 0.1}
SEED = 2024


def _rss_mb() -> float:
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0


def _reference(costs, usable, within):
    from test_profile_noise import reference
    return reference(costs, usable, within)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    opt = ap.parse_args()
    import torch
    from metis_b200 import api, search
    out = dict(_card(), sigma=SIGMA)
    for name in ('c3_homo64_mpl6', 'c4_het128'):
        root = tempfile.mkdtemp()
        profile, _seqs, run = _inputs(name, root)
        res = run(profile)
        row = dict(candidates=len(res))
        row['rss_mb_before'] = _rss_mb()
        for k in (16, 256, 1024):
            res.profile_noise(k, SIGMA, SEED)                 # warm-up
            times = []
            for _ in range(opt.reps):
                t, pn = _timed(lambda: res.profile_noise(k, SIGMA, SEED))
                times.append(t)
            row[f'k{k}'] = dict(profile_noise_s=min(times), chunks=pn.timings['chunks'], chunk=pn.timings['chunk'],
                                rss_mb=_rss_mb(), winner=int(np.argmax(pn.wins)), winner_wins=int(pn.wins.max()),
                                searched_best_wins=int(pn.wins[int(np.nanargmin(res.costs))]),
                                usable_everywhere=int((pn.usable == k).sum()))
        dicts = [search.noisy_profile(profile, SIGMA, SEED, j) for j in range(16)]
        rc = res.recost_profiles(dicts)                       # warm-up
        times = []
        for _ in range(opt.reps):
            t, rc = _timed(lambda: res.recost_profiles(dicts))
            times.append(t)
        row['recost_profiles_k16_s'] = min(times)
        want = _reference(rc.costs, rc.usable, 0.01)
        got = res.profile_noise(16, SIGMA, SEED)
        row['identity_k16'] = all(
            (np.asarray(getattr(got, k)).view(np.uint8) == np.asarray(v).view(np.uint8)).all()
            if np.asarray(v).dtype.kind != 'f' else
            (np.where(np.isnan(getattr(got, k)), np.nan, getattr(got, k)).view(np.uint64)
             == np.where(np.isnan(v), np.nan, v).view(np.uint64)).all()
            for k, v in want.items())
        out[name] = row
        api.release_engines()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
