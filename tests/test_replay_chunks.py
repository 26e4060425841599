"""The what-if replays of a finished search (recost, recost_profiles, profile_noise and the queries) walk each
segment's records _RECOST_CHUNK at a time.  The default chunk (2^20 records) holds every golden's candidates and all of
C4-mpl4's, so no other test crosses a chunk boundary inside a segment.  Here a small odd chunk, which splits every
segment several times and leaves a short last chunk, gives what the default chunk gives, bit for bit, as one search and
in forced windows (GPU only)."""
import numpy as np
import pytest

import oracle_profile as op
import test_profile_recost as tpr
from metis_b200 import search
from test_query import KEY_SETS, filters
from test_recost import Spec, _gpu, _run, variant

CHUNK = 97
NAMES = ['mix32', 'rough_t3']
NOISE_FIELDS = ('best_pos', 'best_cost', 'wins', 'near', 'usable', 'regret', 'mean')


def _what_ifs(res, clusters, profiles, flts):
    """Every array the four replays give on ``res``: host copies, keyed by what they are."""
    out = {}
    rc = res.recost(clusters)
    out.update(bw_costs=rc.costs, bw_best=rc.best_costs, bw_regret=rc.regret)
    rc = res.recost_profiles(profiles)
    out.update(pr_costs=rc.costs, pr_headroom=rc.headroom, pr_status=rc.status, pr_best=rc.best_costs,
               pr_regret=rc.regret)
    noise = res.profile_noise(4, 0.15, 11)
    out.update({f'noise_{k}': getattr(noise, k) for k in NOISE_FIELDS})
    for f, flt in enumerate(flts):
        mask, _group = res._mark(flt, None)
        out[f'mask_{f}'] = mask[:len(res)].cpu().numpy()
        out[f'ranked_{f}'] = res.ranked(7, where=flt)
        for keys in KEY_SETS[f % len(KEY_SETS)::5]:
            g = res.best_by(keys, where=flt)
            out[f'best_by_{f}_{keys}'] = (g.values, g.count, g.position, g.cost)
    return out


def _same(got, want):
    assert got.keys() == want.keys()
    for k, w in want.items():
        g = got[k]
        if isinstance(w, np.ndarray) and w.dtype.kind == 'f':
            assert (op.nan_bits(g) == op.nan_bits(w)).all(), k
        elif isinstance(w, np.ndarray):
            assert (g == w).all(), k
        elif k.startswith('best_by'):
            assert g[0] == w[0] and (g[1] == w[1]).all() and (g[2] == w[2]).all(), k
            assert (op.nan_bits(g[3]) == op.nan_bits(w[3])).all(), k
        else:
            assert [t[:6] for t in g] == [t[:6] for t in w], k
            assert (op.nan_bits([t[6] for t in g]) == op.nan_bits([t[6] for t in w])).all(), k


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['one_search', 'windows'])
@pytest.mark.parametrize('name', NAMES)
def test_small_chunks_change_nothing(name, mode, workload_dir, monkeypatch, tmp_path):
    """recost (costs, best, regret), recost_profiles (costs, headroom, status, best, regret), every ProfileNoise array,
    and the queries (the mask, ranked(where=), best_by's groups) with _RECOST_CHUNK = 97 equal the default chunk's."""
    _gpu()
    from metis_b200 import api
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = _run(spec, spec.root, (), mode, monkeypatch)
    if mode == 'windows':
        assert res.summary['num_windows'] > 1
    assert len(res) > 3 * CHUNK
    _base, var, _corrected = variant(spec.root, 'per_type', str(tmp_path))
    clusters = [spec.cluster(spec.root), spec.cluster(var)]
    profiles = op.scenarios(tpr.base_profile(spec), tpr.SEED, spec.seqs)
    flts = filters(list(res), res.candidates.problem.type_names, spec.seqs, seed=3, n=12)
    want = _what_ifs(res, clusters, profiles, flts)
    assert ((want['pr_status'] != 0) | ~(want['pr_headroom'] >= 0)).any()   # the regret's mask has work to do
    monkeypatch.setattr(search, '_RECOST_CHUNK', CHUNK)
    _same(_what_ifs(res, clusters, profiles, flts), want)
    api.release_engines()
