"""Search what-if (metis_het_search_noise_*, HetSearchResult.search_noise / search_profiles): a fresh search under each
seeded sample of the searched profile, or under given profiles, next to the searched winner held fixed.

CPU: the host build of the whole draw (tests/hostsim/search_noise_sim.cpp), norm_lc included, against
flatten.build_problem(noisy_profile(...)) with the sample's own layer weights, bit for bit; the host search on host-drawn
samples against the oracle's het_search on the samples' dicts; the ScenarioSearch fields against plain-Python
definitions; the ValueError and NotImplementedError cases and the argument checks.  GPU (-m gpu): search_noise and
search_profiles against K fresh api.cost_het_cluster calls under the same dicts, field for field, costs bit for bit;
zero noise; a tiny chunk budget; a what-if taken after list(result) and after a later search.
"""
import copy
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
import oracle_profile as op
import test_profile_noise as tpn
import test_profile_recost as tpr
from metis_b200 import api, flatten, native, search
from metis_b200.utils import DeviceType
from conftest import load_golden
from oracle import metis_oracle as orc
from test_recost import Spec, _gpu, _run

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'search_noise_sim.cpp')
SIM_DEPS = tpn.SIM_DEPS + [SIM_SRC]
DRAW = ['mix32', 'rough_t3', 'rough_q10']
EXC_STATUS = {KeyError: (1, 2), IndexError: (3,), RuntimeError: (4, 5), ZeroDivisionError: (6,)}
_sim = []


def sim():
    """The g++ build of tests/hostsim/search_noise_sim.cpp, hostsim.cpp's flags."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'libsearch_noise_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)                             # atomic: concurrent test processes may race
        _sim.append(C.CDLL(out))
    return _sim[0]


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def norm_args(profile, sigma):
    """(row, DeviceType code, layer-computes sigma) of the profile's first-listed entry, as search_noise passes them."""
    name, row = api.norm_source(profile)
    tname = name[len('DeviceType.'):]
    sig = search.noise_sigmas(sigma)
    return row, search.device_type_code(tname), search._sigma_of(sig, 'layer-computes', tname)


def own_problems(spec, profiles, corrected=()):
    """Each profile flattened as a fresh search flattens it: the searched cluster, flags and corrections, its own
    norm_lc."""
    cluster = spec.cluster(spec.root)
    cfg = hs.load_inputs(spec.root, spec.sub, spec.meta['file_order'], spec.num_layers, spec.hidden_size,
                         spec.sequence_length, spec.vocab_size)[3]
    return [flatten.build_problem(p, cluster, cfg, spec.gbs, spec.max_tp, spec.max_bs, spec.seqs, corrected=corrected)
            for p in profiles]


def host_draw(problem, spec, s, row, code, sigma):
    keep = dict(problem.arrays)
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    K, L = problem.scalars['num_keys'], problem.scalars['lpad']
    out = dict(layer_compute=np.zeros((K, L)), layer_memory=np.zeros((K, L)), exec_full=np.zeros(K),
               fb_sync=np.zeros(K), norm_lc=np.zeros(problem.scalars['norm_len']))
    row = np.ascontiguousarray(row, dtype=np.float64)
    zero = C.c_int32(-1)
    ptr = lambda a: C.c_void_p(a.ctypes.data)               # noqa: E731
    assert sim().search_noise_sim_draw(C.byref(p), C.byref(spec), ptr(row), C.c_int32(code), C.c_double(sigma),
                                       C.c_int32(s), *[ptr(out[k]) for k in ('layer_compute', 'layer_memory',
                                                                             'exec_full', 'fb_sync', 'norm_lc')],
                                       C.byref(zero)) == 0
    return out, zero.value


def check_draw(spec, base, sigma, seed, firsts=(0, 5)):
    """The host draw of samples first, first + 1 equals build_problem of their dicts, every array bit for bit."""
    problem = own_problems(spec, [base])[0]
    row, code, s = norm_args(base, sigma)
    for first in firsts:
        dicts = [search.noisy_profile(base, sigma, seed, j) for j in (first, first + 1)]
        flat = own_problems(spec, dicts)
        ns = tpn.noise_spec(problem, sigma, seed, first, 2)
        for k in range(2):
            got, zero = host_draw(problem, ns, k, row, code, s)
            assert zero == 0
            for name, v in flat[k].arrays.items():
                want = got.get(name, problem.arrays[name])
                assert np.array_equal(np.asarray(v).view(np.uint8), np.asarray(want).view(np.uint8)), (name, k)
            assert flat[k].scalars == problem.scalars
    return problem, got


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', sorted(tpn.SIGMAS))
@pytest.mark.parametrize('name', DRAW)
def test_host_draw_is_build_problem(name, kind, workload_dir):
    """The draw kernels' code gives sample j's layer_compute, layer_memory, exec_full, fb_sync and norm_lc exactly as
    flatten.build_problem of noisy_profile(profile, sigma, seed, j) with the sample's own layer weights does."""
    spec = Spec(name, workload_dir)
    base = tpr.base_profile(spec)
    problem, got = check_draw(spec, base, tpn.SIGMAS[kind], 0x1234_5678_9abc_def0)
    if norm_args(base, tpn.SIGMAS[kind])[2]:
        assert (got['norm_lc'] != problem.arrays['norm_lc']).any()


def test_host_draw_first_entry_not_in_cluster(workload_dir):
    """A profile whose first-listed entry is a device type the cluster does not have: its tp1_bs1 row, under that
    type's sigma and code, gives the layer weights."""
    spec = Spec('mix32', workload_dir)
    base = tpr.base_profile(spec)
    problem = own_problems(spec, [base])[0]
    other = next(t for t in DeviceType.__members__ if t not in problem.type_names)
    entry = copy.deepcopy(base[f'DeviceType.{problem.type_names[0]}'])
    for e in entry.values():
        e['time']['layer-computes'] = [v * 1.5 + 0.25 for v in e['time']['layer-computes']]
    odd = {f'DeviceType.{other}': entry, **base}
    assert next(iter(odd)) == f'DeviceType.{other}'
    sigma = {'layer-computes': {other: 0.4, problem.type_names[0]: 0.1}, 'memory': 0.2}
    own, got = check_draw(spec, odd, sigma, 99)
    assert (own.arrays['norm_lc'] != problem.arrays['norm_lc']).any()
    assert (got['norm_lc'] != own.arrays['norm_lc']).any()


def test_host_draw_zero_sigma_on_the_norm_type(workload_dir):
    """Zero layer-computes sigma on the first-listed type with every other field noisy: norm_lc is the profile's."""
    spec = Spec('rough_t3', workload_dir)
    base = tpr.base_profile(spec)
    first = next(iter(base))[len('DeviceType.'):]
    sigma = {'layer-computes': {t: (0.0 if t == first else 0.3) for t in DeviceType.__members__}, 'memory': 0.2,
             'fb_sync': 0.1}
    problem, got = check_draw(spec, base, sigma, 5)
    assert np.array_equal(_bits(got['norm_lc']), _bits(problem.arrays['norm_lc']))
    assert not np.array_equal(_bits(got['layer_memory']), _bits(problem.arrays['layer_memory']))


def test_host_draw_zero_total_is_flagged(workload_dir):
    """A row whose noisy total is 0 (possible on rough profiles with negative times) is flagged, and the sample keeps
    the base's norm_lc; flatten.norm_layer_duration raises ZeroDivisionError on the same dict."""
    spec = Spec('mix32', workload_dir)
    base = tpr.base_profile(spec)
    problem = own_problems(spec, [base])[0]
    ns = tpn.noise_spec(problem, 0.0, 3, 0, 1)
    got, zero = host_draw(problem, ns, 0, np.zeros(problem.scalars['norm_len']), 1, 0.2)
    assert zero == 1 and np.array_equal(_bits(got['norm_lc']), _bits(problem.arrays['norm_lc']))
    flat = copy.deepcopy(base)
    flat[next(iter(flat))]['tp1_bs1']['time']['layer-computes'] = [0.0] * problem.scalars['norm_len']
    with pytest.raises(ZeroDivisionError):
        flatten.norm_layer_duration(search.noisy_profile(flat, 0.2, 3, 0))


def _status_of(exc) -> tuple:
    return EXC_STATUS[type(exc)]


@pytest.mark.parametrize('name', ['mix32', 'rough_q10'])
def test_host_search_of_drawn_samples_is_the_oracle(name, workload_dir):
    """The host build of the search on host-drawn samples equals the oracle's het_search on the samples' dicts:
    status, count, and best tuple and cost bits."""
    spec = Spec(name, workload_dir)
    base = tpr.base_profile(spec)
    problem, space = spec.problem(spec.root)
    sigma, seed = 0.2, 20260
    row, code, s = norm_args(base, sigma)
    ns = tpn.noise_spec(problem, sigma, seed, 0, 3)
    cl = orc.OracleCluster(os.path.join(spec.root, 'hostfile'), os.path.join(spec.root, 'clusterfile.json'))
    for k in range(3):
        got, zero = host_draw(problem, ns, k, row, code, s)
        assert zero == 0
        sample = flatten.FlatProblem(problem.scalars, dict(problem.arrays, **got), problem.type_names,
                                     problem.key_names, problem.node_sequences)
        rec, det, summary = hs.host_het_search(sample, space, mode=0)
        prof = search.noisy_profile(base, sigma, seed, k)
        model = orc.OracleModel(spec.num_layers, spec.hidden_size, spec.sequence_length, spec.vocab_size,
                                prof['model']['parameters'])
        try:
            cands, _ = orc.het_search(prof, cl, model, spec.seqs, spec.gbs, spec.num_layers, spec.variance,
                                      spec.max_permute_len, spec.max_tp, spec.max_bs)
        except (KeyError, IndexError, RuntimeError, ZeroDivisionError) as exc:
            assert summary.fatal_ordinal != 2 ** 64 - 1 and summary.fatal_code in _status_of(exc)
            continue
        assert summary.fatal_ordinal == 2 ** 64 - 1 or summary.fatal_code == 0
        assert len(rec) == len(cands)
        mine = hs.unpack_candidates(rec, det, space)
        want = sorted(cands, key=lambda c: c[8])[0]
        top = sorted(mine, key=lambda c: c[8])[0]
        assert (top[0], top[1], top[4], top[6], top[7]) == (want[0], want[1], want[4], want[6], want[7])
        assert _bits(top[8]) == _bits(want[8])


GOLDENS = ['mix32', 'rough_q10']
FIELDS = ('status', 'num_candidates', 'best_cost', 'kept_cost', 'kept_usable', 'loss', 'near', 'same', 'same_plan')


def golden_samples(spec, name):
    """The search_noise_<name> golden, its samples' dicts rebuilt from the seed (checked against the sha256s) and each
    sample's expected (status codes, count, best tuple or None)."""
    meta, gold = load_golden(f'search_noise_{name}')
    assert meta['inputs_sha256'] == spec.meta['inputs_sha256']
    dicts = [search.noisy_profile(tpr.base_profile(spec), meta['sigma'], meta['seed'], j) for j in range(meta['samples'])]
    assert [op.sha256(p) for p in dicts] == meta['sample_sha256']
    want = []
    for j, st in enumerate(meta['status']):
        codes = (0,) if st == '' else (4,) if st == 'hang' else EXC_STATUS[{'KeyError': KeyError, 'IndexError': IndexError,
                                                                            'ZeroDivisionError': ZeroDivisionError,
                                                                            'RuntimeError': RuntimeError}[st]]
        best = None
        if st == '' and gold['best_ordinal'][j] >= 0:
            S = int(gold['best_nstage'][j])
            best = (int(gold['best_ordinal'][j]), int(gold['best_step'][j]), int(gold['best_ns_idx'][j]),
                    gold['best_groups'][j, :S].tolist(),
                    list(zip(gold['best_dp'][j, :S].tolist(), gold['best_tp'][j, :S].tolist())),
                    int(gold['best_batches'][j]), gold['best_part'][j, :S + 1].tolist(), int(gold['best_nrep'][j]),
                    float(gold['best_cost'][j]))
        want.append((codes, int(gold['count'][j]), best))
    return meta, gold, dicts, want


def _same_best(got, want):
    assert got[:8] == want[:8]
    assert _bits(got[8]) == _bits(want[8])


@pytest.mark.parametrize('name', GOLDENS)
def test_search_noise_goldens_oracle_and_host_build(name, workload_dir):
    """The search_noise goldens of the unmodified reference (8 samples, at least one won by another plan): the oracle's
    het_search on the samples' dicts and the host build of the search on host-drawn samples equal them, status, count,
    and best tuple and cost bits."""
    spec = Spec(name, workload_dir)
    meta, gold, dicts, want = golden_samples(spec, name)
    assert meta['other_winner'] and meta['searched'] == [int(spec.arr['ordinal'][np.argsort(spec.arr['cost'],
                                                                                           kind='stable')[0]]),
                                                         int(spec.arr['step'][np.argsort(spec.arr['cost'],
                                                                                        kind='stable')[0]])]
    base = tpr.base_profile(spec)
    problem, space = spec.problem(spec.root)
    row, code, s = norm_args(base, meta['sigma'])
    ns = tpn.noise_spec(problem, meta['sigma'], meta['seed'], 0, meta['samples'])
    cl = orc.OracleCluster(os.path.join(spec.root, 'hostfile'), os.path.join(spec.root, 'clusterfile.json'))
    for j, prof in enumerate(dicts):
        codes, count, best = want[j]
        model = orc.OracleModel(spec.num_layers, spec.hidden_size, spec.sequence_length, spec.vocab_size,
                                prof['model']['parameters'])
        try:
            cands, _ = orc.het_search(prof, cl, model, spec.seqs, spec.gbs, spec.num_layers, spec.variance,
                                      spec.max_permute_len, spec.max_tp, spec.max_bs)
            assert codes == (0,) and len(cands) == count
            top = sorted(cands, key=lambda c: c[8])[0]
            _same_best((top[0], top[1], spec.seqs.index(tuple(top[2])) if not isinstance(top[2], int) else top[2],
                        list(top[3]), [tuple(x) for x in top[4]], top[5], list(top[6]), top[7], top[8]), best)
        except (KeyError, IndexError, RuntimeError, ZeroDivisionError) as exc:
            assert _status_of(exc)[0] in codes, (j, exc)
        got, zero = host_draw(problem, ns, j, row, code, s)
        assert zero == 0
        sample = flatten.FlatProblem(problem.scalars, dict(problem.arrays, **got), problem.type_names,
                                     problem.key_names, problem.node_sequences)
        rec, det, summary = hs.host_het_search(sample, space, mode=0)
        fatal = int(summary.fatal_code) if summary.fatal_ordinal != 2 ** 64 - 1 else 0
        assert fatal in codes, j
        if fatal:
            continue
        assert len(rec) == count
        top = sorted(hs.unpack_candidates(rec, det, space), key=lambda c: c[8])[0]
        _same_best((top[0], top[1], top[2], top[3], top[4], top[5], top[6], top[7], top[8]), best)
    nz_meta, nz = load_golden(f'noise_{name}')
    at = int(np.argsort(spec.arr['cost'], kind='stable')[0])
    assert (nz_meta['seed'], nz_meta['sigma']) == (meta['seed'], meta['sigma'])
    assert (_bits(np.where(np.isnan(gold['kept_cost']), np.nan, gold['kept_cost'])) ==
            _bits(np.where(np.isnan(nz['costs'][:, at]), np.nan, nz['costs'][:, at]))).all()


class _Winners:
    def __init__(self, tuples):
        self._t = tuples

    def __len__(self):
        return len(self._t)

    def tuples(self, idx):
        return [self._t[int(i)] for i in idx]


class _Searched:
    def __init__(self, kept_tuple, ordinal):
        self.records = np.zeros(1, dtype=native.RECORD_DTYPE)
        self.records['ordinal'] = ordinal
        self._t = kept_tuple

    def tuples(self, idx):
        return [self._t]


def test_scenario_search_fields():
    """same, same_plan, loss (negative, +inf and NaN cases), near and the winners' order equal their plain-Python
    definitions."""
    kept = (('A100',), [4], [(2, 2)], 8, [0, 10], 1, 5.0)
    other = (('A100',), [4], [(4, 1)], 8, [0, 10], 1, 4.0)
    moved = (('A100',), [4], [(2, 2)], 8, [0, 10], 2, 4.5)
    # per scenario: (status, found, best ordinal, winner, best cost, kept cost, kept usable)
    rows = [(0, True, 7, kept, 5.0, 5.0, True), (0, True, 3, other, 4.0, 4.02, True), (0, True, 3, other, 4.0, 7.0, False),
            (4, False, 0, None, 0.0, 6.0, True), (0, True, 7, moved, 5.5, 5.25, True), (0, True, 3, other, 3.0, 9.0, True),
            (0, False, 0, None, 0.0, np.nan, False)]
    K = len(rows)
    best = np.zeros(K, dtype=native.RECORD_DTYPE)
    best['ordinal'] = [r[2] for r in rows]
    best['cost'] = [r[4] for r in rows]
    found = np.array([r[1] for r in rows])
    winners = _Winners([r[3] for r in rows if r[1]])
    within = 0.01
    got = search.ScenarioSearch(_Searched(kept, 7), 0, np.array([r[0] for r in rows]), np.array([9] * K), best, found,
                                winners, np.array([r[5] for r in rows]), np.array([r[6] for r in rows]), within, {})
    for j, (st, f, o, w, bc, kc, ku) in enumerate(rows):
        assert got.winner(j) == w
        if not f:
            want_loss = np.nan
        else:
            want_loss = kc - bc if ku else np.inf
        assert _bits(got.loss[j]) == _bits(want_loss), j
        assert got.near[j] == bool(f and ku and kc <= bc * (1.0 + within))
        assert got.same[j] == (w is not None and w[:6] == kept[:6])
        assert got.same_plan[j] == (f and o == 7)
    assert got.loss[4] < 0 and np.isinf(got.loss[2]) and np.isnan(got.loss[3])
    assert list(got.near) == [True, True, False, False, True, False, False]
    assert [(t, c, j) for t, c, j in got.winners()] == [(other, 3, 1), (kept, 1, 0), (moved, 1, 4)]


class _FakeCandidates:
    """No search: what the what-ifs check before the device is touched, the window count included."""
    cost = np.zeros(0)

    def __init__(self, problem, segments=1):
        self.problem = problem
        self.segments = [None] * segments

    def __len__(self):
        return 0

    def search_scenarios(self, scenarios, kept, within):
        search.one_search_segment(self)


def test_search_noise_validates(workload_dir):
    """search_noise refuses what profile_noise refuses, with the same messages; search_profiles what recost_profiles
    refuses; a result of more than one window raises NotImplementedError naming the window count."""
    spec = Spec('mix32', workload_dir)
    problem, _space = spec.problem(spec.root)
    res = api.HetSearchResult(_FakeCandidates(problem), None, {'corrected': ()})
    base = tpr.base_profile(spec)
    res._norm_source = api.norm_source(base)
    for bad, match in ((float('nan'), 'finite'), (1.0, r'\[0, 1\)'), ({'time': 0.1}, "unknown field 'time'"),
                       ({'memory': {'X100': 0.1}}, "unknown device type 'X100'")):
        with pytest.raises(ValueError, match=match):
            res.search_noise(4, bad)
    for seed in (-1, 2 ** 64, True):
        with pytest.raises(ValueError, match='seed'):
            res.search_noise(4, 0.1, seed=seed)
    for samples in (0, 65536, 2.0):
        with pytest.raises(ValueError, match='samples'):
            res.search_noise(samples, 0.1)
    for within in (-0.01, float('inf'), '0'):
        with pytest.raises(ValueError, match='within'):
            res.search_noise(4, 0.1, within=within)
    res._norm_source = None
    with pytest.raises(ValueError, match='layer weights'):
        res.search_noise(4, 0.1)
    with pytest.raises(ValueError, match='inputs it was searched on'):
        res.search_profiles([base])
    windowed = api.HetSearchResult(_FakeCandidates(problem, 3), None, {'corrected': ()})
    windowed._norm_source = api.norm_source(base)
    with pytest.raises(NotImplementedError, match='3 windows'):
        windowed.search_noise(4, 0.1)
    fake, _problem = tpr._fake_result(spec)
    fake.candidates = _FakeCandidates(problem)
    with pytest.raises(ValueError, match='at least one profile'):
        fake.search_profiles([])
    no_model = copy.deepcopy(base)
    del no_model['model']
    with pytest.raises(ValueError, match="profile 1: no 'model' section"):
        fake.search_profiles([base, no_model])
    no_type = {k: v for k, v in base.items() if k != f'DeviceType.{problem.type_names[0]}'}
    with pytest.raises(ValueError, match=f'profile 0: no DeviceType.{problem.type_names[0]}'):
        fake.search_profiles([no_type])
    fake.candidates = _FakeCandidates(problem, 2)
    with pytest.raises(NotImplementedError, match='2 windows'):
        fake.search_profiles([base])


def test_search_noise_argument_checks(workload_dir):
    """metis_het_search_noise_* refuse NULLs, sample ranges, a small workspace and a bad norm source with METIS_E_ARG
    (METIS_E_CAPACITY for the workspace) before touching the device; a sample's problem is the base's with its five
    drawn tables in the workspace."""
    lib = native.load_library()
    spec = Spec('mix32', workload_dir)
    problem, _space = spec.problem(spec.root)
    keep = dict(problem.arrays)
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    E_ARG, E_CAPACITY = -2, -3
    need = lib.metis_het_search_noise_workspace_bytes(C.byref(p), C.c_int32(2))
    assert need >= lib.metis_het_profile_noise_workspace_bytes(C.byref(p), C.c_int32(2)) > 0
    for args in ((None, 1), (C.byref(p), 0), (C.byref(p), 65536)):
        assert lib.metis_het_search_noise_workspace_bytes(*args) == E_ARG
    buf = np.zeros(8, dtype=np.float64)
    ptr = C.c_void_p(buf.ctypes.data)
    L = problem.scalars['norm_len']

    def norm(**kw):
        n = native.MetisNormSource(ptr.value, L, 1, 0.1)
        for k, v in kw.items():
            setattr(n, k, v)
        return n

    def draw(base=C.byref(p), spec_=None, nrm=None, ws=ptr, wsb=need, zero=ptr):
        return lib.metis_het_search_noise_draw(base, spec_ if spec_ is not None else C.byref(tpn.noise_spec(
            problem, 0.1, 5, 0, 2)), nrm if nrm is not None else C.byref(norm()), ws, C.c_int64(wsb), zero, None)
    for kw in (dict(base=None), dict(ws=None), dict(zero=None), dict(nrm=C.byref(norm(row=None)))):
        assert draw(**kw) == E_ARG, kw
    assert lib.metis_het_search_noise_draw(C.byref(p), None, C.byref(norm()), ptr, C.c_int64(need), ptr, None) == E_ARG
    assert lib.metis_het_search_noise_draw(C.byref(p), C.byref(tpn.noise_spec(problem, 0.1, 5, 0, 2)), None, ptr,
                                           C.c_int64(need), ptr, None) == E_ARG
    for kw in (dict(count=0), dict(count=65536), dict(first=-1), dict(first=65534)):
        ns = tpn.noise_spec(problem, 0.1, 5, 0, 2)
        for k, v in kw.items():
            setattr(ns, k, v)
        assert draw(spec_=C.byref(ns)) == E_ARG, kw
    for kw in (dict(len=L - 1), dict(len=L + 1), dict(type_code=0), dict(type_code=7), dict(sigma=1.0),
               dict(sigma=float('nan')), dict(sigma=-0.1)):
        assert draw(nrm=C.byref(norm(**kw))) == E_ARG, kw
    assert draw(wsb=need - 1) == E_CAPACITY
    ns = tpn.noise_spec(problem, 0.1, 5, 0, 2)
    out = native.MetisProblem()
    for s in (-1, 2):
        assert lib.metis_het_search_noise_problem(C.byref(p), C.byref(ns), C.c_int32(s), ptr, C.byref(out)) == E_ARG
    assert lib.metis_het_search_noise_problem(C.byref(p), C.byref(ns), C.c_int32(0), None, C.byref(out)) == E_ARG
    assert lib.metis_het_search_noise_problem(C.byref(p), C.byref(ns), C.c_int32(0), ptr, None) == E_ARG
    got = []
    for s in (0, 1):
        assert lib.metis_het_search_noise_problem(C.byref(p), C.byref(ns), C.c_int32(s), ptr, C.byref(out)) == 0
        drawn = ('layer_compute', 'layer_memory', 'exec_full', 'fb_sync', 'norm_lc')
        for name, _t in native.MetisProblem._fields_:
            if name not in drawn:
                assert getattr(out, name) == getattr(p, name), name
        got.append([getattr(out, n) for n in drawn])
    base_at = (ptr.value + 255) // 256 * 256
    K, row = problem.scalars['num_keys'], problem.scalars['num_keys'] * problem.scalars['lpad']
    stride = got[1][0] - got[0][0]
    assert stride > 0 and stride % 256 == 0 and got[0][0] > base_at
    assert [a - got[0][0] for a in got[0]] == [0, 8 * row, 16 * row, 16 * row + 8 * K, 16 * row + 16 * K]
    assert got[0][0] + stride * 2 <= base_at + need


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _fresh(spec, profile, corrected=(), balancer_profile=None):
    """api.cost_het_cluster under ``profile`` (estimator and balancer built from it, or the balancer from
    ``balancer_profile``), the golden's args and cluster: the result, or the exception it raises."""
    from metis_b200.arguments import parse_args
    from metis_b200.utils import ModelConfig
    cluster = spec.cluster(spec.root)
    cfg = ModelConfig(model_name='t', num_layers=spec.num_layers, sequence_length=spec.sequence_length,
                      vocab_size=spec.vocab_size, hidden_size=spec.hidden_size, attention_head_size=32)
    args = parse_args(['--num_layers', str(spec.num_layers), '--gbs', str(spec.gbs),
                       '--hidden_size', str(spec.hidden_size), '--sequence_length', str(spec.sequence_length),
                       '--vocab_size', str(spec.vocab_size), '--attention_head_size', '32',
                       '--max_profiled_tp_degree', str(spec.max_tp), '--max_profiled_batch_size', str(spec.max_bs),
                       '--min_group_scale_variance', str(spec.variance), '--max_permute_len', str(spec.max_permute_len)])
    try:
        volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
        return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                    api.LayerLoadBalancer(cluster, balancer_profile or profile, cfg, args.gbs),
                                    node_sequences=spec.seqs,
                                    device='cuda:0', corrected=corrected)
    except (KeyError, IndexError, RuntimeError, ZeroDivisionError) as exc:
        return exc


def _identity(res, spec, dicts, got, corrected=(), within=0.01):
    """Every field of ``got`` against fresh searches under ``dicts`` and recost_profiles of the searched best."""
    kept = res.best()
    kept_at = res._best_position()
    rc = res.recost_profiles(dicts)
    assert len(got) == len(dicts)
    statuses = set()
    for j, prof in enumerate(dicts):
        fresh = _fresh(spec, prof, corrected)
        if isinstance(fresh, Exception):
            assert got.status[j] in _status_of(fresh), (j, fresh)
            assert got.num_candidates[j] == 0 and got.winner(j) is None and np.isnan(got.best_cost[j])
            statuses.add(int(got.status[j]))
        else:
            assert got.status[j] == 0 and got.num_candidates[j] == len(fresh)
            w = fresh.best()
            assert got.winner(j) == w
            if w is None:
                assert np.isnan(got.best_cost[j])
            else:
                assert _bits(got.best_cost[j]) == _bits(w[6])
        if kept is None:
            assert np.isnan(got.kept_cost[j]) and not got.kept_usable[j]
        else:
            assert _bits(got.kept_cost[j]) == _bits(rc.costs[j, kept_at])
            assert got.kept_usable[j] == rc.usable[j, kept_at]
        w = got.winner(j)
        if w is None:
            assert np.isnan(got.loss[j]) and not got.near[j] and not got.same[j]
        elif not got.kept_usable[j]:
            assert got.loss[j] == np.inf and not got.near[j]
        else:
            assert _bits(got.loss[j]) == _bits(got.kept_cost[j] - got.best_cost[j])
            assert got.near[j] == (got.kept_cost[j] <= got.best_cost[j] * (1.0 + within))
        assert got.same[j] == (w is not None and kept is not None and w[:6] == kept[:6])
    return statuses


def _noise(res, spec, sigma, seed, K, corrected=()):
    got = res.search_noise(K, sigma, seed)
    dicts = [search.noisy_profile(tpr.base_profile(spec), sigma, seed, j) for j in range(K)]
    _identity(res, spec, dicts, got, corrected)
    return got


FRESH = ['mix32', 'rough_q10', 'rough_t3', 'c2_het16', 'node_mem_order', 'lim_s128_l255', 'rough_q10:Q5Q6']


@pytest.mark.gpu
@pytest.mark.parametrize('name', FRESH)
def test_api_search_noise_is_fresh_searches(name, workload_dir, monkeypatch):
    """search_noise equals K fresh cost_het_cluster calls under the samples' dicts, field for field; one sample per
    chunk gives the same."""
    _gpu()
    base, _, fix = name.partition(':')
    corrected = ('Q5', 'Q6') if fix else ()
    spec = Spec(base, workload_dir)
    api.release_engines()
    res = _run(spec, spec.root, corrected)
    got = _noise(res, spec, tpn.SIGMAS['per_type'], 31, 6, corrected)
    assert got.timings['chunks'] == 1
    monkeypatch.setattr(search, '_SCENARIO_BUDGET_BYTES', 1)
    small = res.search_noise(6, tpn.SIGMAS['per_type'], 31)
    assert small.timings['chunks'] == 6
    for k in ('status', 'num_candidates', 'best_cost', 'kept_cost', 'kept_usable', 'loss', 'near', 'same', 'same_plan'):
        assert np.array_equal(np.asarray(getattr(small, k)).view(np.uint8), np.asarray(getattr(got, k)).view(np.uint8))
    assert [small.winner(j) for j in range(6)] == [got.winner(j) for j in range(6)]
    api.release_engines()


@pytest.mark.gpu
def test_api_search_noise_device_listed(workload_dir, monkeypatch):
    """A space the device listing searched as one window."""
    _gpu()
    spec = Spec('mix32', workload_dir)
    api.release_engines()
    res = _run(spec, spec.root, (), 'device_listed', monkeypatch)
    assert res.summary['listing'] == 'device' and res.summary['num_windows'] == 1
    _noise(res, spec, 0.15, 8, 4)
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name', tpr.GOLDENS)
def test_api_search_profiles_is_fresh_searches(name, workload_dir):
    """search_profiles over the profile goldens' six scenarios equals fresh searches under them, a raising one
    included."""
    _gpu()
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = _run(spec, spec.root)
    _gold, profiles = tpr.golden_scenarios(spec)
    got = res.search_profiles(profiles)
    _identity(res, spec, profiles, got)
    assert got.same[0] and got.loss[0] == 0.0                  # the first scenario is the profile itself
    api.release_engines()


@pytest.mark.gpu
def test_api_zero_noise_is_the_result(workload_dir):
    """Under all-zero sigma every sample's search is the result: its best cost bit for bit, same, loss 0."""
    _gpu()
    spec = Spec('rough_t3', workload_dir)
    api.release_engines()
    res = _run(spec, spec.root)
    got = res.search_noise(5, 0.0, 3)
    best = res.best()
    assert (got.status == 0).all() and (got.num_candidates == len(res)).all()
    assert (_bits(got.best_cost) == _bits(best[6])).all() and got.same.all() and got.same_plan.all()
    assert (got.loss == 0.0).all() and got.near.all()
    assert got.winners() == [(best, 5, 0)]
    api.release_engines()


@pytest.mark.gpu
def test_api_windows_raise(workload_dir, monkeypatch):
    """A result searched in forced windows raises NotImplementedError naming the window count."""
    _gpu()
    spec = Spec('mix32', workload_dir)
    api.release_engines()
    res = _run(spec, spec.root, (), 'windows', monkeypatch)
    n = res.summary['num_windows']
    assert n > 1
    with pytest.raises(NotImplementedError, match=f'{n} windows'):
        res.search_noise(2, 0.1)
    with pytest.raises(NotImplementedError, match=f'{n} windows'):
        res.search_profiles([tpr.base_profile(spec)])
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name,K', [('c3_homo64_mpl6', 16), ('c4_het128', 4)])
def test_api_whole_space(name, K, workload_dir):
    """C3-mpl6 at K = 16 and C4-mpl4 at K = 4 match fresh searches."""
    _gpu()
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = _run(spec, spec.root)
    _noise(res, spec, 0.05, 2024, K)
    api.release_engines()


@pytest.mark.gpu
def test_search_noise_survives_list_and_a_later_search(workload_dir):
    """A search what-if taken after list(result) and after a later cost_het_cluster() call on other inputs is
    unchanged, and a search after the what-if returns what it returned before."""
    _gpu()
    spec = Spec('rough_t3', workload_dir)
    api.release_engines()
    first = _run(spec, spec.root)
    before = first.search_noise(6, 0.2, 77)
    after_search = _run(spec, spec.root)
    assert after_search == first
    assert len(list(first)) == len(first)
    after_list = first.search_noise(6, 0.2, 77)
    other = Spec('mix32', workload_dir)
    assert len(_run(other, other.root)) != len(first)
    after = first.search_noise(6, 0.2, 77)
    for got in (after_list, after):
        for k in ('status', 'num_candidates', 'best_cost', 'kept_cost', 'kept_usable', 'loss', 'near', 'same'):
            assert np.array_equal(np.asarray(getattr(got, k)).view(np.uint8),
                                  np.asarray(getattr(before, k)).view(np.uint8)), k
        assert [got.winner(j) for j in range(6)] == [before.winner(j) for j in range(6)]
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name', GOLDENS)
def test_api_search_noise_goldens(name, workload_dir):
    """Both goldens through the api: each sample's status, count, winner and best cost bits are the reference's, and
    the searched best's cost and fit under it are the noise golden's."""
    _gpu()
    spec = Spec(name, workload_dir)
    meta, gold, _dicts, want = golden_samples(spec, name)
    api.release_engines()
    res = _run(spec, spec.root)
    got = res.search_noise(meta['samples'], meta['sigma'], meta['seed'])
    for j, (codes, count, best) in enumerate(want):
        assert got.status[j] in codes
        if codes != (0,):
            continue
        assert got.num_candidates[j] == count
        w = got.winner(j)
        ordinal = int(got._best['ordinal'][j])
        _same_best((ordinal, int(got._best['step'][j]), spec.seqs.index(tuple(w[0])), w[1], w[2], w[3], w[4], w[5],
                    w[6]), best)
        assert _bits(got.best_cost[j]) == _bits(best[8])
        assert got.same_plan[j] == (ordinal == meta['searched'][0])
    usable = (gold['kept_cost_exc'] == 0) & (gold['kept_memory_exc'] == 0) & (gold['kept_headroom'] >= 0)
    assert (got.kept_usable == usable).all()
    assert (_bits(np.where(np.isnan(got.kept_cost), np.nan, got.kept_cost)) ==
            _bits(np.where(np.isnan(gold['kept_cost']), np.nan, gold['kept_cost']))).all()
    assert (~got.same_plan).sum() >= len(meta['other_winner']) > 0
    api.release_engines()


@pytest.mark.gpu
def test_api_statuses_hang(workload_dir):
    """Seeded scenario profiles of C3-mpl6 under some of which the reference's balancer loop never ends: those come back
    as METIS_FATAL_HANG (a status; nothing hangs on the device), the rest as fresh searches."""
    _gpu()
    spec = Spec('c3_homo64_mpl6', workload_dir)
    api.release_engines()
    res = _run(spec, spec.root)
    base = tpr.base_profile(spec)
    profiles = [op.scenario(base, op.KINDS[s % len(op.KINDS)], s, spec.seqs) for s in range(1000, 1024)]
    got = res.search_profiles(profiles)
    statuses = _identity(res, spec, profiles, got)
    assert 4 in statuses, statuses
    api.release_engines()


@pytest.mark.gpu
def test_api_statuses_keyerror_and_zero_norm(workload_dir, monkeypatch):
    """A profile whose search raises KeyError and one whose layer-weight total is 0 (METIS_FATAL_ZERODIV, nothing
    searched) through search_profiles; and search_noise on a result whose profile lists first a device type outside the
    cluster with an all-zero tp1_bs1 row, so that every sample's drawn total is 0 and is flagged on the device, with the
    default chunk and one sample per chunk."""
    _gpu()
    spec = Spec('mix32', workload_dir)
    api.release_engines()
    res = _run(spec, spec.root)
    base = tpr.base_profile(spec)
    problem, _space = spec.problem(spec.root)
    missing = copy.deepcopy(base)
    del missing[f'DeviceType.{problem.type_names[-1]}']['tp1_bs1']
    zero = copy.deepcopy(base)
    first = next(iter(zero))
    zero[first]['tp1_bs1']['time']['layer-computes'] = [0.0] * len(zero[first]['tp1_bs1']['time']['layer-computes'])
    got = res.search_profiles([base, missing, zero])
    statuses = _identity(res, spec, [base, missing, zero], got)
    assert got.status[0] == 0 and got.status[1] in (1, 2) and got.status[2] == native.FATAL_ZERODIV
    assert statuses == {int(got.status[1]), native.FATAL_ZERODIV}
    other = next(t for t in DeviceType.__members__ if t not in problem.type_names)
    entry = copy.deepcopy(base[first])
    entry['tp1_bs1']['time']['layer-computes'] = [0.0] * len(entry['tp1_bs1']['time']['layer-computes'])
    odd = {f'DeviceType.{other}': entry, **base}
    searched = _fresh(spec, odd, balancer_profile=base)
    assert not isinstance(searched, Exception) and searched.best() == res.best()
    sigma = {'layer-computes': {other: 0.2}, 'memory': 0.1}
    for budget in (None, 1):
        if budget is not None:
            monkeypatch.setattr(search, '_SCENARIO_BUDGET_BYTES', budget)
        got = searched.search_noise(5, sigma, 9)
        assert got.timings['chunks'] == (5 if budget else 1)
        assert (got.status == native.FATAL_ZERODIV).all() and (got.num_candidates == 0).all()
        dicts = [search.noisy_profile(odd, sigma, 9, j) for j in range(5)]
        assert _identity(searched, spec, dicts, got) == {native.FATAL_ZERODIV}
    api.release_engines()
