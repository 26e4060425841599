"""Profile-noise what-if of a finished search (metis_het_profile_noise_*, HetSearchResult.profile_noise): how often each
candidate wins, stays near the best and fits over seeded samples of the searched profile drawn on the device.

CPU: Philox4x32-10 against the Random123 known answers; the host build of the draw (tests/hostsim/noise_sim.cpp)
against flatten.build_problem(noisy_profile(...)) bit for bit; the host build of the reduction against the numpy
definitions on ties, empty samples, chunk sizes and visit orders; the noise_* goldens of the unmodified reference
against the oracle and the host build; the ValueError cases and the argument checks.  GPU (-m gpu): the device Philox
against curand; profile_noise against the numpy definitions over recost_profiles of the samples' dicts, as one search,
in forced windows and device-listed, with small and default chunks, and on all of C3-mpl6 and C4-mpl4; zero noise; the
goldens through the api; a what-if taken after list(result) and after a later search.
"""
import copy
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
import oracle_profile as op
import test_profile_recost as tpr
from conftest import load_golden
from metis_b200 import native, search
from test_recost import Spec, _gpu, _run, host_search

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'noise_sim.cpp')
SIM_DEPS = [SIM_SRC] + [os.path.join(HERE, '..', 'metis_b200', 'csrc', f)
                        for f in ('metis_eval.cuh', 'metis_noise.cuh', 'metis_query.cuh')] + \
    [os.path.join(HERE, '..', 'include', 'metis_b200.h')]
NOISE_GOLDENS = ['mix32', 'rough_q10']
DRAW = ['mix32', 'rough_t3', 'rough_q10', 'long_profile', 'lim_s128_l255']
SIGMAS = {
    'all': 0.2,
    'per_field': {'layer-computes': 0.3, 'memory': 0.0, 'fb_sync': 0.05},
    'per_type': {'layer-computes': {'A100': 0.25, 'H100': 0.1, 'V100': 0.5, 'T4': 0.4, 'P100': 0.3},
                 'memory': {'H100': 0.5, 'A100': 0.0}, 'fb_sync': {'V100': 0.9, 'A100': 0.15}},
}
_sim = []


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def sim():
    """The g++ build of tests/hostsim/noise_sim.cpp, hostsim.cpp's flags."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'libnoise_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)                             # atomic: concurrent test processes may race
        _sim.append(C.CDLL(out))
    return _sim[0]


# ---- the numpy definitions ------------------------------------------------------------------------------------------
def reference(costs, usable, within):
    """The per-sample best and per-candidate statistics of HetSearchResult.profile_noise, defined on c [K, n] and
    usable [K, n] (what recost_profiles gives the samples)."""
    K, n = costs.shape
    t = 1.0 + within
    best_pos, best_cost = np.full(K, -1, dtype=np.int64), np.full(K, np.nan)
    for j in range(K):
        idx = np.nonzero(usable[j])[0]
        if len(idx):
            i = int(idx[np.nonzero(costs[j, idx] == costs[j, idx].min())[0][0]])
            best_pos[j], best_cost[j] = i, costs[j, i]
    wins = np.bincount(best_pos[best_pos >= 0], minlength=n)[:n]
    count = usable.sum(axis=0)
    with np.errstate(invalid='ignore'):
        near = (usable & (costs <= (best_cost * t)[:, None])).sum(axis=0)
        regret = np.where(usable.all(axis=0), (costs - best_cost[:, None]).max(axis=0), np.inf)
    total = np.zeros(n)
    for j in range(K):                                      # left to right in j
        total = np.where(usable[j], total + costs[j], total)
    with np.errstate(invalid='ignore', divide='ignore'):
        mean = np.where(count > 0, total / np.maximum(count, 1), np.nan)
    return dict(best_pos=best_pos, best_cost=best_cost, wins=wins, near=near, usable=count, regret=regret, mean=mean)


def same_stats(got, want):
    for k, v in want.items():
        g = got[k] if isinstance(got, dict) else getattr(got, k)
        if np.asarray(v).dtype.kind == 'f':
            assert (op.nan_bits(g) == op.nan_bits(v)).all(), k
        else:
            assert (np.asarray(g) == np.asarray(v)).all(), k


# ---- host builds ----------------------------------------------------------------------------------------------------
def noise_spec(problem, sigma, seed, first=0, count=1, within=0.01):
    sig = search.noise_sigmas(sigma)
    spec = native.MetisNoiseSpec()
    for f, field in enumerate(search.NOISE_FIELDS):
        for t, name in enumerate(problem.type_names):
            spec.sigma[f][t] = search._sigma_of(sig, field, name)
    for t, name in enumerate(problem.type_names):
        spec.type_code[t] = search.device_type_code(name)
    spec.seed, spec.first, spec.count, spec.near_factor = seed, first, count, 1.0 + within
    return spec


def host_draw(problem, spec, s):
    keep = dict(problem.arrays)
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    K, L = problem.scalars['num_keys'], problem.scalars['lpad']
    lc, lm, ef, fb = np.zeros((K, L)), np.zeros((K, L)), np.zeros(K), np.zeros(K)
    assert sim().noise_sim_draw(C.byref(p), C.byref(spec), C.c_int32(s), C.c_void_p(lc.ctypes.data),
                                C.c_void_p(lm.ctypes.data), C.c_void_p(ef.ctypes.data), C.c_void_p(fb.ctypes.data)) == 0
    return dict(layer_compute=lc, layer_memory=lm, exec_full=ef, fb_sync=fb)


def host_reduce(costs, usable, within, chunk, rng):
    K, n = costs.shape
    acc = dict(wins=np.zeros(n, np.int32), near=np.zeros(n, np.int32), usable=np.zeros(n, np.int32),
               regret=np.full(n, -np.inf), sum=np.zeros(n))
    best_pos, best_cost = np.zeros(K, np.int64), np.zeros(K)
    p = lambda a: C.c_void_p(a.ctypes.data)                 # noqa: E731
    for first in range(0, K, chunk):
        c = np.ascontiguousarray(costs[first:first + chunk])
        u = np.ascontiguousarray(usable[first:first + chunk]).astype(np.uint8)
        visit = rng.permutation(n).astype(np.int64)
        bp, bc = np.zeros(len(c), np.int64), np.zeros(len(c))
        assert sim().noise_sim_reduce(C.c_int32(len(c)), C.c_double(1.0 + within), p(c), p(u), C.c_int64(n), p(visit),
                                      p(bp), p(bc), p(acc['wins']), p(acc['near']), p(acc['usable']),
                                      p(acc['regret']), p(acc['sum'])) == 0
        best_pos[first:first + len(c)], best_cost[first:first + len(c)] = bp, bc
    with np.errstate(invalid='ignore', divide='ignore'):
        mean = np.where(acc['usable'] > 0, acc['sum'] / np.maximum(acc['usable'], 1), np.nan)
    return dict(best_pos=best_pos, best_cost=best_cost, wins=acc['wins'], near=acc['near'], usable=acc['usable'],
                regret=acc['regret'], mean=mean)


def noise_dicts(spec, sigma, seed, K):
    base = tpr.base_profile(spec)
    return [search.noisy_profile(base, sigma, seed, j) for j in range(K)]


# ---- CPU ------------------------------------------------------------------------------------------------------------
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


def test_philox_known_answers():
    """Philox4x32-10 in Python and in the host build of metis_noise.cuh give the Random123 known answers, and agree on
    seeded counters and keys."""
    rng = np.random.default_rng(1)
    ctr = np.concatenate([np.array([c for c, _k, _r in KAT], np.uint32),
                          rng.integers(0, 2 ** 32, (300, 4), dtype=np.uint32)])
    key = np.concatenate([np.array([k for _c, k, _r in KAT], np.uint32),
                          rng.integers(0, 2 ** 32, (300, 2), dtype=np.uint32)])
    out = np.zeros_like(ctr)
    assert sim().noise_sim_philox(C.c_void_p(ctr.ctypes.data), C.c_void_p(key.ctypes.data),
                                  C.c_void_p(out.ctypes.data), C.c_int64(len(ctr))) == 0
    for i, (_c, _k, want) in enumerate(KAT):
        assert tuple(out[i].tolist()) == want
        assert search.philox4x32_10(ctr[i].tolist(), key[i].tolist()) == want
    for i in range(len(ctr)):
        assert search.philox4x32_10(ctr[i].tolist(), key[i].tolist()) == tuple(out[i].tolist())


@pytest.mark.parametrize('kind', sorted(SIGMAS))
@pytest.mark.parametrize('name', DRAW)
def test_host_draw_is_build_problem(name, kind, workload_dir):
    """The draw kernels' code, from the searched problem's flat tables, gives sample j's layer_compute, layer_memory,
    exec_full and fb_sync exactly as flatten.build_problem of noisy_profile(profile, sigma, seed, j) does; the sample's
    other tables are the searched problem's."""
    spec = Spec(name, workload_dir)
    problem, _space = spec.problem(spec.root)
    seed = 0x1234_5678_9abc_def0
    for first in (0, 5):
        dicts = [search.noisy_profile(tpr.base_profile(spec), SIGMAS[kind], seed, j) for j in (first, first + 1)]
        flat = tpr.scenario_problems(spec, dicts)
        ns = noise_spec(problem, SIGMAS[kind], seed, first, 2)
        for s in range(2):
            got = host_draw(problem, ns, s)
            for k, v in flat[s].arrays.items():
                want = got.get(k, problem.arrays[k])
                assert np.array_equal(np.asarray(v).view(np.uint8), np.asarray(want).view(np.uint8)), (k, s)
            assert flat[s].scalars == problem.scalars
    if kind == 'all':
        assert (got['exec_full'] != problem.arrays['exec_full']).any()


def test_zero_sigma_is_the_profile(workload_dir):
    """Under sigma 0 a sample is the profile itself, ints included; the 'model' section is never touched."""
    spec = Spec('rough_q10', workload_dir)
    base = tpr.base_profile(spec)
    for sigma in (0.0, {}, {'memory': {'A100': 0.0}}):
        got = search.noisy_profile(base, sigma, 3, 7)
        assert got == base and got is not base
        assert op.sha256(got) == op.sha256(base)
    got = search.noisy_profile(base, 0.3, 3, 7)
    assert got['model'] == base['model']
    assert got != base and search.noisy_profile(base, 0.3, 3, 7) == got


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_host_reduce_equals_numpy(seed):
    """The reduction's code equals the numpy definitions on tied and duplicate costs, samples where nothing is
    usable, a candidate usable in every sample, chunks of 1, 3 and K samples and random visit orders."""
    rng = np.random.default_rng(seed)
    K, n = 11, 37
    costs = rng.choice([1.0, 2.0, 2.0, 3.5, -0.0, 0.0, 7.25], size=(K, n))
    usable = rng.random((K, n)) < 0.6
    usable[:, 5] = True
    usable[4] = False
    costs[~usable & (rng.random((K, n)) < 0.5)] = np.nan
    want = reference(costs, usable, 0.25)
    assert (want['best_pos'][4] == -1) and np.isnan(want['best_cost'][4])
    for chunk in (1, 3, K):
        same_stats(host_reduce(costs, usable, 0.25, chunk, rng), want)
    assert (want['usable'][5] == K - 1) and np.isinf(want['regret'][5]) and (want['wins'] > 1).any()


@pytest.mark.parametrize('name', NOISE_GOLDENS)
def test_noise_goldens_oracle_and_host_build(name, workload_dir):
    """The noise_* goldens of the unmodified reference (8 samples): the samples rebuilt from the seed hash as
    recorded; the oracle and the host build of the profile what-if equal them bit for bit, statuses included."""
    spec = Spec(name, workload_dir)
    meta, gold = load_golden(f'noise_{name}')
    assert meta['inputs_sha256'] == spec.meta['inputs_sha256']
    dicts = noise_dicts(spec, meta['sigma'], meta['seed'], meta['samples'])
    assert [op.sha256(p) for p in dicts] == meta['sample_sha256']
    costs, head, cexc, mexc = tpr.oracle_scenarios(spec, dicts)
    assert (op.nan_bits(costs) == op.nan_bits(gold['costs'])).all()
    assert (op.nan_bits(head) == op.nan_bits(gold['headroom'])).all()
    assert (cexc == gold['cost_exc']).all() and (mexc == gold['memory_exc']).all()
    problem, space = spec.problem(spec.root)
    rec, det = host_search(problem, space)
    got = tpr.host_profile_recost(tpr.scenario_problems(spec, dicts), space, rec, det)
    tpr.same(got, gold['costs'], gold['headroom'], gold['cost_exc'], gold['memory_exc'])
    usable = (gold['cost_exc'] == 0) & (gold['memory_exc'] == 0) & (gold['headroom'] >= 0)
    assert usable.any(axis=1).all() and (~usable).any()


class _FakeCandidates:
    def __init__(self, problem):
        self.problem = problem

    def profile_noise(self, *args):
        return args


def test_profile_noise_validates(workload_dir):
    """Every ValueError case of noisy_profile and profile_noise, each naming what it refuses; the sigma table and
    device type codes reaching the device are per device type of the searched problem."""
    from metis_b200 import api
    spec = Spec('mix32', workload_dir)
    problem, _space = spec.problem(spec.root)
    res = api.HetSearchResult(_FakeCandidates(problem), None, {'corrected': ()})
    base = tpr.base_profile(spec)
    for bad, match in ((float('nan'), 'finite'), (1.0, r'\[0, 1\)'), (-0.1, r'\[0, 1\)'), ('0.1', 'finite'),
                       (True, 'finite'), ({'time': 0.1}, "unknown field 'time'"),
                       ({'memory': {'X100': 0.1}}, "unknown device type 'X100'"),
                       ({'fb_sync': {'A100': float('inf')}}, 'finite'), ({'memory': 1.5}, r'\[0, 1\)')):
        with pytest.raises(ValueError, match=match):
            search.noisy_profile(base, bad, 0, 0)
        with pytest.raises(ValueError, match=match):
            res.profile_noise(4, bad)
    for seed in (-1, 2 ** 64, 1.0, True):
        with pytest.raises(ValueError, match='seed'):
            search.noisy_profile(base, 0.1, seed, 0)
        with pytest.raises(ValueError, match='seed'):
            res.profile_noise(4, 0.1, seed=seed)
    for j in (-1, 2 ** 32, 0.0):
        with pytest.raises(ValueError, match='sample index'):
            search.noisy_profile(base, 0.1, 0, j)
    for samples in (0, 65536, 2.0, True):
        with pytest.raises(ValueError, match='samples'):
            res.profile_noise(samples, 0.1)
    for within in (-0.01, float('inf'), float('nan'), '0'):
        with pytest.raises(ValueError, match='within'):
            res.profile_noise(4, 0.1, within=within)
    odd = copy.deepcopy(base)
    odd['DeviceType.X100'] = odd[next(k for k in odd if k.startswith('DeviceType.'))]
    with pytest.raises(ValueError, match="unknown device type 'X100'"):
        search.noisy_profile(odd, 0.1, 0, 0)
    assert search.noisy_profile(odd, 0.0, 0, 0) == odd
    table, codes, seed, samples, within = res.profile_noise(9, {'memory': {problem.type_names[-1]: 0.5}}, 2 ** 64 - 1,
                                                            0.5)
    assert (seed, samples, within) == (2 ** 64 - 1, 9, 0.5)
    assert table.shape == (3, native.METIS_MAX_TYPES) and table[1, len(problem.type_names) - 1] == 0.5
    assert table.sum() == 0.5
    assert codes == [search.device_type_code(t) for t in problem.type_names]


def test_profile_noise_argument_checks(workload_dir):
    """metis_het_profile_noise_* refuse bad arguments with METIS_E_ARG (METIS_E_CAPACITY for a small workspace)
    before touching the device."""
    lib = native.load_library()
    spec = Spec('mix32', workload_dir)
    problem, space = spec.problem(spec.root)
    keep = dict(problem.arrays)
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sk = dict(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    sp = space.as_struct(lambda n: sk[n].ctypes.data)
    buf = np.zeros(4096, dtype=np.float64)
    ptr = C.c_void_p(buf.ctypes.data)
    E_ARG, E_CAPACITY = -2, -3
    need = lib.metis_het_profile_noise_workspace_bytes(C.byref(p), C.c_int32(2))
    assert need > lib.metis_het_profile_noise_workspace_bytes(C.byref(p), C.c_int32(1)) > 0
    for args in ((None, 1), (C.byref(p), 0), (C.byref(p), 65536)):
        assert lib.metis_het_profile_noise_workspace_bytes(*args) == E_ARG

    def ns(**kw):
        s = noise_spec(problem, 0.1, 5, 0, 2)
        for k, v in kw.items():
            if k == 'sigma':
                s.sigma[1][0] = v
            elif k == 'type_code':
                s.type_code[0] = v
            else:
                setattr(s, k, v)
        return s

    bad_specs = [dict(count=0), dict(count=65536), dict(first=-1), dict(first=65534), dict(sigma=float('nan')),
                 dict(sigma=1.0), dict(sigma=-0.5), dict(type_code=0), dict(type_code=7),
                 dict(near_factor=float('nan')), dict(near_factor=0.5)]

    def draw(base=C.byref(p), spec_=None, ws=ptr, wsb=need):
        return lib.metis_het_profile_noise_draw(base, spec_ if spec_ is not None else C.byref(ns()), ws,
                                                C.c_int64(wsb), None)
    for kw in (dict(base=None), dict(ws=None)):
        assert draw(**kw) == E_ARG, kw
    assert lib.metis_het_profile_noise_draw(C.byref(p), None, ptr, C.c_int64(need), None) == E_ARG
    for kw in bad_specs:
        assert draw(spec_=C.byref(ns(**kw))) == E_ARG, kw
    assert draw(wsb=need - 1) == E_CAPACITY
    stride = 3 * int(space.blocks['num_stage'].max()) + 1

    def ev(space_=C.byref(sp), spec_=None, ws=ptr, rec=ptr, n=1, det=ptr, st=stride, cost=ptr, u=ptr, ld=1):
        return lib.metis_het_profile_noise_eval(space_, spec_ if spec_ is not None else C.byref(ns()), ws, rec,
                                                C.c_int64(n), det, C.c_int32(st), cost, u, C.c_int64(ld), None)
    for kw in (dict(space_=None), dict(ws=None), dict(rec=None), dict(det=None), dict(cost=None), dict(u=None),
               dict(n=-1, ld=0), dict(n=2, ld=1), dict(st=stride - 1), dict(spec_=C.byref(ns(count=0)))):
        assert ev(**kw) == E_ARG, kw
    assert lib.metis_het_profile_noise_eval(C.byref(sp), None, ptr, ptr, C.c_int64(1), ptr, C.c_int32(stride), ptr,
                                            ptr, C.c_int64(1), None) == E_ARG

    def red(spec_=None, n=1, **kw):
        a = dict(cost=ptr, u=ptr, bp=ptr, bc=ptr, w=ptr, nr=ptr, uc=ptr, r=ptr, s=ptr)
        a.update(kw)
        return lib.metis_het_profile_noise_reduce(spec_ if spec_ is not None else C.byref(ns()), a['cost'], a['u'],
                                                  C.c_int64(n), a['bp'], a['bc'], a['w'], a['nr'], a['uc'], a['r'],
                                                  a['s'], None)
    for kw in (dict(cost=None), dict(u=None), dict(bp=None), dict(bc=None), dict(w=None), dict(nr=None),
               dict(uc=None), dict(r=None), dict(s=None), dict(n=-1), dict(spec_=C.byref(ns(count=0))),
               dict(spec_=C.byref(ns(near_factor=0.5)))):
        assert red(**kw) == E_ARG, kw
    assert lib.metis_het_profile_noise_reduce(None, ptr, ptr, C.c_int64(1), *([ptr] * 7), None) == E_ARG


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_philox_equals_curand(tmp_path):
    """metis_noise.cuh's Philox4x32-10 on the device equals curand's curand_Philox4x32_10 on 400 counters and keys,
    the Random123 known answers among them."""
    _gpu()
    from metis_b200 import build
    out = str(tmp_path / 'libphilox_check.so')
    proc = subprocess.run([build.nvcc_path()] + build.NVCC_FLAGS + ['-o', out,
                          os.path.join(HERE, 'devsim', 'philox_check.cu')], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    lib = C.CDLL(out)
    rng = np.random.default_rng(2)
    ctr = np.concatenate([np.array([c for c, _k, _r in KAT], np.uint32),
                          rng.integers(0, 2 ** 32, (397, 4), dtype=np.uint32)])
    key = np.concatenate([np.array([k for _c, k, _r in KAT], np.uint32),
                          rng.integers(0, 2 ** 32, (397, 2), dtype=np.uint32)])
    ours, theirs = np.zeros_like(ctr), np.zeros_like(ctr)
    assert lib.philox_check(C.c_void_p(ctr.ctypes.data), C.c_void_p(key.ctypes.data), C.c_void_p(ours.ctypes.data),
                            C.c_void_p(theirs.ctypes.data), C.c_int(len(ctr))) == 0
    assert (ours == theirs).all()
    for i, (_c, _k, want) in enumerate(KAT):
        assert tuple(ours[i].tolist()) == want


def _identity(res, spec, sigma, seed, K, within=0.01):
    """profile_noise against the numpy definitions over recost_profiles of the samples' dicts, every array bit for
    bit; returns the ProfileNoise."""
    got = res.profile_noise(K, sigma, seed, within)
    rc = res.recost_profiles(noise_dicts(spec, sigma, seed, K))
    want = reference(rc.costs, rc.usable, within)
    same_stats(got, want)
    return got, want


IDENTITY = tpr.GOLDENS + ['c2_het16', 'lim_s128_l255', 'rough_q10:Q5Q6']


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['one_search', 'windows', 'device_listed'])
@pytest.mark.parametrize('name', IDENTITY)
def test_api_identity(name, mode, workload_dir, monkeypatch):
    """profile_noise equals the numpy definitions over recost_profiles of noisy_profile(profile, sigma, seed, j), with
    default chunks and with one sample per chunk; the rankings follow the statistics."""
    _gpu()
    from metis_b200 import api
    base, _, fix = name.partition(':')
    corrected = ('Q5', 'Q6') if fix else ()
    spec = Spec(base, workload_dir)
    api.release_engines()
    res = _run(spec, spec.root, corrected, mode, monkeypatch)
    if mode == 'windows':
        assert res.summary['num_windows'] > 1
    sigma = SIGMAS['per_type'] if mode == 'one_search' else 0.15
    got, want = _identity(res, spec, sigma, 11, 8)
    assert got.timings['chunks'] == 1
    monkeypatch.setattr(search, '_NOISE_BUDGET_BYTES', 1)
    small = res.profile_noise(8, sigma, 11)
    assert small.timings['chunks'] == 8
    same_stats(small, want)
    n = len(res)
    for by, key in (('wins', -want['wins']), ('near', -want['near']), ('regret', want['regret']),
                    ('mean', want['mean'])):
        order = np.lexsort((np.arange(n), res.costs, key))
        got_t = got.ranked(by, 5)
        assert [t[:6] for t in got_t] == [t[:6] for t in res.candidates.tuples(order[:5])]
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['c3_homo64_mpl6', 'c4_het128'])
def test_api_identity_whole_space(name, workload_dir, monkeypatch):
    """The identity on every candidate of C3-mpl6 and C4-mpl4 at K = 64, and zero noise: the searched best winning
    every sample, usable exactly where the search's headroom is >= 0, and the search's costs as the mean of one and of
    two samples (a left-to-right sum of more equal costs may round, so that its mean is the cost to within rounding)."""
    _gpu()
    from metis_b200 import api
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = tpr._headroom_run(spec, (), 'one_search', monkeypatch)
    if name == 'c3_homo64_mpl6':
        assert len(res) == 273688
    _identity(res, spec, 0.05, 2024, 64)
    zero = res.profile_noise(16, 0.0, 5)
    fits = res.headroom >= 0
    assert (zero.usable == np.where(fits, 16, 0)).all()
    for k in (1, 2):
        mean = res.profile_noise(k, 0.0, 5).mean
        assert (_bits(mean[fits]) == _bits(res.costs[fits])).all() and np.isnan(mean[~fits]).all()
    assert np.allclose(zero.mean[fits], res.costs[fits], rtol=16 * 2.0 ** -52, atol=0)
    best = int(np.lexsort((np.arange(len(res)), np.where(fits, res.costs, np.inf)))[0])
    assert zero.wins[best] == 16 and (zero.best_pos == best).all()
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name', NOISE_GOLDENS)
def test_api_noise_goldens(name, workload_dir):
    """The noise goldens through the api: recost_profiles of the samples equals the reference, and profile_noise the
    numpy definitions over the reference's own costs and fit."""
    _gpu()
    from metis_b200 import api
    spec = Spec(name, workload_dir)
    meta, gold = load_golden(f'noise_{name}')
    api.release_engines()
    res = _run(spec, spec.root)
    dicts = noise_dicts(spec, meta['sigma'], meta['seed'], meta['samples'])
    pos = [res.candidates.index_of(o, s) for o, s in zip(spec.arr['ordinal'].tolist(), spec.arr['step'].tolist())]
    assert sorted(pos) == list(range(len(res)))
    rc = res.recost_profiles(dicts)
    tpr.same((rc.costs[:, pos], rc.headroom[:, pos], rc.status[:, pos]), gold['costs'], gold['headroom'],
             gold['cost_exc'], gold['memory_exc'])
    usable = (gold['cost_exc'] == 0) & (gold['memory_exc'] == 0) & (gold['headroom'] >= 0)
    costs = np.full(rc.costs.shape, np.nan)
    use = np.zeros(rc.costs.shape, dtype=bool)
    costs[:, pos], use[:, pos] = gold['costs'], usable
    got = res.profile_noise(meta['samples'], meta['sigma'], meta['seed'])
    same_stats(got, reference(costs, use, 0.01))
    api.release_engines()


@pytest.mark.gpu
def test_profile_noise_survives_list_and_a_later_search(workload_dir):
    """A noise what-if taken after list(result), and one after a later cost_het_cluster() call on other inputs, are
    unchanged."""
    _gpu()
    from metis_b200 import api
    spec = Spec('rough_t3', workload_dir)
    api.release_engines()
    first = _run(spec, spec.root)
    before = first.profile_noise(12, 0.2, 77)
    assert len(list(first)) == len(first)
    after_list = first.profile_noise(12, 0.2, 77)
    other = Spec('mix32', workload_dir)
    assert len(_run(other, other.root)) != len(first)
    after = first.profile_noise(12, 0.2, 77)
    want = {k: getattr(before, k) for k in ('best_pos', 'best_cost', 'wins', 'near', 'usable', 'regret', 'mean')}
    same_stats(after_list, want)
    same_stats(after, want)
    assert math.isfinite(before.best_cost[0])
    api.release_engines()
