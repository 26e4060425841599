"""Profile what-if of a finished search (metis_het_profile_recost, HetSearchResult.recost_profiles): every candidate's
cost, memory headroom and status under other profiles, with its device groups, strategies and layer partition held
fixed.

CPU: the oracle's fixed-argument restatement (tests/oracle_profile.py) against the profile_* goldens of the unmodified
reference; the host build of the kernel's loop body (tests/hostsim/profile_recost_sim.cpp) against the goldens, against
the search under its own profile (the identity), against the oracle on seeded scenario transforms, and per scenario
kind; planted defects that these checks catch; the ValueError cases and the argument checks.  GPU (-m gpu): the goldens
and the identity through the api, as one search, in forced windows and on a device-listed space, on all of C3-mpl6 and
C4-mpl4; the oracle on 20 seeded scenario sets; the rankings, regret and robust plans against numpy; a what-if taken
after list(result) and after a later search.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
import oracle_profile as op
import test_headroom as th
from conftest import load_golden
from metis_b200 import flatten, native
from metis_b200.data_loader import ProfileDataLoader
from oracle import metis_oracle as orc
from test_recost import Spec, _gpu, _run, host_search

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'profile_recost_sim.cpp')
SIM_DEPS = [SIM_SRC, hs.SRC] + [os.path.join(HERE, '..', 'metis_b200', 'csrc', f)
                                for f in ('metis_eval.cuh', 'metis_coop.cuh', 'metis_trace.cuh', 'metis_rows.cuh',
                                          'metis_recost.cuh')] + [os.path.join(HERE, '..', 'include', 'metis_b200.h')]
GOLDENS = ['mix32', 'rough_t3', 'rough_q10', 'node_mem_order']
NODE = ['node_bw_mix32', 'node_bw_t1', 'node_homo', 'node_mem_order', 'node_q10']
IDENTITY = ['c1', 'mix32', 'c2_het16', 'rough_mix2', 'rough_t3', 'rough_q10', 'het32_tight', 'lim_s128_l255',
            'lim_s128_t2'] + NODE
SEED = 7                                  # tests/golden/make_profile_golden.py
_sim = []


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def sim():
    """The g++ build of tests/hostsim/profile_recost_sim.cpp at the compiled limits, hostsim.cpp's flags."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'libprofile_recost_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)                             # atomic: concurrent test processes may race
        lib = C.CDLL(out)
        lib.profile_recost_sim_het.restype = C.c_int
        _sim.append(lib)
    return _sim[0]


# ---- inputs ---------------------------------------------------------------------------------------------------------
def base_profile(spec):
    return ProfileDataLoader(os.path.join(spec.root, spec.sub), spec.meta['file_order']).load_profile_data_all()[0]


def scenario_problems(spec, profiles, corrected=()):
    """Each profile flattened like HetSearchResult.recost_profiles does: the searched cluster, flags and corrections,
    the searched problem's norm_lc."""
    cluster = spec.cluster(spec.root)
    cfg = hs.load_inputs(spec.root, spec.sub, spec.meta['file_order'], spec.num_layers, spec.hidden_size,
                         spec.sequence_length, spec.vocab_size)[3]
    base, _space = spec.problem(spec.root, corrected)
    return [flatten.build_problem(p, cluster, cfg, spec.gbs, spec.max_tp, spec.max_bs, spec.seqs,
                                  base.arrays['norm_lc'], corrected=corrected) for p in profiles]


def host_profile_recost(problems, space, rec, det, mutant=0):
    """profile_recost_sim_het: (costs, headroom, status) [K, n]."""
    lib = sim()
    keep = [dict(p.arrays) for p in problems]
    sk = dict(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    sp = space.as_struct(lambda n: sk[n].ctypes.data)
    scen = (native.MetisProblem * len(problems))(*[p.as_struct(lambda n, k=k: k[n].ctypes.data)
                                                   for p, k in zip(problems, keep)])
    K, n = len(problems), len(rec)
    costs, head = np.full((K, n), -1.0), np.full((K, n), -1.0)
    status = np.full((K, n), 255, dtype=np.uint8)
    assert lib.profile_recost_sim_het(C.byref(sp), C.byref(scen), C.c_int32(K), C.c_void_p(rec.ctypes.data),
                                      C.c_int64(n), C.c_void_p(det.ctypes.data), C.c_int32(det.shape[1]),
                                      C.c_void_p(costs.ctypes.data), C.c_void_p(head.ctypes.data),
                                      C.c_void_p(status.ctypes.data), C.c_int32(mutant)) == 0
    return costs, head, status


def oracle_scenarios(spec, profiles, corrected=()):
    """oracle_profile.profile_recost of the golden's candidates under each profile: [K, n] arrays."""
    cl = orc.OracleCluster(os.path.join(spec.root, 'hostfile'), os.path.join(spec.root, 'clusterfile.json'),
                           corrected=corrected)
    cands = op.candidate_args(spec.arr, spec.seqs)
    dims = (spec.num_layers, spec.hidden_size, spec.sequence_length, spec.vocab_size)
    got = [op.profile_recost(p, cl, dims, spec.gbs, spec.max_bs, cands, corrected) for p in profiles]
    return tuple(np.stack([g[k] for g in got]) for k in range(4))


def golden_scenarios(spec):
    """The profile_<name> golden and the scenario dicts rebuilt from its seed, checked against its sha256."""
    meta, gold = load_golden(f'profile_{spec.meta["workload"]}')
    assert meta['inputs_sha256'] == spec.meta['inputs_sha256']
    profiles = op.scenarios(base_profile(spec), meta['seed'], spec.seqs)
    assert [op.sha256(p) for p in profiles] == meta['scenario_sha256']
    assert meta['kinds'] == list(op.KINDS)
    return gold, profiles


def same(got, want_costs, want_head, want_cexc, want_mexc):
    costs, head, status = got
    cexc, mexc = op.device_exceptions(status)
    assert (op.nan_bits(costs) == op.nan_bits(want_costs)).all()
    assert (op.nan_bits(head) == op.nan_bits(want_head)).all()
    assert (cexc == want_cexc).all() and (mexc == want_mexc).all()


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', GOLDENS)
def test_oracle_is_the_reference(name, workload_dir):
    """The oracle's fixed-argument restatement equals the profile_* goldens bit for bit, exceptions included; every
    get_cost exception of these inputs is a KeyError; every scenario kind leaves some candidates usable, and the memory
    scenario makes some of them stop fitting."""
    spec = Spec(name, workload_dir)
    gold, profiles = golden_scenarios(spec)
    costs, head, cexc, mexc = oracle_scenarios(spec, profiles)
    assert (op.nan_bits(costs) == op.nan_bits(gold['costs'])).all()
    assert (op.nan_bits(head) == op.nan_bits(gold['headroom'])).all()
    assert (cexc == gold['cost_exc']).all() and (mexc == gold['memory_exc']).all()
    assert set(np.unique(gold['cost_exc']).tolist()) <= {0, op.EXC['KeyError']}
    assert (gold['cost_exc'][op.KINDS.index('keys')] != 0).any()
    usable = (gold['cost_exc'] == 0) & (gold['memory_exc'] == 0) & (gold['headroom'] >= 0)
    assert usable[0].all() and usable.any(axis=1).all()
    mem = op.KINDS.index('memory')
    assert (usable[0] & ~usable[mem]).any()


@pytest.mark.parametrize('name', GOLDENS)
def test_host_build_equals_the_goldens(name, workload_dir):
    """The host build of the kernel's loop body, on the base search's candidates under each scenario, equals the
    reference bit for bit, statuses included."""
    spec = Spec(name, workload_dir)
    gold, profiles = golden_scenarios(spec)
    problem, space = spec.problem(spec.root)
    rec, det = host_search(problem, space)
    assert (_bits(rec['cost']) == _bits(spec.arr['cost'])).all()
    got = host_profile_recost(scenario_problems(spec, profiles), space, rec, det)
    same(got, gold['costs'], gold['headroom'], gold['cost_exc'], gold['memory_exc'])


@pytest.mark.parametrize('name', IDENTITY + ['rough_q10:Q5Q6'])
def test_own_profile_is_the_search(name, workload_dir):
    """Under the searched profile the host build gives every candidate the search's cost and the search's headroom bit
    for bit, with status 0 (also for a ('Q5', 'Q6') corrected run)."""
    base, _, fix = name.partition(':')
    corrected = ('Q5', 'Q6') if fix else ()
    spec = Spec(base, workload_dir)
    problem, space = spec.problem(spec.root, corrected)
    ordinals = None if corrected else set(spec.arr['ordinal'].tolist())
    rec, det = host_search(problem, space, ordinals)
    hrec, head = th._host_search(problem, space, 0)
    keep = np.isin(hrec['ordinal'], rec['ordinal'])
    hrec, head = hrec[keep], head[keep]
    assert (hrec['ordinal'] == rec['ordinal']).all() and (hrec['step'] == rec['step']).all()
    profile = base_profile(spec)
    costs, got_head, status = host_profile_recost(scenario_problems(spec, [profile, profile], corrected), space, rec, det)
    assert (status == 0).all()
    assert (_bits(costs) == _bits(np.stack([rec['cost']] * 2))).all()
    assert (_bits(got_head) == _bits(np.stack([head] * 2))).all()


FUZZ = [('mix32', 5), ('rough_t3', 3), ('rough_q10', 2)]          # seeds per golden: 6 scenarios each, 60 in all


@pytest.mark.parametrize('name,seeds', FUZZ)
def test_host_build_equals_the_oracle_fuzz(name, seeds, workload_dir):
    """The host build equals the oracle bit for bit on seeded scenario transforms."""
    spec = Spec(name, workload_dir)
    problem, space = spec.problem(spec.root)
    rec, det = host_search(problem, space)
    base = base_profile(spec)
    for seed in range(100, 100 + seeds):
        profiles = op.scenarios(base, seed, spec.seqs)
        got = host_profile_recost(scenario_problems(spec, profiles), space, rec, det)
        same(got, *oracle_scenarios(spec, profiles))


def test_scenario_kinds_change_what_they_should(workload_dir):
    """A memory-only scenario changes headroom and no cost; a model-section scenario changes costs and no headroom; a
    compute scenario changes costs (and the headroom of mixed-type stages, whose data split it weighs); a keys scenario
    makes some candidates unusable."""
    spec = Spec('rough_t3', workload_dir)
    problem, space = spec.problem(spec.root)
    rec, det = host_search(problem, space)
    profiles = op.scenarios(base_profile(spec), SEED, spec.seqs)
    costs, head, status = host_profile_recost(scenario_problems(spec, profiles), space, rec, det)
    k = {kind: j for j, kind in enumerate(op.KINDS)}
    assert (_bits(costs[k['memory']]) == _bits(costs[0])).all() and (head[k['memory']] != head[0]).any()
    assert (_bits(head[k['model']]) == _bits(head[0])).all() and (costs[k['model']] != costs[0]).any()
    assert (costs[k['compute']] != costs[0]).any()
    assert (status[k['keys']] != 0).any() and (status[0] == 0).all()


@pytest.mark.parametrize('mutant,name', [(1, 'rough_t3'), (2, 'mix32'), (3, 'rough_t3')])
def test_planted_defects_are_caught(mutant, name, workload_dir):
    """Memory demand from the stage's own device type (1), the dp / update terms from the searched profile's model
    section (2) and headroom over the costed stages only (3) each break the golden comparison."""
    spec = Spec(name, workload_dir)
    gold, profiles = golden_scenarios(spec)
    problem, space = spec.problem(spec.root)
    rec, det = host_search(problem, space)
    got = host_profile_recost(scenario_problems(spec, profiles), space, rec, det, mutant)
    with pytest.raises(AssertionError):
        same(got, gold['costs'], gold['headroom'], gold['cost_exc'], gold['memory_exc'])


class _FakeCandidates:
    def __init__(self, problem):
        self.problem = problem

    def recost_profiles(self, problems):
        return problems


def _fake_result(spec):
    from metis_b200 import api
    problem, _space = spec.problem(spec.root)
    cfg = hs.load_inputs(spec.root, spec.sub, spec.meta['file_order'], spec.num_layers, spec.hidden_size,
                         spec.sequence_length, spec.vocab_size)[3]
    res = api.HetSearchResult(_FakeCandidates(problem), None, {'corrected': ()})
    res._flat_inputs = (spec.cluster(spec.root), cfg, spec.gbs, spec.max_tp, spec.max_bs, spec.seqs, ())
    return res, problem


def test_recost_profiles_validates_the_profiles(workload_dir):
    """A profile without a 'model' section, one of its three fields, or an entry of a device type of the cluster is
    refused with a ValueError naming the scenario and the item; a wrong value is not refused.  The scenarios are
    flattened like the search's problem."""
    import copy
    spec = Spec('mix32', workload_dir)
    res, problem = _fake_result(spec)
    base = base_profile(spec)
    got = res.recost_profiles([base])
    assert len(got) == 1
    for k, v in problem.arrays.items():
        assert np.array_equal(np.asarray(v).view(np.uint8), np.asarray(got[0].arrays[k]).view(np.uint8)), k
    assert got[0].scalars == problem.scalars
    bad = []
    p = copy.deepcopy(base)
    del p['model']
    bad.append((p, "no 'model' section"))
    for field in ('parameters', 'optimizer_time', 'batch_generator'):
        p = copy.deepcopy(base)
        del p['model'][field]
        bad.append((p, field))
    p = copy.deepcopy(base)
    del p['DeviceType.' + problem.type_names[-1]]
    bad.append((p, 'DeviceType.' + problem.type_names[-1]))
    for p, what in bad:
        with pytest.raises(ValueError, match='profile 1: .*' + what):
            res.recost_profiles([base, p])
    with pytest.raises(ValueError, match='at least one'):
        res.recost_profiles([])
    odd = copy.deepcopy(base)
    odd['model']['optimizer_time'] = -1.0
    first = next(k for k in odd if k.startswith('DeviceType.'))
    odd[first]['tp1_bs1']['time']['fb_sync'] = 0.0
    assert len(res.recost_profiles([odd])) == 1


def test_profile_recost_argument_checks(workload_dir):
    """metis_het_profile_recost refuses bad arguments with METIS_E_ARG (METIS_E_CAPACITY for a small workspace) before
    touching the device."""
    lib = native.load_library()
    spec = Spec('mix32', workload_dir)
    problem, space = spec.problem(spec.root)
    profile = base_profile(spec)
    probs = scenario_problems(spec, [profile, profile])
    keep = [dict(p.arrays) for p in probs]
    scen = (native.MetisProblem * 2)(*[p.as_struct(lambda n, k=k: k[n].ctypes.data) for p, k in zip(probs, keep)])
    sk = dict(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    sp = space.as_struct(lambda n: sk[n].ctypes.data)
    buf = np.zeros(4096, dtype=np.float64)
    ptr = C.c_void_p(buf.ctypes.data)
    stride = 3 * int(space.blocks['num_stage'].max()) + 1
    E_ARG, E_CAPACITY = -2, -3
    sptr = C.c_void_p(C.addressof(scen))
    need = lib.metis_het_profile_recost_workspace_bytes(sptr, C.c_int32(2))
    assert need > 0

    def call(n=1, k=2, scen_=sptr, rec=ptr, det=ptr, st=stride, cost=ptr, head=ptr, status=ptr, ws=ptr, wsb=need,
             space_=C.byref(sp)):
        return lib.metis_het_profile_recost(space_, scen_, C.c_int32(k), rec, C.c_int64(n), det, C.c_int32(st), cost,
                                            head, status, ws, C.c_int64(wsb), None)
    for kw in (dict(space_=None), dict(scen_=None), dict(rec=None), dict(det=None), dict(cost=None), dict(head=None),
               dict(status=None), dict(ws=None), dict(n=-1), dict(k=0), dict(k=65536), dict(st=stride - 1)):
        assert call(**kw) == E_ARG, kw
    assert call(wsb=need - 1) == E_CAPACITY
    for field, value in (('gbs', 2 * probs[0].scalars['gbs']), ('uniform_bw', 1 - probs[0].scalars['uniform_bw']),
                         ('corrected', 2), ('q10_devices', 1), ('num_layers', 1)):
        saved = getattr(scen[1], field)
        setattr(scen[1], field, value)
        assert call() == E_ARG, field
        assert b'outside the profile' in lib.metis_last_error()
        setattr(scen[1], field, saved)
    scen[1].num_keys = 0                                      # check_problem of every scenario
    assert call() == E_ARG
    assert lib.metis_het_profile_recost_workspace_bytes(sptr, C.c_int32(2)) == E_ARG
    assert lib.metis_het_profile_recost_workspace_bytes(sptr, C.c_int32(0)) == E_ARG
    assert lib.metis_het_profile_recost_workspace_bytes(None, C.c_int32(1)) == E_ARG


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _check_views(rc):
    """ranked / best / regret / robust against numpy and Python definitions over the returned arrays."""
    usable = (rc.status == 0) & (rc.headroom >= 0)
    assert (rc.usable == usable).all()
    masked = np.where(usable, rc.costs, np.inf)
    n = rc.costs.shape[1]
    best = masked.min(axis=1) if n else np.full(len(masked), np.inf)
    assert (_bits(rc.best_costs) == _bits(best)).all()
    if n:
        with np.errstate(invalid='ignore'):
            regret = np.fmax.reduce(masked - best[:, None], axis=0)
        assert (op.nan_bits(rc.regret) == op.nan_bits(regret)).all()
        everywhere = usable.all(axis=0)
        order = [i for i in np.argsort(rc.regret, kind='stable').tolist() if everywhere[i]]
        for k in (0, 1, 5, n):
            pos, r = rc.robust(k)
            assert pos.tolist() == order[:k] and (_bits(r) == _bits(rc.regret[order[:k]])).all()
    tuples = rc.candidates.tuples(np.arange(n))
    for j in range(len(rc.costs)):
        want = sorted((i for i in range(n) if usable[j, i]), key=lambda i: rc.costs[j, i])
        got = rc.ranked(j)
        assert [t[:6] for t in got] == [tuples[i][:6] for i in want]
        assert _bits([t[6] for t in got]).tolist() == _bits(rc.costs[j, want]).tolist()
        b = rc.best(j)
        assert (b is None) == (not want)
        if want:
            assert b[:6] == tuples[want[0]][:6] and _bits(b[6]) == _bits(rc.costs[j, want[0]])


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['one_search', 'windows', 'device_listed'])
@pytest.mark.parametrize('name', IDENTITY + ['rough_q10:Q5Q6'])
def test_api_own_profile_is_the_search(name, mode, workload_dir, monkeypatch):
    """Through the api: under the searched profile (twice), costs and headroom are the search's (headroom=True) bit for
    bit with status 0; on the profile_* goldens, every scenario equals the reference bit for bit."""
    _gpu()
    from metis_b200 import api
    base, _, fix = name.partition(':')
    corrected = ('Q5', 'Q6') if fix else ()
    spec = Spec(base, workload_dir)
    api.release_engines()
    res = _headroom_run(spec, corrected, mode, monkeypatch)
    if mode == 'windows':
        assert res.summary['num_windows'] > 1
    profile = base_profile(spec)
    rc = res.recost_profiles([profile, profile])
    assert rc.costs.shape == (2, len(res)) and (rc.status == 0).all()
    assert (_bits(rc.costs) == _bits(np.stack([res.costs] * 2))).all()
    assert (_bits(rc.headroom) == _bits(np.stack([res.headroom] * 2))).all()
    if base in GOLDENS and not corrected:
        gold, profiles = golden_scenarios(spec)
        rc = res.recost_profiles(profiles)
        pos = [res.candidates.index_of(o, s) for o, s in zip(spec.arr['ordinal'].tolist(), spec.arr['step'].tolist())]
        same((rc.costs[:, pos], rc.headroom[:, pos], rc.status[:, pos]), gold['costs'], gold['headroom'],
             gold['cost_exc'], gold['memory_exc'])
        _check_views(rc)
    api.release_engines()


def _headroom_run(spec, corrected=(), mode='one_search', monkeypatch=None):
    """test_recost._run with headroom=True."""
    from metis_b200 import api
    orig = api.cost_het_cluster

    def with_headroom(*a, **k):
        return orig(*a, headroom=True, **k)
    if monkeypatch is None:
        monkeypatch = pytest.MonkeyPatch()
    monkeypatch.setattr(api, 'cost_het_cluster', with_headroom)
    try:
        return _run(spec, spec.root, corrected, mode, monkeypatch)
    finally:
        monkeypatch.setattr(api, 'cost_het_cluster', orig)


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['one_search', 'windows'])
@pytest.mark.parametrize('name', ['c3_homo64_mpl6', 'c4_het128'])
def test_api_own_profile_whole_space(name, mode, workload_dir, monkeypatch):
    """The identity on every candidate of C3-mpl6 and C4-mpl4, and the views on a seeded scenario set."""
    _gpu()
    from metis_b200 import api
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = _headroom_run(spec, (), mode, monkeypatch)
    profile = base_profile(spec)
    rc = res.recost_profiles([profile])
    assert (rc.status == 0).all()
    assert (_bits(rc.costs[0]) == _bits(res.costs)).all()
    assert (_bits(rc.headroom[0]) == _bits(res.headroom)).all()
    if name == 'c3_homo64_mpl6':
        assert len(res) == 273688
    if mode == 'one_search':
        rc = res.recost_profiles(op.scenarios(profile, 3, spec.seqs))
        assert rc.costs.shape == (len(op.KINDS), len(res))
        assert (_bits(rc.costs[0]) == _bits(res.costs)).all()
    api.release_engines()


@pytest.mark.gpu
def test_api_equals_the_oracle_on_seeded_scenarios(workload_dir):
    """20 seeded scenario sets on rough_t3's candidates, each set in one call: the oracle bit for bit, statuses
    included, and the views against numpy."""
    _gpu()
    from metis_b200 import api
    spec = Spec('rough_t3', workload_dir)
    api.release_engines()
    res = _run(spec, spec.root)
    pos = [res.candidates.index_of(o, s) for o, s in zip(spec.arr['ordinal'].tolist(), spec.arr['step'].tolist())]
    base = base_profile(spec)
    for seed in range(200, 220):
        profiles = op.scenarios(base, seed, spec.seqs)
        rc = res.recost_profiles(profiles)
        same((rc.costs[:, pos], rc.headroom[:, pos], rc.status[:, pos]), *oracle_scenarios(spec, profiles))
        if seed % 5 == 0:
            _check_views(rc)
    api.release_engines()


@pytest.mark.gpu
def test_profile_recost_survives_list_and_a_later_search(workload_dir):
    """A what-if taken after list(result), and one taken after a later cost_het_cluster() call on other inputs, are
    unchanged."""
    _gpu()
    from metis_b200 import api
    spec = Spec('rough_t3', workload_dir)
    api.release_engines()
    first = _run(spec, spec.root)
    profiles = op.scenarios(base_profile(spec), SEED, spec.seqs)
    before = first.recost_profiles(profiles)
    assert len(list(first)) == len(first)
    after_list = first.recost_profiles(profiles)
    other = Spec('mix32', workload_dir)
    assert len(_run(other, other.root)) != len(first)
    after = first.recost_profiles(profiles)
    for got in (after_list, after):
        assert (op.nan_bits(got.costs) == op.nan_bits(before.costs)).all()
        assert (op.nan_bits(got.headroom) == op.nan_bits(before.headroom)).all()
        assert (got.status == before.status).all()
        assert (op.nan_bits(got.regret) == op.nan_bits(before.regret)).all()
        assert [t[:6] for t in got.ranked(2)] == [t[:6] for t in before.ranked(2)]
    api.release_engines()
