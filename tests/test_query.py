"""Plan queries of a finished search (metis_query_mark / metis_query_groups / metis_mask_select,
HetSearchResult.ranked(where=) / count / best_by): filters on the reference's candidates and the best candidate per
key.

The definitions are Python: search.PlanFilter.admits on one 7-tuple, search.query_key, and the first admitted
candidate per key of sorted(result, key=cost).  CPU: the host build of the filter / key function
(tests/hostsim/query_sim.cpp) equals them on every candidate of seven goldens under 60 seeded filters; the group-best
passes, visited in random orders, equal a numpy reference; the ValueError cases and the argument checks.  GPU (-m gpu):
ranked / count / best_by through the api against the Python definitions over list(result), as one search, in forced
windows and on a device-listed space, C3-mpl6 and C4-mpl4 included.
"""
import ctypes as C
import itertools
import os
import random
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import hostsim_util as hs
from metis_b200 import native, search
from metis_b200.search import PlanFilter
from test_recost import Spec, host_search

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'query_sim.cpp')
SIM_DEPS = [SIM_SRC, hs.SRC] + [os.path.join(HERE, '..', 'metis_b200', 'csrc', f)
                                for f in ('metis_eval.cuh', 'metis_coop.cuh', 'metis_trace.cuh', 'metis_rows.cuh',
                                          'metis_query.cuh')] + [os.path.join(HERE, '..', 'include', 'metis_b200.h')]
GOLDENS = ['c1', 'mix32', 'c2_het16', 'rough_t3', 'rough_q10', 'het32_tight', 'lim_s128_l255']
NUM_FILTERS = 60
KEY_SETS = [k for r in (1, 2) for k in itertools.combinations(search.QUERY_KEYS, r)]
_sim = []


def sim():
    """The g++ build of the queries (tests/hostsim/query_sim.cpp), hostsim.cpp's flags."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'libquery_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)                             # atomic: concurrent test processes may race
        _sim.append(C.CDLL(out))
    return _sim[0]


def placement(cluster, node_sequence):
    """The reference's rank_device_map (model/device_group.py:22-32) of ``node_sequence`` on ``cluster``."""
    types = []
    for t in node_sequence:
        name = search.flatten._type_name(t)
        types += [name] * cluster.get_num_nodes_by_device_type(name)
    return types[:cluster.get_total_num_devices()]


def filters(tuples, type_names, seqs, seed=0, n=NUM_FILTERS):
    """``n`` seeded filters drawn from the values the candidates have: every field alone first, then combinations."""
    rng = random.Random(seed)
    stages = sorted({len(t[1]) for t in tuples}) or [1]
    batches = sorted({t[3] for t in tuples}) or [1]
    tps = [1, 2, 4, 8]

    def field(name):
        if name == 'min_stages':
            return rng.choice(stages)
        if name == 'max_stages':
            return rng.choice(stages)
        if name == 'node_sequences':
            return rng.sample(seqs, rng.randint(1, len(seqs)))
        if name == 'batches':
            return rng.sample(batches, rng.randint(1, len(batches)))
        if name == 'max_tp':
            return rng.choice(tps)
        if name == 'max_tp_by_type':
            return {t: rng.choice(tps) for t in rng.sample(type_names, rng.randint(1, len(type_names)))}
        if name == 'uniform_tp':
            return True
        return rng.choice([1, 2, 3])
    names = ['min_stages', 'max_stages', 'node_sequences', 'batches', 'max_tp', 'max_tp_by_type', 'uniform_tp',
             'max_repartition']
    out = [PlanFilter()] + [PlanFilter(**{f: field(f)}) for f in names]
    while len(out) < n:
        kw = {f: field(f) for f in rng.sample(names, rng.randint(2, 5))}
        if 'min_stages' in kw and 'max_stages' in kw and kw['min_stages'] > kw['max_stages']:
            kw['min_stages'], kw['max_stages'] = kw['max_stages'], kw['min_stages']
        out.append(PlanFilter(**kw))
    return out


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def _host_case(name, workload_dir):
    spec = Spec(name, workload_dir)
    problem, space = spec.problem(spec.root)
    sample = set(spec.arr['ordinal'].tolist()) if name.startswith('lim_') else None
    rec, det = host_search(problem, space, sample)
    assert (_bits(rec['cost']) == _bits(spec.arr['cost'])).all()
    cand = search.Candidates(rec, det, space, spec.seqs, problem=problem)
    tuples = cand.tuples(np.arange(len(rec)))
    return spec, problem, space, rec, det, tuples


def _sim_mark(problem, space, flt, rec, det):
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sp = space.as_struct(lambda n: keep[n].ctypes.data)
    mask = np.full(len(rec), 7, dtype=np.uint8)
    group = np.zeros(len(rec), dtype=np.uint32)
    assert sim().query_sim_mark(C.byref(p), C.byref(sp), C.byref(flt), C.c_void_p(rec.ctypes.data),
                                C.c_int64(len(rec)), C.c_void_p(det.ctypes.data), C.c_int32(det.shape[1]),
                                C.c_void_p(mask.ctypes.data), C.c_void_p(group.ctypes.data)) == 0
    return mask, group


def _with_keys(flt, keys, ranges):
    flt.num_keys = len(keys)
    for j, k in enumerate(keys):
        flt.key_field[j] = search.QUERY_KEYS.index(k)
        flt.key_range[j] = ranges[k]
    return flt


def _ranges(problem, space, rec, seqs):
    return {'node_sequence': len(seqs), 'num_stage': int(rec['num_stage'].max()), 'batches': len(space.batches),
            'max_tp': int(problem.scalars['num_tp']), 'num_repartition': 3}


def _decode(keys, ranges, gid, seqs, batches):
    out = []
    for k in reversed(keys):
        d = gid % ranges[k]
        gid //= ranges[k]
        out.append({'node_sequence': lambda: seqs[d], 'num_stage': lambda: d + 1,
                    'batches': lambda: int(batches[len(batches) - 1 - d]), 'max_tp': lambda: 1 << d,
                    'num_repartition': lambda: d + 1}[k]())
    return tuple(out[::-1])


@pytest.mark.parametrize('name', GOLDENS)
def test_host_filter_and_keys_are_the_definition(name, workload_dir):
    """CPU item 1: on every candidate, the host build's mask is PlanFilter.admits under 60 seeded filters (every field
    alone and in combination; the placement from the reference's formula on the cluster), and its group, with all five
    key fields, decodes to search.query_key."""
    spec, problem, space, rec, det, tuples = _host_case(name, workload_dir)
    cluster = spec.cluster(spec.root)
    place = {s: placement(cluster, s) for s in spec.seqs}
    for i, s in enumerate(spec.seqs):
        assert search.rank_device_map(problem, i) == place[s]
    ranges = _ranges(problem, space, rec, spec.seqs)
    keys = search.QUERY_KEYS
    for flt in filters(tuples, problem.type_names, spec.seqs, seed=len(name)):
        st = _with_keys(flt.to_struct(problem.type_names, spec.seqs, space.batches), keys, ranges)
        mask, group = _sim_mark(problem, space, st, rec, det)
        want = np.array([flt.admits(t, place[t[0]]) for t in tuples], dtype=np.uint8)
        assert (mask == want).all(), (flt, np.nonzero(mask != want)[0][:5])
        assert (group[mask == 0] == native.QUERY_NO_GROUP).all()
        for i in np.nonzero(mask)[0][:: max(1, int(mask.sum()) // 500)].tolist():
            assert _decode(keys, ranges, int(group[i]), spec.seqs, space.batches) == search.query_key(tuples[i], keys)
    # the admitted sets of the fields alone are neither all nor nothing somewhere: the filters select
    counts = [int(_sim_mark(problem, space, f.to_struct(problem.type_names, spec.seqs, space.batches), rec, det)[0].sum())
              for f in filters(tuples, problem.type_names, spec.seqs, seed=len(name))[1:9]]
    assert any(0 < c < len(rec) for c in counts) or len(rec) < 2, counts


def test_host_filter_bounds_outside_int32(workload_dir):
    """Stage and repartition bounds that do not fit the struct's int32 fields keep their meaning: the host build's mask
    is still PlanFilter.admits."""
    spec, problem, space, rec, det, tuples = _host_case('mix32', workload_dir)
    for flt in (PlanFilter(min_stages=2 ** 32), PlanFilter(min_stages=-2 ** 35), PlanFilter(max_stages=-2 ** 32 + 5),
                PlanFilter(max_stages=2 ** 40), PlanFilter(max_repartition=-2 ** 40),
                PlanFilter(max_repartition=2 ** 33 + 1), PlanFilter(min_stages=-2 ** 33, max_stages=2 ** 33 + 2)):
        mask, _group = _sim_mark(problem, space, flt.to_struct(problem.type_names, spec.seqs, space.batches), rec, det)
        want = np.array([flt.admits(t) for t in tuples], dtype=np.uint8)
        assert (mask == want).all(), flt


def _numpy_group_best(cost, group, num_groups):
    at = np.nonzero(group != native.QUERY_NO_GROUP)[0]
    g = group[at].astype(np.int64)
    order = np.lexsort((at, cost[at], g))                     # by group, then cost (-0.0 == 0.0), then position
    count = np.bincount(g, minlength=num_groups)
    first = np.full(num_groups, -1, dtype=np.int64)
    best = np.full(num_groups, np.inf)
    head = order[np.r_[True, g[order][1:] != g[order][:-1]]] if len(order) else order
    first[g[head]] = at[head]
    best[g[head]] = cost[at[head]]
    return count, best, first


@pytest.mark.parametrize('name', GOLDENS)
def test_host_group_best_is_numpy(name, workload_dir):
    """CPU item 1: the group-best passes (visited in three random orders) equal a numpy reference for every key subset
    of size 1 and 2 under a few filters, including ties (equal costs, -0.0 against +0.0)."""
    spec, problem, space, rec, det, tuples = _host_case(name, workload_dir)
    ranges = _ranges(problem, space, rec, spec.seqs)
    rng = np.random.default_rng(7)
    rec2 = rec.copy()
    if len(rec2) > 3:                                         # ties: repeat some costs, and a signed zero pair
        rec2['cost'][1::3] = rec2['cost'][0:len(rec2) - 1:3][:len(rec2['cost'][1::3])]
        rec2['cost'][-1], rec2['cost'][-2] = 0.0, -0.0
    for flt in filters(tuples, problem.type_names, spec.seqs, seed=3, n=4):
        for keys in KEY_SETS:
            st = _with_keys(flt.to_struct(problem.type_names, spec.seqs, space.batches), keys, ranges)
            _mask, group = _sim_mark(problem, space, st, rec, det)
            G = int(np.prod([ranges[k] for k in keys]))
            want = _numpy_group_best(rec2['cost'], group, G)
            for _ in range(3):
                visit = rng.permutation(len(rec2)).astype(np.int64)
                count = np.zeros(G, dtype=np.uint64)
                cost = np.zeros(G)
                first = np.zeros(G, dtype=np.int64)
                assert sim().query_sim_groups(C.c_void_p(rec2.ctypes.data), C.c_void_p(group.ctypes.data),
                                              C.c_int64(len(rec2)), C.c_void_p(visit.ctypes.data), C.c_int64(G),
                                              C.c_void_p(count.ctypes.data), C.c_void_p(cost.ctypes.data),
                                              C.c_void_p(first.ctypes.data)) == 0
                assert count.astype(np.int64).tolist() == want[0].tolist()
                assert first.tolist() == want[2].tolist()
                has = want[2] >= 0                            # the passes return -0.0 as +0.0: compare as numbers
                assert (cost[has] == want[1][has]).all() and np.isinf(cost[~has]).all()


def test_filter_validation():
    """CPU item 1: invalid fields raise a ValueError naming the field."""
    types = ['A100', 'V100']
    seqs = [('A100', 'V100'), ('V100', 'A100')]
    batches = np.array([8, 4, 2, 1], dtype=np.int32)
    bad = [(PlanFilter(max_tp_by_type={'H100': 2}), 'max_tp_by_type'),
           (PlanFilter(max_tp_by_type={'V100': 3}), 'max_tp_by_type'),
           (PlanFilter(max_tp_by_type={'V100': 0}), 'max_tp_by_type'),
           (PlanFilter(node_sequences=[('A100',)]), 'node_sequences'),
           (PlanFilter(node_sequences=[('A100', 'H100')]), 'node_sequences'),
           (PlanFilter(node_sequences=['A100V100']), 'node_sequences'),
           (PlanFilter(max_tp=0), 'max_tp'), (PlanFilter(max_tp=-2), 'max_tp'), (PlanFilter(max_tp=6), 'max_tp'),
           (PlanFilter(max_tp=2.0), 'max_tp'), (PlanFilter(max_tp=True), 'max_tp'),
           (PlanFilter(min_stages=5, max_stages=4), 'min_stages'),
           (PlanFilter(min_stages='2'), 'min_stages'), (PlanFilter(max_repartition=1.5), 'max_repartition'),
           (PlanFilter(batches=[2.5]), 'batches')]
    for flt, field in bad:
        with pytest.raises(ValueError, match=field):
            flt.to_struct(types, seqs, batches)
    ok = PlanFilter(min_stages=2, max_stages=2, node_sequences=[['V100', 'A100']], batches=[4], max_tp=4,
                    max_tp_by_type={'V100': 2}, uniform_tp=True, max_repartition=1).to_struct(types, seqs, batches)
    assert ok.ns_mask[0] == 2 and ok.div_mask[0] == 2 and ok.max_tp_code == 2 and ok.type_tp_code[1] == 1
    assert ok.type_tp_code[0] == 255 and ok.flags == native.QUERY_NEEDS_TP | native.QUERY_BY_TYPE
    assert PlanFilter(max_stages=3).to_struct(types, seqs, batches).flags == 0
    for keys, msg in ((('cost',), 'unknown key'), ((), 'at least one'), (('num_stage', 'num_stage'), 'repeats')):
        with pytest.raises(ValueError, match=msg):
            search.check_keys(keys)
    assert search.check_keys('batches') == ('batches',)


def test_best_by_refuses_too_many_groups():
    """CPU item 1: best_by refuses more than 2^24 groups with a ValueError, before touching the device."""
    from metis_b200 import api
    rec = np.zeros(2, dtype=native.RECORD_DTYPE)
    rec['num_stage'] = 128
    space = SimpleNamespace(batches=np.arange(256, 0, -1, dtype=np.int32))
    cand = SimpleNamespace(node_sequences=[('A',)] * 256, records=rec, cost=rec['cost'], segments=[SimpleNamespace(space=space)],
                           problem=SimpleNamespace(type_names=['A'], scalars={'num_tp': 8}))
    res = api.HetSearchResult(cand, None, {})
    with pytest.raises(ValueError, match='2\\^24'):
        res.best_by(('node_sequence', 'num_stage', 'batches', 'max_tp'))
    with pytest.raises(TypeError, match='PlanFilter'):
        res.count(where={'max_tp': 2})


def test_query_argument_checks():
    """metis_query_mark, metis_query_groups and metis_mask_select refuse bad arguments with METIS_E_ARG before touching
    the device."""
    lib = native.load_library()
    buf = np.zeros(4096, dtype=np.float64)
    ptr = C.c_void_p(buf.ctypes.data)
    p, sp = native.MetisProblem(), native.MetisPlanSpace()
    p.num_types, sp.max_stage, sp.num_div = 2, 4, 4
    E_ARG, E_CAPACITY = -2, -3

    def flt(**kw):
        f = native.MetisPlanFilter()
        for k, v in kw.items():
            if k in ('key_field', 'key_range'):
                for j, x in enumerate(v):
                    getattr(f, k)[j] = x
            else:
                setattr(f, k, v)
        return f

    def mark(f=None, n=1, rec=ptr, det=ptr, st=13, head=None, x=0.0, mask=ptr, group=ptr, prob=C.byref(p),
             space_=C.byref(sp)):
        return lib.metis_query_mark(prob, space_, C.byref(f) if f is not None else None, rec, C.c_int64(n), det,
                                    C.c_int32(st), head, C.c_double(x), mask, group, None)
    for kw in (dict(f=None), dict(f=flt(), prob=None), dict(f=flt(), space_=None), dict(f=flt(), rec=None),
               dict(f=flt(), mask=None), dict(f=flt(), n=-1), dict(f=flt(num_keys=6)),
               dict(f=flt(num_keys=1, key_field=[5], key_range=[2])), dict(f=flt(num_keys=1, key_field=[0], key_range=[0])),
               dict(f=flt(num_keys=2, key_field=[0, 1], key_range=[1 << 13, 1 << 12])),
               dict(f=flt(num_keys=1, key_field=[0], key_range=[2]), group=None),
               dict(f=flt(flags=1), det=None), dict(f=flt(num_keys=1, key_field=[3], key_range=[4]), det=None),
               dict(f=flt(flags=1), st=12), dict(f=flt(), head=ptr, x=float('nan'))):
        assert mark(**kw) == E_ARG, kw
    assert b'metis_query_mark' in lib.metis_last_error()

    def groups(n=1, G=4, rec=ptr, grp=ptr, cnt=ptr, cost=ptr, first=ptr, pres=ptr):
        return lib.metis_query_groups(rec, grp, C.c_int64(n), C.c_int64(G), cnt, cost, first, pres, None)
    for kw in (dict(n=-1), dict(G=0), dict(G=(1 << 24) + 1), dict(rec=None), dict(grp=None), dict(cnt=None),
               dict(cost=None), dict(first=None), dict(pres=None)):
        assert groups(**kw) == E_ARG, kw

    def select(n=1, k=1, mask=ptr, out=ptr, cnt=ptr, ws=ptr, wsb=1 << 20):
        return lib.metis_mask_select(mask, None, C.c_int64(n), C.c_int64(k), out, cnt, ws, C.c_int64(wsb), None)
    for kw in (dict(n=-1), dict(n=1 << 32), dict(mask=None), dict(cnt=None), dict(ws=None), dict(k=-1),
               dict(out=None)):
        assert select(**kw) == E_ARG, kw
    assert select(wsb=8) == E_CAPACITY


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()
    return torch


def _run(spec, mode='one_search', monkeypatch=None, headroom=False):
    """api.cost_het_cluster on the golden's inputs (test_recost._run, with headroom when asked)."""
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.utils import ModelConfig
    if mode == 'windows':
        from test_windowed_search import _force_windows
        _force_windows(monkeypatch, 3)
    elif mode == 'device_listed':
        monkeypatch.setattr(api, '_DEVICE_LISTING_COMPS', 0)
    cluster = spec.cluster(spec.root)
    profile, _ = ProfileDataLoader(os.path.join(spec.root, spec.sub), spec.meta['file_order']).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=spec.num_layers, sequence_length=spec.sequence_length,
                      vocab_size=spec.vocab_size, hidden_size=spec.hidden_size, attention_head_size=32)
    args = parse_args(['--num_layers', str(spec.num_layers), '--gbs', str(spec.gbs),
                       '--hidden_size', str(spec.hidden_size), '--sequence_length', str(spec.sequence_length),
                       '--vocab_size', str(spec.vocab_size), '--attention_head_size', '32',
                       '--max_profiled_tp_degree', str(spec.max_tp), '--max_profiled_batch_size', str(spec.max_bs),
                       '--min_group_scale_variance', str(spec.variance), '--max_permute_len', str(spec.max_permute_len)])
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=spec.seqs,
                                device='cuda:0', headroom=headroom)


class Truth:
    """The Python definitions over list(result)."""

    def __init__(self, res, spec):
        self.tuples = list(res)
        self.ranked = sorted(range(len(self.tuples)), key=lambda i: self.tuples[i][6])     # stable, like the reference
        cluster = spec.cluster(spec.root)
        self.place = {s: placement(cluster, s) for s in spec.seqs}
        self.headroom = res.headroom

    def admitted(self, flt, min_headroom=None):
        return [i for i in self.ranked if flt.admits(self.tuples[i], self.place[self.tuples[i][0]])
                and (min_headroom is None or self.headroom[i] >= min_headroom)]

    def best_by(self, keys, adm):
        out = {}
        for i in adm:
            key = search.query_key(self.tuples[i], keys)
            if key not in out:
                out[key] = [i, 0]
            out[key][1] += 1
        order = sorted(out, key=lambda v: tuple(search._names(x) if k == 'node_sequence' else x for k, x in zip(keys, v)))
        return order, [out[v][1] for v in order], [out[v][0] for v in order]


def _same(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a[:6] == b[:6] and _bits(a[6]) == _bits(b[6]), (a, b)


def _check(res, truth, flt, key_sets, k=(None, 1, 7), min_headroom=None):
    adm = truth.admitted(flt, min_headroom)
    for kk in k:
        _same(res.ranked(kk, min_headroom=min_headroom, where=flt), [truth.tuples[i] for i in adm[:kk]])
    assert res.count(flt, min_headroom) == len(adm)
    for keys in key_sets:
        g = res.best_by(keys, where=flt, min_headroom=min_headroom)
        values, counts, first = truth.best_by(keys, adm)
        assert g.values == values and g.count.tolist() == counts and g.position.tolist() == first, (flt, keys)
        assert (_bits(g.cost) == _bits(res.costs[first])).all()
        _same(g.tuples(), [truth.tuples[i] for i in first])


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['one_search', 'windows', 'device_listed'])
@pytest.mark.parametrize('name', GOLDENS)
def test_api_queries_are_the_definition(name, mode, workload_dir, monkeypatch):
    """GPU item 2 on the goldens: ranked(k, where=), count and best_by (every key subset of size 1 and 2) equal the
    Python definitions over list(result) for 60 seeded filters, tuple for tuple, costs bit for bit; ranked(k,
    where=PlanFilter()) is ranked(k)."""
    _gpu()
    from metis_b200 import api
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = _run(spec, mode, monkeypatch)
    if mode == 'windows':
        assert res.summary['num_windows'] > 1
    truth = Truth(res, spec)
    # lim_s128_l255's 128-stage plans make the Python side slow: a quarter of the filters there
    flts = filters(truth.tuples, res.candidates.problem.type_names, spec.seqs, seed=len(name),
                   n=NUM_FILTERS // 4 if name.startswith('lim_') else NUM_FILTERS)
    for j, flt in enumerate(flts):
        _check(res, truth, flt, KEY_SETS if j % 4 == 0 else KEY_SETS[j % len(KEY_SETS)::7])
    for kk in (None, 0, 3, -2):
        _same(res.ranked(kk, where=PlanFilter()), res.ranked(kk))
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name,mode', [('c3_homo64_mpl6', 'one_search'), ('c4_het128', 'windows'),
                                       ('c4_het128', 'device_listed')])
def test_api_queries_whole_space(name, mode, workload_dir, monkeypatch):
    """GPU item 2 on all of C3-mpl6 as one search (with one min_headroom query) and on C4-mpl4 in forced windows and
    as a device-listed space."""
    _gpu()
    from metis_b200 import api
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = _run(spec, mode, monkeypatch, headroom=name.startswith('c3'))
    truth = Truth(res, spec)
    if name.startswith('c3'):
        assert len(res) == 273688
    types = res.candidates.problem.type_names
    flts = [PlanFilter(max_stages=8), PlanFilter(max_tp=2, max_repartition=1),
            PlanFilter(max_tp_by_type={types[0]: 2}, uniform_tp=True, min_stages=2),
            filters(truth.tuples, types, spec.seqs, seed=11, n=12)[-1]]
    for flt in flts:
        _check(res, truth, flt, [('num_stage',), ('node_sequence', 'max_tp')], k=(100,))
    if name.startswith('c3'):
        x = float(np.quantile(res.headroom, 0.6))
        _check(res, truth, PlanFilter(max_tp=4), [('num_stage',)], k=(100,), min_headroom=x)
    api.release_engines()


@pytest.mark.gpu
def test_windowed_strategy_filter_is_the_one_search(workload_dir, monkeypatch):
    """GPU item 2: a strategy filter on a windowed result gives the one-search result's answer on the same space."""
    _gpu()
    from metis_b200 import api
    spec = Spec('c4_het128', workload_dir)
    flt = PlanFilter(max_tp_by_type={spec.seqs[0][0]: 2}, uniform_tp=True)
    api.release_engines()
    one = _run(spec)
    a = (one.ranked(100, where=flt), one.count(flt), one.best_by(('node_sequence', 'max_tp'), where=flt))
    api.release_engines()
    win = _run(spec, 'windows', monkeypatch)
    assert win.summary['num_windows'] > 1
    b = (win.ranked(100, where=flt), win.count(flt), win.best_by(('node_sequence', 'max_tp'), where=flt))
    _same(b[0], a[0])
    assert b[1] == a[1] and b[2].values == a[2].values and b[2].position.tolist() == a[2].position.tolist()
    assert b[2].count.tolist() == a[2].count.tolist()
    api.release_engines()


@pytest.mark.gpu
def test_query_survives_a_later_search(workload_dir):
    """GPU item 2: a query taken after a later cost_het_cluster() call on other inputs is unchanged."""
    _gpu()
    from metis_b200 import api
    spec = Spec('rough_t3', workload_dir)
    api.release_engines()
    first = _run(spec)
    flt = PlanFilter(max_tp=2, max_stages=3)
    before = (first.ranked(20, where=flt), first.count(flt), first.best_by(('num_stage', 'max_tp'), where=flt))
    other = Spec('mix32', workload_dir)
    assert len(_run(other)) != len(first)
    after = (first.ranked(20, where=flt), first.count(flt), first.best_by(('num_stage', 'max_tp'), where=flt))
    _same(after[0], before[0])
    assert after[1] == before[1] and after[2].values == before[2].values
    assert after[2].position.tolist() == before[2].position.tolist()
    api.release_engines()


@pytest.mark.gpu
def test_windowed_geometry_query_behind_a_busy_stream(workload_dir, monkeypatch):
    """A geometry-only query on a windowed result reloads each window's tables into the pinned staging arena and
    uploads them asynchronously, with nothing in between that waits for the device.  With the stream held up by a long
    kernel queued first, every window's kernel must still read that window's tables: the answers equal the
    definitions."""
    torch = _gpu()
    from metis_b200 import api
    spec = Spec('c2_het16', workload_dir)
    api.release_engines()
    res = _run(spec, 'windows', monkeypatch)
    assert res.summary['num_windows'] > 1
    truth = Truth(res, spec)
    flt = PlanFilter(max_stages=4, max_repartition=2)
    assert not flt.reads_strategies
    adm = truth.admitted(flt)
    values, counts, first = truth.best_by(('num_stage', 'batches'), adm)
    for _ in range(3):
        torch.cuda._sleep(200_000_000)                       # about 0.1 s of work ahead of the uploads
        assert res.count(flt) == len(adm)
        torch.cuda._sleep(200_000_000)
        g = res.best_by(('num_stage', 'batches'), where=flt)
        assert g.values == values and g.count.tolist() == counts and g.position.tolist() == first
        torch.cuda._sleep(200_000_000)
        _same(res.ranked(25, where=flt), [truth.tuples[i] for i in adm[:25]])
    api.release_engines()
