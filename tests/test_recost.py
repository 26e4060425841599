"""Network what-if of a finished search (metis_het_recost / metis_recost_regret, HetSearchResult.recost): every
candidate re-costed under other bandwidths, without a new search.

Bandwidth enters only the cost model, so a search under a cluster that differs only in bandwidth returns the same
candidates.  CPU: that invariance on the pinned oracle; the host build of the recost (tests/hostsim/recost_sim.cpp)
against the goldens under the search's own bandwidths and against the oracle under other ones (per type, per node
within a type, and the between-node bandwidth of a 'Q2' run); the bw_* goldens of the unmodified reference; the
argument checks and the validation of the scenarios.  GPU (-m gpu): the same identities through the api, as one search,
in forced windows and on a device-listed space; recost against a fresh search under each scenario; regret against
numpy; a recost taken after a later search.
"""
import ctypes as C
import json
import os
import random
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
from conftest import C1_DIR, golden_rows, load_golden
from metis_b200 import flatten, native
from oracle import metis_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'recost_sim.cpp')
SIM_DEPS = [SIM_SRC, hs.SRC] + [os.path.join(HERE, '..', 'metis_b200', 'csrc', f)
                                for f in ('metis_eval.cuh', 'metis_coop.cuh', 'metis_trace.cuh', 'metis_rows.cuh',
                                          'metis_recost.cuh')] + [os.path.join(HERE, '..', 'include', 'metis_b200.h')]
INVARIANCE = ['c1', 'mix32', 'c2_het16', 'rough_mix2', 'rough_t3', 'rough_q10', 'het32_tight']
SAMPLED = {'het32_tight': 150}         # the oracle walks these goldens' plans in minutes: a spread of them, and the
                                       # plans of retried candidates
IDENTITY = INVARIANCE + ['lim_s128_l255', 'lim_s128_t2']
VARIANTS = ['per_type', 'per_node', 'q2']
C1 = dict(num_layers=10, hidden_size=4096, sequence_length=1024, vocab_size=51200, gbs=128, variance=1,
          max_permute_len=4, max_tp=4, max_bs=4)
_sim = []


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def sim():
    """The g++ build of the recost (tests/hostsim/recost_sim.cpp) at the compiled limits, hostsim.cpp's flags."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'librecost_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)                             # atomic: concurrent test processes may race
        lib = C.CDLL(out)
        lib.recost_sim_het.restype = C.c_int
        _sim.append(lib)
    return _sim[0]


# ---- inputs ---------------------------------------------------------------------------------------------------------
class Spec:
    """A golden's search: where its files are and its model / search flags."""

    def __init__(self, name, workload_dir):
        if name == 'c1':
            self.meta, self.arr = load_golden('c1_het')
            self.root, self.sub = C1_DIR, 'profile_data_samples'
            for k, v in C1.items():
                setattr(self, k, v)
        else:
            self.meta, self.arr = load_golden(name)
            w, self.root, digest = workload_dir(name)
            assert digest == self.meta['inputs_sha256']
            self.sub = 'profile'
            for k in C1:
                setattr(self, k, getattr(w, k))
        self.seqs = [tuple(s) for s in self.meta['node_sequences']]

    def oracle(self, root, corrected=(), sample=None):
        """oracle.het_search under the cluster files in ``root`` (only the plans of ``sample`` when given):
        {(ordinal, step): (strategies, partition, nrep, cost)} in estimate_costs order."""
        cl = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'),
                               corrected=corrected)
        prof, _ = orc.load_profile_dir(os.path.join(self.root, self.sub), self.meta['file_order'])
        model = orc.OracleModel(self.num_layers, self.hidden_size, self.sequence_length, self.vocab_size,
                                prof['model']['parameters'])
        cands, _ = orc.het_search(prof, cl, model, self.seqs, self.gbs, self.num_layers, self.variance,
                                  self.max_permute_len, self.max_tp, self.max_bs, corrected=corrected,
                                  plan_filter=sample.__contains__ if sample is not None else None)
        return {(c[0], c[1]): (c[4], c[6], c[7], c[8]) for c in cands}

    def cluster(self, root):
        from metis_b200.gpu_cluster import GPUCluster
        return GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))

    def problem(self, root, corrected=()):
        cluster, profile, _types, cfg = hs.load_inputs(self.root, self.sub, self.meta['file_order'], self.num_layers,
                                                       self.hidden_size, self.sequence_length, self.vocab_size)
        cluster = self.cluster(root)
        problem = flatten.build_problem(profile, cluster, cfg, self.gbs, self.max_tp, self.max_bs, self.seqs,
                                        corrected=corrected)
        space = flatten.build_plan_space(len(self.seqs), cluster.get_total_num_devices(), self.gbs, self.num_layers,
                                         self.variance, self.max_permute_len, corrected=corrected)
        return problem, space


def _hosts(root):
    """(ip, GPU count) of every hostfile line."""
    cl = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    return list(zip(cl.node_ip, cl.node_ndev)), cl.info


def _write(dst, hosts, info):
    os.makedirs(dst, exist_ok=True)
    with open(os.path.join(dst, 'hostfile'), 'w') as fh:
        fh.write(''.join(f'{ip} slots={n}\n' for ip, n in hosts))   # utils.py:15 reads the 7th character
    with open(os.path.join(dst, 'clusterfile.json'), 'w') as fh:
        json.dump(info, fh, indent=2)
    return dst


def variant(root, kind, tmp, seed=0):
    """(base cluster dir, variant cluster dir, corrected) of one kind of bandwidth change; the base is the searched
    cluster (for 'per_node': the same nodes, each under an IP of its own, so that a clusterfile entry is a node)."""
    hosts, info = _hosts(root)
    rng = random.Random(seed)
    if kind == 'per_type':
        var = {ip: dict(v, intra_bandwidth=v['intra_bandwidth'] * rng.choice([0.125, 0.5, 3.0, 16.0]))
               for ip, v in info.items()}
        return root, _write(os.path.join(tmp, 'var'), hosts, var), ()
    if kind == 'per_node':
        split = [(f'N{k}', n) for k, (_ip, n) in enumerate(hosts)]
        base = {f'N{k}': dict(info[ip]) for k, (ip, _n) in enumerate(hosts)}
        var = {ip: dict(v, intra_bandwidth=v['intra_bandwidth'] * rng.choice([0.0625, 0.25, 1.0, 2.0, 8.0]))
               for ip, v in base.items()}
        return _write(os.path.join(tmp, 'base'), split, base), _write(os.path.join(tmp, 'var'), split, var), ()
    var = {ip: dict(v, inter_bandwidth=v['inter_bandwidth'] * rng.choice([0.1, 0.5, 4.0, 40.0]))
           for ip, v in info.items()}
    return root, _write(os.path.join(tmp, 'var'), hosts, var), ('Q2',)


def host_search(problem, space, ordinals=None):
    """The host build's candidates in estimate_costs order (those of the plans ``ordinals`` when given): (records,
    detail rows)."""
    rec, det, _summary = hs.host_het_search(problem, space, mode=0, want_detail=True)
    order = np.lexsort((rec['step'], rec['ordinal']))
    if ordinals is not None:
        order = order[np.isin(rec['ordinal'][order], list(ordinals))]
    return np.ascontiguousarray(rec[order]), np.ascontiguousarray(det[order])


def sample_ordinals(arr, n):
    """Evenly spaced golden ordinals and those of retried candidates."""
    o = arr['ordinal']
    pick = set(o[np.linspace(0, len(o) - 1, min(n, len(o))).astype(np.int64)].tolist())
    for nrep in (2, 3):
        pick |= set(o[arr['nrep'] == nrep][:20].tolist())
    return pick


def bandwidths(clusters, type_names, corrected=()):
    """[K, 2, num_types] scenario tables (flatten.cluster_bandwidths), what HetSearchResult.recost passes down."""
    return np.array([flatten.cluster_bandwidths(c, type_names, corrected) for c in clusters], dtype=np.float64)


def host_recost(problem, space, rec, det, bw):
    """recost_sim_het: costs [K, n]."""
    lib = sim()
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sp = space.as_struct(lambda n: keep[n].ctypes.data)
    bw = np.ascontiguousarray(bw, dtype=np.float64)
    out = np.full((len(bw), len(rec)), -1.0)
    assert lib.recost_sim_het(C.byref(p), C.byref(sp), C.c_void_p(rec.ctypes.data), C.c_int64(len(rec)),
                              C.c_void_p(det.ctypes.data), C.c_int32(det.shape[1]), C.c_void_p(bw.ctypes.data),
                              C.c_int32(len(bw)), C.c_void_p(out.ctypes.data)) == 0
    return out


def _keys(want):
    return [(k, v[0], v[1], v[2]) for k, v in want.items()]


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', INVARIANCE)
def test_bandwidth_changes_only_the_costs(name, workload_dir, tmp_path):
    """Items 1 and 3: under a bandwidth variant (per type, per node within a type, between nodes with 'Q2') the oracle
    visits the same candidates with the same strategies, partitions and num_repartition; the host recost of the
    base search's candidates under the variant's tables is the oracle's cost bit for bit, and under the base's own
    tables the base's cost."""
    spec = Spec(name, workload_dir)
    sample = sample_ordinals(spec.arr, SAMPLED[name]) if name in SAMPLED else None
    original = _keys(spec.oracle(spec.root, sample=sample))
    for k, kind in enumerate(VARIANTS):
        base, var, corrected = variant(spec.root, kind, str(tmp_path / kind), seed=k)
        want_base, want_var = spec.oracle(base, corrected, sample), spec.oracle(var, corrected, sample)
        assert _keys(want_base) == _keys(want_var), kind
        if not corrected:
            assert _keys(want_base) == original, kind
        problem, space = spec.problem(base, corrected)
        rec, det = host_search(problem, space, sample)
        assert list(zip(rec['ordinal'].tolist(), rec['step'].tolist())) == list(want_base)
        bw = bandwidths([spec.cluster(base), spec.cluster(var)], problem.type_names, corrected)
        got = host_recost(problem, space, rec, det, bw)
        assert (_bits(got[0]) == _bits([v[3] for v in want_base.values()])).all(), kind
        assert (_bits(got[1]) == _bits([v[3] for v in want_var.values()])).all(), kind
        if len(rec) > 1:
            assert (got[0] != got[1]).any(), f'{kind}: the variant changes no cost'


@pytest.mark.parametrize('name', IDENTITY + ['rough_q10:Q5Q6'])
def test_host_recost_under_own_bandwidths_is_the_search(name, workload_dir):
    """Item 2: the general bandwidth path under the search's own tables gives every candidate's cost bit for bit
    (the search takes the derived tables of a uniform cluster), also for a ('Q5', 'Q6') corrected run."""
    base, _, fix = name.partition(':')
    corrected = ('Q5', 'Q6') if fix else ()
    spec = Spec(base, workload_dir)
    problem, space = spec.problem(spec.root, corrected)
    # the limit goldens hold a sample of their space's plans
    rec, det = host_search(problem, space, None if corrected else set(spec.arr['ordinal'].tolist()))
    if not corrected:
        assert (_bits(rec['cost']) == _bits(spec.arr['cost'])).all()
    bw = np.array([[problem.arrays['type_bw_first'], problem.arrays['type_bw_min']]])
    got = host_recost(problem, space, rec, det, np.concatenate([bw, bw]))
    assert (_bits(got) == _bits(np.stack([rec['cost'], rec['cost']]))).all()


@pytest.mark.parametrize('name', ['bw_mix32', 'bw_rough_t3'])
def test_bandwidth_goldens(name, workload_dir):
    """Item 4: the oracle equals the bw_* goldens of the unmodified reference (bandwidths that differ by type), and the
    host recost of the base golden's candidates under the bw_* cluster gives the bw_* costs bit for bit."""
    spec = Spec(name, workload_dir)
    want = spec.oracle(spec.root)
    gold = golden_rows(spec.arr)
    assert [(g[0], g[1], g[4], g[6], g[7]) for g in gold] == [(k[0], k[1], *v[:3]) for k, v in want.items()]
    assert _bits([g[8] for g in gold]).tolist() == _bits([v[3] for v in want.values()]).tolist()
    base = Spec(name[len('bw_'):], workload_dir)
    problem, space = base.problem(base.root)
    rec, det = host_search(problem, space)
    assert list(zip(rec['ordinal'].tolist(), rec['step'].tolist())) == [(g[0], g[1]) for g in gold]
    got = host_recost(problem, space, rec, det, bandwidths([spec.cluster(spec.root)], problem.type_names))
    assert (_bits(got[0]) == _bits(spec.arr['cost'])).all()
    assert (got[0] != rec['cost']).any()


@pytest.mark.parametrize('name', ['bw_mix32', 'bw_rough_t3'])
def test_bandwidth_workloads_differ_only_in_bandwidth(name, tmp_path):
    """The bw_* workloads' hostfile and profile files are byte-identical to their base's; the clusterfiles differ only
    in intra_bandwidth."""
    from metis_b200.workloads import WORKLOADS, materialize
    a, b = str(tmp_path / 'bw'), str(tmp_path / 'base')
    materialize(WORKLOADS[name], a)
    materialize(WORKLOADS[name[len('bw_'):]], b)
    assert open(os.path.join(a, 'hostfile'), 'rb').read() == open(os.path.join(b, 'hostfile'), 'rb').read()
    files = sorted(os.listdir(os.path.join(b, 'profile')))
    assert files == sorted(os.listdir(os.path.join(a, 'profile'))) and files
    for f in files:
        assert open(os.path.join(a, 'profile', f), 'rb').read() == open(os.path.join(b, 'profile', f), 'rb').read()
    ca, cb = (json.load(open(os.path.join(d, 'clusterfile.json'))) for d in (a, b))
    assert ca.keys() == cb.keys()
    assert any(ca[ip]['intra_bandwidth'] != cb[ip]['intra_bandwidth'] for ip in ca)
    for ip in ca:
        assert {k: v for k, v in ca[ip].items() if k != 'intra_bandwidth'} == \
            {k: v for k, v in cb[ip].items() if k != 'intra_bandwidth'}


@pytest.mark.parametrize('name', ['mix32', 'rough_t3', 'rough_q10', 'c1'])
def test_cluster_bandwidths_are_build_problems(name, workload_dir, tmp_path):
    """flatten.cluster_bandwidths is what build_problem puts in MetisProblem, with and without 'Q2'."""
    spec = Spec(name, workload_dir)
    _base, var, _ = variant(spec.root, 'q2', str(tmp_path))
    for corrected in ((), ('Q2',)):
        problem, _space = spec.problem(var, corrected)
        first, low = flatten.cluster_bandwidths(spec.cluster(var), problem.type_names, corrected)
        assert _bits(first).tolist() == _bits(problem.arrays['type_bw_first']).tolist()
        assert _bits(low).tolist() == _bits(problem.arrays['type_bw_min']).tolist()
    assert problem.scalars['uniform_bw'] == 0


class _FakeCandidates:
    def __init__(self, problem):
        self.problem = problem

    def recost(self, bw):
        return bw


def _fake_result(spec, root, corrected=()):
    from metis_b200 import api
    problem, _space = spec.problem(root, corrected)
    res = api.HetSearchResult(_FakeCandidates(problem), None, {'corrected': tuple(corrected)})
    res._searched = api.cluster_signature(spec.cluster(root), problem.type_names)
    return res


def _edit(root, dst, hosts=None, **change):
    """A copy of the cluster in ``root`` with ``change`` = {field: {ip: value}} and optionally other hosts."""
    h, info = _hosts(root)
    info = {ip: dict(v) for ip, v in info.items()}
    for field, by_ip in change.items():
        for ip, v in by_ip.items():
            info[ip][field] = v
    return _write(dst, hosts if hosts is not None else h, info)


def test_recost_validates_the_scenarios(workload_dir, tmp_path):
    """Item 5: a scenario that differs in anything but bandwidth, or whose bandwidth is not a finite number > 0, is
    refused with a ValueError naming the node and the field; 'Q2' runs check inter_bandwidth too."""
    spec = Spec('mix32', workload_dir)
    res = _fake_result(spec, spec.root)
    hosts, info = _hosts(spec.root)
    ip0, ip1 = hosts[0][0], hosts[-1][0]
    cl = lambda d: spec.cluster(d)                                            # noqa: E731
    ok = res.recost([cl(_edit(spec.root, str(tmp_path / 'ok'), intra_bandwidth={ip0: 1e9}))])
    assert ok.shape == (1, 2, 2) and ok[0, 0, 0] == 1e9
    bad = [
        (dict(instance_type={ip0: 'V100'}), 'instance_type'),
        (dict(memory={ip1: 1}), 'memory'),
        (dict(intra_bandwidth={ip0: 0.0}), 'intra_bandwidth'),
        (dict(intra_bandwidth={ip1: -5e9}), 'intra_bandwidth'),
        (dict(intra_bandwidth={ip1: float('nan')}), 'intra_bandwidth'),
        (dict(intra_bandwidth={ip0: float('inf')}), 'intra_bandwidth'),
        (dict(intra_bandwidth={ip0: '5e9'}), 'intra_bandwidth'),
    ]
    for k, (change, field) in enumerate(bad):
        with pytest.raises(ValueError, match=field):
            res.recost([cl(_edit(spec.root, str(tmp_path / f'b{k}'), **change))])
    with pytest.raises(ValueError, match='GPU count'):
        res.recost([cl(_edit(spec.root, str(tmp_path / 'n'), hosts=[(hosts[0][0], 4)] + hosts[1:]))])
    with pytest.raises(ValueError, match='ip'):
        res.recost([cl(_edit(spec.root, str(tmp_path / 'o'), hosts=hosts[::-1]))])
    with pytest.raises(ValueError, match='hostfile entries'):
        res.recost([cl(_edit(spec.root, str(tmp_path / 'h'), hosts=hosts[:-1]))])
    with pytest.raises(ValueError, match='at least one'):
        res.recost([])
    # the second scenario is named
    with pytest.raises(ValueError, match='cluster 1, node 0'):
        res.recost([cl(spec.root), cl(_edit(spec.root, str(tmp_path / 's'), intra_bandwidth={ip0: 0}))])
    # inter_bandwidth is read only by a 'Q2' search
    odd = cl(_edit(spec.root, str(tmp_path / 'q'), inter_bandwidth={ip1: float('nan')}))
    res.recost([odd])
    with pytest.raises(ValueError, match='inter_bandwidth'):
        _fake_result(spec, spec.root, ('Q2',)).recost([odd])


def test_recost_argument_checks(workload_dir):
    """metis_het_recost and metis_recost_regret refuse bad arguments with METIS_E_ARG before touching the device."""
    lib = native.load_library()
    spec = Spec('mix32', workload_dir)
    problem, space = spec.problem(spec.root)
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sp = space.as_struct(lambda n: keep[n].ctypes.data)
    buf = np.zeros(4096, dtype=np.float64)
    ptr = C.c_void_p(buf.ctypes.data)
    stride = 3 * int(space.blocks['num_stage'].max()) + 1
    E_ARG, E_CAPACITY = -2, -3                                # METIS_E_ARG, METIS_E_CAPACITY

    def recost(n=1, det=ptr, rec=ptr, bw=ptr, cost=ptr, k=1, st=stride, ws=ptr, prob=C.byref(p), space_=C.byref(sp)):
        return lib.metis_het_recost(prob, space_, rec, C.c_int64(n), det, C.c_int32(st), bw, C.c_int32(k), cost, ws,
                                    C.c_int64(1 << 30), None)
    for kw in (dict(rec=None), dict(det=None), dict(bw=None), dict(cost=None), dict(ws=None), dict(n=-1), dict(k=0),
               dict(k=-3), dict(st=stride - 1), dict(prob=None), dict(space_=None)):
        assert recost(**kw) == E_ARG, kw
    assert b'metis_het_recost' in lib.metis_last_error()

    def regret(n=1, k=1, cost=ptr, best=ptr, reg=ptr, ws=ptr, wsb=1 << 20):
        return lib.metis_recost_regret(cost, C.c_int32(k), C.c_int64(n), best, reg, ws, C.c_int64(wsb), None)
    for kw in (dict(n=-1), dict(k=0), dict(k=65536), dict(cost=None), dict(best=None), dict(reg=None), dict(ws=None)):
        assert regret(**kw) == E_ARG, kw
    assert regret(wsb=8) == E_CAPACITY
    assert lib.metis_recost_regret_workspace_bytes(C.c_int32(0), C.c_int64(1)) == E_ARG
    assert lib.metis_recost_regret_workspace_bytes(C.c_int32(3), C.c_int64(2049)) == 256 + 3 * 2 * 8


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()
    return torch


def _run(spec, root, corrected=(), mode='one_search', monkeypatch=None):
    """api.cost_het_cluster on the golden's inputs under the cluster files in ``root``."""
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.utils import ModelConfig
    if mode == 'windows':
        from test_windowed_search import _force_windows
        _force_windows(monkeypatch, 3)
    elif mode == 'device_listed':
        monkeypatch.setattr(api, '_DEVICE_LISTING_COMPS', 0)
    cluster = spec.cluster(root)
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
                                device='cuda:0', corrected=corrected)


def _same_ranked(got, want):
    """Tuple for tuple, in order, costs bit for bit."""
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a[:6] == b[:6]
        assert _bits(a[6]) == _bits(b[6]), (a, b)


def _check_regret(rc):
    """regret / robust against numpy on the costs, ties included."""
    costs = rc.costs
    if costs.shape[1] == 0:
        assert len(rc.regret) == 0 and rc.robust(3)[0].size == 0
        return
    best = costs.min(axis=1)
    assert (_bits(rc.best_costs) == _bits(best)).all()
    regret = (costs - best[:, None]).max(axis=0)
    assert (_bits(rc.regret) == _bits(regret)).all()
    order = np.argsort(regret, kind='stable')
    for k in (0, 1, 5, len(regret)):
        pos, r = rc.robust(k)
        assert pos.tolist() == order[:k].tolist() and (_bits(r) == _bits(regret[order[:k]])).all()
    for j in range(len(costs)):
        assert rc.order(j).tolist() == np.argsort(costs[j], kind='stable').tolist()


GPU_IDENTITY = IDENTITY + ['bw_mix32', 'bw_rough_t3']


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['one_search', 'windows', 'device_listed'])
@pytest.mark.parametrize('name', GPU_IDENTITY + ['rough_q10:Q5Q6'])
def test_api_recost_under_own_cluster_is_the_search(name, mode, workload_dir, monkeypatch):
    """GPU item 1 (and 3 for the bw_* goldens): recost([own cluster]).costs[0] == result.costs bit for bit, as one
    search, in forced windows and on a device-listed space; the result equals the golden."""
    _gpu()
    from metis_b200 import api
    base, _, fix = name.partition(':')
    corrected = ('Q5', 'Q6') if fix else ()
    spec = Spec(base, workload_dir)
    api.release_engines()
    res = _run(spec, spec.root, corrected, mode, monkeypatch)
    if mode == 'windows':
        assert res.summary['num_windows'] > 1
    if not corrected:                                         # the limit goldens hold a sample of the plans
        pos = [res.candidates.index_of(o, s) for o, s in zip(spec.arr['ordinal'].tolist(), spec.arr['step'].tolist())]
        assert (_bits(res.costs[pos]) == _bits(spec.arr['cost'])).all()
    rc = res.recost([spec.cluster(spec.root), spec.cluster(spec.root)])
    assert rc.costs.shape == (2, len(res))
    assert (_bits(rc.costs) == _bits(np.stack([res.costs, res.costs]))).all()
    _same_ranked(rc.ranked(1), res.ranked())
    assert rc.best(0) == res.best() and _bits(rc.best(0)[6]) == _bits(res.best()[6])
    _check_regret(rc)
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['one_search', 'windows'])
@pytest.mark.parametrize('name', ['c3_homo64_mpl6', 'c4_het128'])
def test_api_recost_whole_space(name, mode, workload_dir, monkeypatch):
    """GPU item 1 on every candidate of C3-mpl6 (one bandwidth: the search's derived tables against the general path)
    and C4-mpl4."""
    _gpu()
    from metis_b200 import api
    spec = Spec(name, workload_dir)
    api.release_engines()
    res = _run(spec, spec.root, (), mode, monkeypatch)
    rc = res.recost([spec.cluster(spec.root)])
    assert (_bits(rc.costs[0]) == _bits(res.costs)).all()
    if name == 'c3_homo64_mpl6':
        assert len(res) == 273688
    api.release_engines()


FRESH = ['mix32', 'rough_t3', 'het32_tight', 'rough_q10', 'lim_s128_l255']


@pytest.mark.gpu
@pytest.mark.parametrize('name', FRESH + ['rough_t3:Q2', 'rough_q10:Q5Q6'])
def test_api_recost_is_a_fresh_search(name, workload_dir, tmp_path):
    """GPU item 2: for each bandwidth variant B, result_A.recost([B]).ranked(0) is cost_het_cluster(..., B).ranked()
    tuple for tuple, in order, costs bit for bit, and best(0) is the fresh best()."""
    _gpu()
    from metis_b200 import api
    base, _, fix = name.partition(':')
    corrected = {'Q2': ('Q2',), 'Q5Q6': ('Q5', 'Q6')}.get(fix, ())
    spec = Spec(base, workload_dir)
    kinds = ['q2'] if fix == 'Q2' else ['per_type', 'per_node']
    for k, kind in enumerate(kinds):
        a, b, _ = variant(spec.root, kind, str(tmp_path / kind), seed=k)
        api.release_engines()
        res = _run(spec, a, corrected)
        clusters = [spec.cluster(a), spec.cluster(b)]
        rc = res.recost(clusters)
        fresh = _run(spec, b, corrected)
        _same_ranked(rc.ranked(1), fresh.ranked())
        assert rc.best(1)[:6] == fresh.best()[:6] and _bits(rc.best(1)[6]) == _bits(fresh.best()[6])
        assert (_bits(rc.costs[0]) == _bits(res.costs)).all()
        _check_regret(rc)
    api.release_engines()


@pytest.mark.gpu
def test_api_recost_random_clusters(workload_dir, tmp_path):
    """GPU item 2 on 20 seeded random clusters with random per-node bandwidths (rough_t3's nodes, each under an IP of
    its own), all re-costed in one call, each against a fresh search."""
    _gpu()
    from metis_b200 import api
    spec = Spec('rough_t3', workload_dir)
    base, _, _ = variant(spec.root, 'per_node', str(tmp_path / 'b'))
    hosts, info = _hosts(base)
    rng = random.Random(2026)
    dirs = []
    for k in range(20):
        var = {ip: dict(v, intra_bandwidth=float(rng.choice([1, 2, 5, 10, 25, 50, 100, 400])) * 1e8 * rng.uniform(0.5, 2))
               for ip, v in info.items()}
        dirs.append(_write(str(tmp_path / f'r{k}'), hosts, var))
    api.release_engines()
    res = _run(spec, base)
    rc = res.recost([spec.cluster(d) for d in dirs])
    assert rc.costs.shape == (20, len(res))
    _check_regret(rc)
    for j, d in enumerate(dirs):
        fresh = _run(spec, d)
        _same_ranked(rc.ranked(j), fresh.ranked())
        assert rc.best(j)[:6] == fresh.best()[:6]
    api.release_engines()


@pytest.mark.gpu
def test_recost_survives_a_later_search(workload_dir, tmp_path):
    """GPU item 5: a recost taken after a later cost_het_cluster() call on other inputs is unchanged."""
    _gpu()
    from metis_b200 import api
    spec = Spec('rough_t3', workload_dir)
    _a, b, _ = variant(spec.root, 'per_type', str(tmp_path))
    api.release_engines()
    first = _run(spec, spec.root)
    scen = [spec.cluster(spec.root), spec.cluster(b)]
    before = first.recost(scen)
    other = Spec('mix32', workload_dir)
    assert len(_run(other, other.root)) != len(first)
    after = first.recost(scen)
    assert (_bits(before.costs) == _bits(after.costs)).all()
    assert (_bits(before.regret) == _bits(after.regret)).all()
    _same_ranked(after.ranked(1), before.ranked(1))
    api.release_engines()
