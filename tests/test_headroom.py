"""Memory headroom of every searched candidate, written by the search kernels (metis_het_search_headroom), and the two
views built on it: the headroom-constrained ranking (metis_headroom_select) and the cost / headroom Pareto front
(metis_headroom_front).

CPU: the host build of the evaluators with a sink that reads Scratch::mstate like DeviceSink (tests/hostsim/
headroom_sim.cpp) in the three host schedules, against the breakdown replay and the oracle twins; argument checks; the
multi-rank window merge carrying headroom (gloo, world size 2).  GPU (-m gpu): the same through the api, as one search
and in forced windows, in the bulk+chain and chain-only schedules; whole-space checks of the front and the filtered
ranking on C3-mpl6 and C4; the two kernels on synthetic arrays against numpy.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
import test_breakdown as tb
from conftest import load_golden
from metis_b200 import native, search

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'headroom_sim.cpp')
SIM_DEPS = [SIM_SRC] + tb.SIM_DEPS
TRANSCRIPT = ['c1', 'c2_het16', 'mix32']
ORACLE = ['rough_mix2', 'rough_t3', 'rough_q10', 'rough_long_int', 'rough_keys', 'q10_big_first', 'lim_s128_l255']
_sim = []


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def sim():
    """g++ build of tests/hostsim/headroom_sim.cpp at the compiled limits, hostsim.cpp's flags."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'libheadroom_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)
        lib = C.CDLL(out)
        lib.headroom_sim_search.restype = C.c_int
        _sim.append(lib)
    return _sim[0]


def _host_search(problem, space, mode):
    """headroom_sim_search -> (records, headroom) in estimate_costs order."""
    lib = sim()
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sp = space.as_struct(lambda n: keep[n].ctypes.data)
    cap = max(1024, space.num_plans * 4)
    rec = np.zeros(cap, dtype=native.RECORD_DTYPE)
    head = np.full(cap, np.nan)
    summary = native.MetisSearchSummary()
    assert lib.headroom_sim_search(C.byref(p), C.byref(sp), C.c_void_p(rec.ctypes.data), C.c_void_p(head.ctypes.data),
                                   C.c_int64(cap), C.byref(summary), C.c_int32(mode)) == 0
    n = int(summary.num_records)
    assert n <= cap
    order = np.lexsort((rec['step'][:n], rec['ordinal'][:n]))
    return rec[:n][order], head[:n][order]


def _inputs(name, workload_dir, corrected=()):
    if name in TRANSCRIPT:
        _meta, args, cluster, profile, cfg, seqs, api = tb._transcript_inputs(name, workload_dir)
        problem, space, _ = api.het_problem(args, cluster, profile, cfg, None, seqs, corrected=corrected)
        return problem, space, None
    meta, arr, w, root, seqs, problem, space = tb._golden_inputs(name, workload_dir, corrected=corrected)
    return problem, space, (meta, arr, w, root, seqs)


def _check_against_oracle(rec, head, oracle, corrected=(), n=30):
    meta, arr, w, root, seqs = oracle
    o = rec['ordinal']
    sample = set(o[np.linspace(0, len(o) - 1, min(n, len(o))).astype(np.int64)].tolist())
    for mask in (rec['num_repartition'] == 2, rec['num_repartition'] == 3):
        sample |= set(o[mask][:10].tolist())
    want = tb._oracle_want(w, root, meta, seqs, sample, corrected=corrected)
    assert want
    for ordinal, step, _nrep, _cost, _terms, stages in want:
        k = int(np.nonzero((rec['ordinal'] == ordinal) & (rec['step'] == step))[0][0])
        assert _bits(head[k]) == _bits(min(stages['memory_state'])), (ordinal, step)


@pytest.mark.parametrize('mode', [0, 1, 2], ids=['sequential', 'first_task_then_chain', 'chain_only'])
@pytest.mark.parametrize('name', TRANSCRIPT + ORACLE)
def test_host_headroom(name, mode, workload_dir):
    """Every emitted record's headroom is the breakdown replay's min_headroom bit for bit, and the oracle's
    min(memory_state) on sampled candidates (retried ones included)."""
    problem, space, oracle = _inputs(name, workload_dir)
    rec, head = _host_search(problem, space, mode)
    assert len(rec) > 0 and not np.isnan(head).any()
    bd = tb._host_breakdown(problem, space, rec)
    assert (_bits(head) == _bits(bd.min_headroom)).all()
    if oracle is not None and mode == 1:
        _check_against_oracle(rec, head, oracle, n=12 if name.startswith('lim') else 30)


def test_host_headroom_corrected(workload_dir):
    """A ('Q5', 'Q6') corrected search: the headroom follows the corrected demand and state."""
    fix = ('Q5', 'Q6')
    problem, space, oracle = _inputs('rough_q10', workload_dir, corrected=fix)
    for mode in (0, 1, 2):
        rec, head = _host_search(problem, space, mode)
        assert (_bits(head) == _bits(tb._host_breakdown(problem, space, rec).min_headroom)).all()
        if mode == 1:
            _check_against_oracle(rec, head, oracle, corrected=fix)


@pytest.mark.parametrize('bad', [float('nan'), float('inf'), -float('inf'), 'x', None, True])
def test_threshold_must_be_finite(bad):
    with pytest.raises(ValueError, match='finite'):
        search.check_threshold(bad)
    assert search.check_threshold(np.float32(1.5)) == 1.5 and search.check_threshold(-3) == -3.0


class _NoHeadroom:
    def __init__(self):
        self.records = np.zeros(3, dtype=native.RECORD_DTYPE)
        self.cost = self.records['cost']
        self.headroom = None

    def __len__(self):
        return 3


def test_headroom_views_need_the_flag():
    """pareto() and ranked(min_headroom=...) on a result searched without headroom=True raise, naming the flag."""
    from metis_b200 import api
    res = api.HetSearchResult(_NoHeadroom(), np.arange(3, dtype=np.uint32), {})
    assert res.headroom is None
    with pytest.raises(ValueError, match='headroom=True'):
        res.pareto()
    with pytest.raises(ValueError, match='headroom=True'):
        res.ranked(2, min_headroom=0.0)
    with pytest.raises(ValueError, match='finite'):
        res.ranked(2, min_headroom=float('nan'))


WORKER = r'''
import os, sys
sys.path.insert(0, os.environ['REPO'])
import numpy as np
import torch, torch.distributed as dist
dist.init_process_group('gloo', init_method='tcp://127.0.0.1:' + os.environ['PORT'],
                        rank=int(os.environ['RANK']), world_size=2)
from metis_b200 import native, search
rank = dist.get_rank()

def head_of(ordinal, step):                                  # any value that identifies the record
    return ordinal * 1000.0 + step + 0.25

rng = np.random.default_rng(7)
merge = search.WindowMerge(4, with_headroom=True)
for w, base in enumerate([0, 100, 250, 400]):
    n = int(rng.integers(0, 9)) if w != 2 else 0             # window 2 holds no record of either rank
    if rank == 1 and w == 1:
        n = 5
    ords = np.sort(rng.choice(np.arange(rank, 100, 2), size=n, replace=False)).astype(np.uint32)
    rec = np.zeros(2 * n, dtype=native.RECORD_DTYPE)
    rec['ordinal'] = np.repeat(ords, 2)
    rec['step'] = np.tile([0, 1], n)
    rec['cost'] = rng.random(2 * n)
    rec['num_stage'] = 2
    merge.add(base, dict(num_records=len(rec)), None, rec, head_of(rec['ordinal'].astype(np.float64) + base, rec['step']))
merged = merge.result()
assert len(merged.headroom) == len(merged.records)
out = search.gather_window_records(merged, 'cpu')
win = np.searchsorted(out.firsts, np.arange(len(out.records)), side='right') - 1
glob = out.bases[win] + out.records['ordinal'].astype(np.int64)
assert len(out.headroom) == len(out.records) > 0
assert (out.headroom == head_of(glob.astype(np.float64), out.records['step'])).all()
key = list(zip(glob.tolist(), out.records['step'].tolist()))
assert key == sorted(key)
total = torch.tensor([len(merged.records)]); dist.all_reduce(total)
assert int(total) == len(out.records)
dist.barrier(); dist.destroy_process_group()
print('rank', rank, 'ok')
'''


def test_two_rank_window_gather_carries_headroom(tmp_path):
    """world size 2 over gloo, synthetic per-rank windows: gather_window_records merges every rank's records in
    estimate_costs order and the headroom travels with its record, across windows (one of them empty)."""
    import socket
    import sys
    script = tmp_path / 'worker.py'
    script.write_text(WORKER)
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    repo = os.path.dirname(HERE)
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(os.environ, REPO=repo, RANK=str(r), PORT=str(port)),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=300)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), '\n'.join(outs)


# ---- numpy references -----------------------------------------------------------------------------------------------
def front_reference(cost, head):
    """Positions of the Pareto front by the rule itself: not dominated (cost <= and headroom >=, one strict), first of
    equal (cost, headroom) pairs; by ascending cost."""
    n = len(cost)
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    ucost, inv = np.unique(cost, return_inverse=True)
    run_max = np.full(len(ucost), -np.inf)
    np.maximum.at(run_max, inv, head)
    lower = np.concatenate([[-np.inf], np.maximum.accumulate(run_max)[:-1]])   # best headroom at a lower cost
    ok = (head >= run_max[inv]) & (head > lower[inv])
    cand = np.nonzero(ok)[0]                                  # positions ascending: the first of equal pairs first
    _, first = np.unique(inv[cand], return_index=True)        # one per cost (its maximum, first position)
    pos = cand[first]
    return pos[np.argsort(cost[pos], kind='stable')]


def front_brute(cost, head):
    keep = []
    for i in range(len(cost)):
        dom = (cost <= cost[i]) & (head >= head[i]) & ((cost < cost[i]) | (head > head[i]))
        same = (cost == cost[i]) & (head == head[i]) & (np.arange(len(cost)) < i)
        if not dom.any() and not same.any():
            keep.append(i)
    keep = np.array(keep, dtype=np.int64)
    return keep[np.argsort(cost[keep], kind='stable')] if len(keep) else keep


def select_reference(rank, head, x, k):
    hits = rank[head[rank] >= x].astype(np.int64)
    return hits[:k] if k is not None else hits, len(hits)


def test_front_reference_is_the_rule():
    """The vectorised reference equals the rule checked pair by pair, with heavy ties of cost and of (cost, headroom)."""
    rng = np.random.default_rng(3)
    for n in (0, 1, 2, 7, 300, 1500):
        cost = rng.integers(0, 12, n).astype(np.float64)
        head = rng.integers(0, 9, n).astype(np.float64)
        assert (front_reference(cost, head) == front_brute(cost, head)).all()


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()
    return torch


def _synthetic(n, seed, ncost, nhead):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, dtype=native.RECORD_DTYPE)
    rec['cost'] = rng.integers(0, ncost, n) * 0.5 + 1.0
    rec['ordinal'] = np.arange(n, dtype=np.uint32)
    head = rng.integers(-nhead, nhead, n) * 64.0
    return rec, head, np.argsort(rec['cost'], kind='stable').astype(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [0, 1, 2047, 2048, 2049, 3 * 2048 + 5, 10 ** 7])
def test_select_and_front_kernels_on_synthetic_arrays(n):
    """metis_headroom_select / metis_headroom_front against numpy: empty, one entry, around the 2048-entry tile and
    10^7 entries; heavy cost ties with differing headrooms and repeated (cost, headroom) pairs."""
    _gpu()
    shapes = [(64, 16), (3, 1000), (n + 1, 4 * n + 8)] if n < 10 ** 6 else [(50000, 4000), (7, 10 ** 6)]
    for seed, (ncost, nhead) in enumerate(shapes):
        rec, head, rank = _synthetic(n, seed, ncost, nhead)
        idx = search.HeadroomIndex(rec, head, rank, 'cuda:0')
        want = front_reference(rec['cost'], head)
        got = idx.front()
        assert (got == want).all(), (n, seed, len(got), len(want))
        if n:
            assert (np.diff(head[got]) > 0).all() and (np.diff(rec['cost'][got]) > 0).all()
        levels = [-1e300, 0.0, 1e300] + ([float(head[n // 2]), float(head.max())] if n else [])
        for x in levels:
            for k in (None, 0, 1, 5000):
                pos, total = idx.select(x, k)
                wpos, wtotal = select_reference(rank, head, x, k)
                assert total == wtotal and (pos == wpos).all(), (n, x, k)


def _run(name, workload_dir, headroom):
    from metis_b200 import api
    if name in TRANSCRIPT:
        _meta, args, cluster, profile, cfg, seqs, api = tb._transcript_inputs(name, workload_dir)
        volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
        return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                    api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                                    device='cuda:0', headroom=headroom)
    meta, arr = load_golden(name)
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    w, root, _ = workload_dir(name)
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), meta['file_order']).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                      vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
    args = parse_args(w.cli_args(root))
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                api.LayerLoadBalancer(cluster, profile, cfg, args.gbs),
                                node_sequences=[tuple(s) for s in meta['node_sequences']], device='cuda:0',
                                headroom=headroom)


def _schedule(monkeypatch, reserved):
    shard = native.MetisShard
    monkeypatch.setattr(native, 'MetisShard', lambda rank, world, tile, _r: shard(rank, world, tile, reserved))


_ORACLE_WANT = {}


@pytest.mark.gpu
@pytest.mark.parametrize('reserved', [1, 2 ** 31 - 1], ids=['bulk_then_chain', 'chain_only'])
@pytest.mark.parametrize('split', [False, True], ids=['one_search', 'windows'])
@pytest.mark.parametrize('name', TRANSCRIPT + ORACLE)
def test_api_headroom(name, split, reserved, workload_dir, monkeypatch):
    """headroom=True leaves the tuples, summary and best() as they are; result.headroom is the breakdown replay's
    min_headroom bit for bit (aligned with the records across window boundaries) and the oracle's on samples;
    pareto() and ranked(k, min_headroom=x) on the result, one search or windowed, equal the numpy references."""
    torch = _gpu()
    from metis_b200 import api
    api.release_engines()
    _schedule(monkeypatch, reserved)
    if split:
        from test_windowed_search import _force_windows
        _force_windows(monkeypatch, 3)
    plain = _run(name, workload_dir, False)
    with_h = _run(name, workload_dir, True)
    assert plain.headroom is None and 'headroom_s' not in plain.timings and 'headroom_s' in with_h.timings
    assert (with_h.summary['num_windows'] > 1) == split
    assert with_h.summary == plain.summary
    assert list(with_h) == list(plain) and with_h.best() == plain.best()
    assert with_h.headroom.dtype == np.float64 and len(with_h.headroom) == len(with_h)
    bd = with_h.breakdown(slice(None), per_stage=False)
    assert (_bits(with_h.headroom) == _bits(bd.min_headroom)).all()
    # the two views on this result (a WindowedCandidates with the window ranker when split)
    pos, cost, head = with_h.pareto()
    assert (pos == front_reference(with_h.costs, with_h.headroom)).all() and (head == with_h.headroom[pos]).all()
    x = float(np.median(with_h.headroom))
    want, _ = select_reference(with_h.rank_order, with_h.headroom, x, 7)
    assert with_h.ranked(7, min_headroom=x) == with_h.candidates.tuples(want)
    assert with_h.ranked(7) == plain.ranked(7)
    assert with_h._index().device == torch.device('cuda:0')
    with pytest.raises(ValueError, match='k must be'):
        with_h.ranked(-1, min_headroom=x)
    if name in ORACLE:
        if name not in _ORACLE_WANT:
            meta, arr, w, root, seqs, *_ = tb._golden_inputs(name, workload_dir)
            _ORACLE_WANT[name] = tb._oracle_want(w, root, meta, seqs, tb._sample_ordinals(arr, 12))
        want = _ORACLE_WANT[name]
        pos = tb._result_positions(with_h, want)
        assert (_bits(with_h.headroom[pos]) == _bits([min(x[5]['memory_state']) for x in want])).all()
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['c3_homo64_mpl6', 'c4_het128'])
def test_whole_space_front_and_filter(name, workload_dir):
    """Every candidate: headroom equals the breakdown and is never negative; pareto() equals the numpy rule;
    ranked(k, min_headroom=x) equals a stable filter of ranked() below, at tied values of, and above every headroom."""
    _gpu()
    from metis_b200 import api
    api.release_engines()
    res = _run(name, workload_dir, True)
    h = res.headroom
    bd = res.breakdown(slice(None), per_stage=False)
    assert (_bits(h) == _bits(bd.min_headroom)).all() and (h >= 0).all()
    if name == 'c3_homo64_mpl6':
        assert len(res) == 273688
    pos, cost, head = res.pareto()
    assert (pos == front_reference(res.costs, h)).all()
    assert (cost == res.costs[pos]).all() and (np.diff(head) > 0).all()
    res.ranked(1)
    rank = res.rank_order
    vals, counts = np.unique(h, return_counts=True)
    tied = float(vals[np.argmax(counts)])                     # the most repeated headroom
    for x in (float(h.min()) - 1.0, tied, float(np.median(h)), float(h.max()) + 1.0):
        for k in (1, 100, None):
            got, total = res._index().select(x, k)
            want, wtotal = select_reference(rank, h, x, k)
            assert total == wtotal and (got == want).all(), (x, k)
    assert res.ranked(20, min_headroom=float(h.min()) - 1.0) == res.ranked(20)
    assert res.ranked(20, min_headroom=float(h.max()) + 1.0) == []
    want, _ = select_reference(rank, h, tied, 10)
    assert res.ranked(10, min_headroom=tied) == res.candidates.tuples(want)
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('split', [False, True], ids=['one_search', 'windows'])
def test_multi_rank_gather_carries_headroom(split, workload_dir, monkeypatch):
    """With torch.distributed initialised (NCCL, a world of one rank) cost_het_cluster takes the multi-rank path:
    gather_records (one search: padded all_gather, position sort, headroom permuted with the records) or
    gather_window_records (windows).  The headroom stays aligned with its records: bit for bit the single-process
    result's."""
    import socket
    torch = _gpu()
    import torch.distributed as dist
    from metis_b200 import api
    api.release_engines()
    want = _run('rough_t3', workload_dir, True)
    if split:
        from test_windowed_search import _force_windows
        _force_windows(monkeypatch, 3)
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    torch.cuda.set_device(0)
    dist.init_process_group('nccl', init_method=f'tcp://127.0.0.1:{port}', rank=0, world_size=1)
    try:
        api.release_engines()
        got = _run('rough_t3', workload_dir, True)
    finally:
        dist.destroy_process_group()
        api.release_engines()
    assert (got.summary['num_windows'] > 1) == split
    if not split:
        assert got.summary['records_per_rank'] == [len(want)]   # the gather path ran
    assert list(got) == list(want)
    assert (_bits(got.headroom) == _bits(want.headroom)).all()
    assert (got.pareto()[0] == want.pareto()[0]).all()
