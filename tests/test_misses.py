"""Out-of-memory partition attempts of a search ("misses"), written by the search kernels (metis_het_search_outputs),
and the views built on them: HetSearchResult.misses, closest_misses(k) and miss_detail(idx).

CPU: the host build of the evaluators with the miss hook of MissSink (tests/hostsim/misses_sim.cpp) in the host
schedules, against the misses read off the reference's transcripts and against the oracle twin (tests/oracle_misses.py)
on goldens, a corrected run and a cluster on which nothing fits; the identity of the counters; argument checks; the
multi-rank window merge carrying misses (gloo, world size 2).  GPU (-m gpu): the same through the api in the bulk+chain
and chain-only schedules, the replay path, forced windows and a device-listed space; whole-space checks on C3-mpl6 and
C4-mpl4.
"""
import ctypes as C
import gzip
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
import oracle_misses as om
import test_breakdown as tb
from conftest import GOLDEN, load_golden
from metis_b200 import native, search
from oracle import metis_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'misses_sim.cpp')
SIM_DEPS = [SIM_SRC] + tb.SIM_DEPS
TRANSCRIPT = ['c1', 'c2_het16', 'mix32']
ORACLE = ['het32_tight', 'rough_mix2', 'rough_t3', 'rough_q10', 'rough_long_int', 'rough_keys', 'q10_big_first',
          'lim_s128_l255']
MODES = [0, 1, 2, 3, 4]
MODE_IDS = ['sequential', 'first_task_then_chain', 'chain_only', 'chain_only_reversed', 'first_task_then_replay']
_sim = []


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def sim():
    """g++ build of tests/hostsim/misses_sim.cpp at the compiled limits, hostsim.cpp's flags."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'libmisses_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)
        lib = C.CDLL(out)
        lib.misses_sim_search.restype = C.c_int
        _sim.append(lib)
    return _sim[0]


def _host_search(problem, space, mode, miss_capacity=None):
    """misses_sim_search -> (records, misses in reference order, summary)."""
    lib = sim()
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sp = space.as_struct(lambda n: keep[n].ctypes.data)
    cap = max(1024, space.num_plans * 4)
    mcap = cap if miss_capacity is None else miss_capacity
    rec = np.zeros(cap, dtype=native.RECORD_DTYPE)
    summary = native.MetisSearchSummary()
    while True:                                               # like HetSearcher.run: regrow past the count, search again
        miss = np.zeros(max(mcap, 1), dtype=native.MISS_DTYPE)
        assert lib.misses_sim_search(C.byref(p), C.byref(sp), C.c_void_p(rec.ctypes.data), C.c_int64(cap),
                                     C.c_void_p(miss.ctypes.data), C.c_int64(mcap), C.byref(summary),
                                     C.c_int32(mode)) == 0
        if miss_capacity is not None or int(summary.reserved[3]) <= mcap:
            break
        mcap = int(summary.reserved[3])
    n, m = int(summary.num_records), int(summary.reserved[3])
    assert n <= cap
    miss = miss[:min(m, mcap)]
    order = np.lexsort((miss['key'], miss['ordinal']))
    return rec[:n], miss[order], summary


def _tuples(miss):
    """(ordinal, call, attempt, deficit bits, stage) per miss."""
    return list(zip(miss['ordinal'].tolist(), (miss['key'] >> 2).tolist(), (miss['key'] & 3).tolist(),
                    _bits(miss['deficit']).tolist(), miss['stage'].tolist()))


# ---- the reference's transcripts --------------------------------------------------------------------------------------
def transcript_misses(name):
    """Every partition attempt of the reference's transcript whose printed memory_state has a negative entry:
    (ordinal, call, attempt, deficit bits, stage), in the transcript's order; and the number of attempts."""
    out, ordinal, call, attempt, attempts = [], -1, -1, 0, 0
    for line in gzip.open(os.path.join(GOLDEN, f'transcript_{name}.txt.gz'), 'rt'):
        if line.startswith('inter_stage_plan:'):
            ordinal, call = ordinal + 1, -1
        elif line.startswith('valid_strategies:'):
            call, attempt = call + 1, 0
        else:
            m = re.match(r'stage_memory_demand: \[.*\], memory_state: \[(.*)\]$', line.rstrip('\n'))
            if m:
                attempt += 1
                attempts += 1
                state = [float(t) for t in m.group(1).split(',')]
                low = min(state)
                if low < 0:
                    out.append((ordinal, call, attempt, int(_bits(-low)), state.index(low)))
    return out, attempts


def test_transcript_counts():
    """The transcripts hold what the misses must reproduce: 32 of 388 attempts of mix32, 2 953 of 4 000 of c2_het16,
    none of c1's 19; every attempt is a candidate or a miss."""
    want = {'mix32': (388, 32), 'c2_het16': (4000, 2953), 'c1': (19, 0)}
    for name, (attempts, n) in want.items():
        got, total = transcript_misses(name)
        assert (total, len(got)) == (attempts, n)
        meta = json.load(open(os.path.join(GOLDEN, f'transcript_{name}.json')))
        assert meta['costs'] == attempts - n


@pytest.mark.parametrize('mode', MODES, ids=MODE_IDS)
@pytest.mark.parametrize('name', TRANSCRIPT)
def test_host_misses_equal_the_transcript(name, mode, workload_dir):
    """Every out-of-memory attempt the reference printed, bit for bit and in its order, in every host schedule; the
    counters satisfy num_balancer_runs == num_records + num_keyerror + num_oom_attempts."""
    _meta, args, cluster, profile, cfg, seqs, api = tb._transcript_inputs(name, workload_dir)
    problem, space, _ = api.het_problem(args, cluster, profile, cfg, None, seqs)
    rec, miss, summary = _host_search(problem, space, mode)
    want, _ = transcript_misses(name)
    assert _tuples(miss) == want
    assert (miss['deficit'] > 0).all() and (miss['stage'] < miss['num_stage']).all()
    assert summary.num_balancer_runs == summary.num_records + summary.num_keyerror + summary.reserved[3]


def test_host_count_is_exact_past_capacity(workload_dir):
    """A miss buffer smaller than the count: the first ones are written, the count stays exact."""
    _meta, args, cluster, profile, cfg, seqs, api = tb._transcript_inputs('c2_het16', workload_dir)
    problem, space, _ = api.het_problem(args, cluster, profile, cfg, None, seqs)
    _rec, full, _ = _host_search(problem, space, 0)
    for cap in (0, 1, 100):
        _rec, part, summary = _host_search(problem, space, 0, miss_capacity=cap)
        assert int(summary.reserved[3]) == len(full) and len(part) == min(cap, len(full))
        assert set(_tuples(part)) <= set(_tuples(full))


# ---- the oracle twin --------------------------------------------------------------------------------------------------
def _sample(miss, num_plans, n=40):
    """Plans for the oracle: evenly spaced ones, and those whose misses reach a later call or the third attempt."""
    pick = set(np.linspace(0, num_plans - 1, min(n, num_plans)).astype(np.int64).tolist())
    for mask in (miss['key'] >> 2 > 0, miss['key'] & 3 == 3, miss['key'] & 3 == 2):
        pick |= set(miss['ordinal'][mask][:10].tolist())
    return pick


def _restricted(miss, sample):
    return miss[np.isin(miss['ordinal'], list(sample))]


def _oracle_misses(name, workload_dir, corrected=(), root=None, meta=None, w=None, sample=None):
    if root is None:
        meta, _arr, w, root, _seqs, *_ = tb._golden_inputs(name, workload_dir, corrected=corrected)
    seqs = [tuple(s) for s in meta['node_sequences']]
    ocl = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'), corrected=corrected)
    oprof, _ = orc.load_profile_dir(os.path.join(root, 'profile'), meta['file_order'])
    omodel = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size, oprof['model']['parameters'])
    return om.het_misses(oprof, ocl, omodel, seqs, w.gbs, w.num_layers, w.variance, w.max_permute_len, w.max_tp,
                         w.max_bs, corrected=corrected, plan_filter=None if sample is None else sample.__contains__)


def _oracle_tuples(misses):
    return [(m.ordinal, m.call, m.attempt, int(_bits(m.deficit)), m.stage) for m in misses]


def test_oracle_twin_keeps_the_oracles_search(workload_dir):
    """Wrapping partition_layer changes nothing the oracle returns; its misses and candidates add up to the balancer
    runs."""
    meta, arr, w, root, seqs, *_ = tb._golden_inputs('rough_t3', workload_dir)
    cands, counters, misses = _oracle_misses('rough_t3', workload_dir)
    plain, plain_counters = orc.het_search(*_oracle_args(meta, w, root))
    assert cands == plain and counters == plain_counters
    assert counters['runs'] == counters['C'] + counters['keyerr'] + len(misses)
    assert misses and all(m.deficit > 0 for m in misses)


def _oracle_args(meta, w, root):
    seqs = [tuple(s) for s in meta['node_sequences']]
    ocl = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    oprof, _ = orc.load_profile_dir(os.path.join(root, 'profile'), meta['file_order'])
    omodel = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size, oprof['model']['parameters'])
    return oprof, ocl, omodel, seqs, w.gbs, w.num_layers, w.variance, w.max_permute_len, w.max_tp, w.max_bs


@pytest.mark.parametrize('name', ORACLE)
def test_host_misses_equal_the_oracle(name, workload_dir):
    """The golden spaces (retries, Q1 blocks, Q10 clusters, S = 128 and L = 255): the host build's misses are the
    oracle twin's, in reference order, in the sequential and first-task-then-chain schedules."""
    _meta, _arr, _w, _root, _seqs, problem, space = tb._golden_inputs(name, workload_dir)
    _rec, miss1, summary = _host_search(problem, space, 1)
    assert summary.num_balancer_runs == summary.num_records + summary.num_keyerror + summary.reserved[3]
    sample = _sample(miss1, space.num_plans)
    _c, _counters, want = _oracle_misses(name, workload_dir, sample=sample)
    assert _tuples(_restricted(miss1, sample)) == _oracle_tuples(want), name
    if not name.startswith('lim'):
        _rec, miss0, _ = _host_search(problem, space, 0)
        assert _tuples(miss0) == _tuples(miss1)


def test_host_misses_corrected(workload_dir):
    """A ('Q5', 'Q6') corrected search: the misses follow the corrected balancer and demand."""
    fix = ('Q5', 'Q6')
    _meta, _arr, _w, _root, _seqs, problem, space = tb._golden_inputs('rough_q10', workload_dir, corrected=fix)
    _rec, miss1, _ = _host_search(problem, space, 1)
    sample = _sample(miss1, space.num_plans)
    _c, _counters, want = _oracle_misses('rough_q10', workload_dir, corrected=fix, sample=sample)
    assert want
    for mode in (0, 1, 2):
        _rec, miss, _ = _host_search(problem, space, mode)
        assert _tuples(_restricted(miss, sample)) == _oracle_tuples(want)


def infeasible_inputs(workload_dir, dst):
    """The c1 cluster with every device's memory cut until no partition attempt fits: (root, meta, workload)."""
    meta, _arr = load_golden('rough_t3')
    w, root, _ = workload_dir('rough_t3')
    if not os.path.exists(dst):
        shutil.copytree(root, dst)
        path = os.path.join(dst, 'clusterfile.json')
        cfg = json.load(open(path))
        for node in cfg.values():
            if isinstance(node, dict) and 'memory' in node:
                node['memory'] = node['memory'] // 64
        json.dump(cfg, open(path, 'w'))
    return dst, meta, w


def test_infeasible_cluster(workload_dir, tmp_path_factory):
    """Memory cut until nothing fits: the reference returns no candidate; the host build's misses are the oracle's, and
    the closest one is the oracle's smallest deficit."""
    root, meta, w = infeasible_inputs(workload_dir, str(tmp_path_factory.mktemp('infeasible') / 'w'))
    cands, counters, want = _oracle_misses(None, workload_dir, root=root, meta=meta, w=w)
    assert cands == [] and want and counters['runs'] == len(want)
    problem, space = _flat_inputs(root, meta, w)
    for mode in (0, 1, 2):
        rec, miss, summary = _host_search(problem, space, mode)
        assert len(rec) == 0 and _tuples(miss) == _oracle_tuples(want)
        assert summary.num_balancer_runs == summary.reserved[3]


def _flat_inputs(root, meta, w):
    from metis_b200 import flatten
    cluster, profile, _types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                   w.sequence_length, w.vocab_size)
    seqs = [tuple(s) for s in meta['node_sequences']]
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
    space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance,
                                     w.max_permute_len)
    return problem, space


# ---- argument checks and views without the flag -----------------------------------------------------------------------
class _NoMisses:
    def __init__(self):
        self.records = np.zeros(3, dtype=native.RECORD_DTYPE)
        self.cost = self.records['cost']

    def __len__(self):
        return 3


def test_miss_views_need_the_flag():
    """misses, closest_misses and miss_detail on a result searched without misses=True raise, naming the flag."""
    from metis_b200 import api
    res = api.HetSearchResult(_NoMisses(), np.arange(3, dtype=np.uint32), {})
    for view in (lambda: res.misses, lambda: res.closest_misses(3), lambda: res.miss_detail([0])):
        with pytest.raises(ValueError, match='misses=True'):
            view()


def test_record_layout_matches_the_sort_key():
    """MetisMiss keeps the deficit, ordinal and call/attempt key where MetisRecord keeps cost, ordinal and step, so one
    record sort orders both; the host form packs into whole int64 words for the gathers."""
    rec, miss = np.dtype(native.RECORD_DTYPE), np.dtype(native.MISS_DTYPE)
    assert rec.itemsize == miss.itemsize == 16
    for r, m in (('cost', 'deficit'), ('ordinal', 'ordinal'), ('step', 'key')):
        assert rec.fields[r][1] == miss.fields[m][1] and rec.fields[r][0].itemsize == miss.fields[m][0].itemsize
    assert np.dtype(search.MISS_HOST_DTYPE).itemsize % 8 == 0


def test_host_rows_on_the_device_equal_the_host_conversion():
    """HetSearcher.run converts MetisMiss rows with torch (host_rows_device); WindowMerge with numpy (misses_to_host):
    the same words for every field value, extremes included."""
    import torch
    rng = np.random.default_rng(5)
    raw = np.zeros(4099, dtype=native.MISS_DTYPE)
    raw['deficit'] = rng.random(len(raw)) * 1e6
    raw['ordinal'] = rng.integers(0, 2 ** 32, len(raw), dtype=np.uint64)
    raw['key'] = rng.integers(0, 2 ** 16, len(raw))
    raw['stage'] = rng.integers(0, 256, len(raw))
    raw['num_stage'] = rng.integers(0, 256, len(raw))
    raw[:2] = [(1.0, 2 ** 32 - 1, 2 ** 16 - 1, 255, 255), (0.5, 0, 0, 0, 0)]
    dev = search.host_rows_device(torch.from_numpy(raw.view(np.int64).copy())).numpy().view(np.uint64)
    host = search.misses_to_host(raw)
    assert (dev.reshape(-1) == host.view(np.uint64)).all()
    assert (host['call'] == raw['key'] >> 2).all() and (host['attempt'] == raw['key'] & 3).all()
    assert (host['ordinal'] == raw['ordinal'].astype(np.int64)).all() and (host['num_stage'] == raw['num_stage']).all()


def test_window_merge_makes_ordinals_global():
    """WindowMerge appends each window's misses with its base added, counts them, and keeps an empty table for a search
    without any."""
    merge = search.WindowMerge(3, with_misses=True)
    for base, ords in ((0, [1, 1, 7]), (100, []), (250, [3])):
        raw = np.zeros(len(ords), dtype=native.MISS_DTYPE)
        raw['ordinal'] = ords
        raw['key'] = [(i << 2) | 1 for i in range(len(ords))]
        raw['deficit'] = 1.5
        merge.add(base, dict(num_oom_attempts=len(ords)), None, None, misses=raw)
    out = merge.result()
    assert out.misses['ordinal'].tolist() == [1, 1, 7, 253] and out.summary['num_oom_attempts'] == 4
    assert out.misses['call'].tolist() == [0, 1, 2, 0] and (out.misses['attempt'] == 1).all()
    empty = search.WindowMerge(1, with_misses=True)
    empty.add(0, {}, None, None, misses=np.zeros(0, dtype=native.MISS_DTYPE))
    assert len(empty.result().misses) == 0


def test_host_memory_capacity_is_the_evaluators(workload_dir):
    """search.memory_capacity (used by miss_detail) equals the capacity the breakdown replay reports, bit for bit."""
    _meta, args, cluster, profile, cfg, seqs, api = tb._transcript_inputs('mix32', workload_dir)
    problem, space, _ = api.het_problem(args, cluster, profile, cfg, None, seqs)
    rec, _det, _summary = hs.host_het_search(problem, space, mode=0, want_detail=False)
    rec = rec[np.lexsort((rec['step'], rec['ordinal']))][:200]
    bd = tb._host_breakdown(problem, space, rec)
    for k in range(len(rec)):
        ns, _label, _row, _batches, codes = space.locate(int(rec['ordinal'][k]))
        groups = [1 << int(c) for c in codes]
        got = search.memory_capacity(problem, ns, groups)
        S = len(groups)
        assert (_bits(got) == _bits(bd.memory_capacity[k, :S])).all()


def test_search_outputs_argument_checks(workload_dir):
    """metis_het_search_outputs refuses a negative miss capacity and a positive one without a buffer, before touching
    the device, naming the mismatch; NULL misses with capacity 0 passes these checks."""
    from metis_b200 import api
    _meta, args, cluster, profile, cfg, seqs, _api = tb._transcript_inputs('c1', workload_dir)
    problem, space, _ = api.het_problem(args, cluster, profile, cfg, None, seqs)
    lib = native.load_library()
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sp = space.as_struct(lambda n: keep[n].ctypes.data)
    shard = native.MetisShard(0, 1, 128, 0)
    rec = np.zeros(4, dtype=native.RECORD_DTYPE)
    summary = native.MetisSearchSummary()
    dummy = np.zeros(16, dtype=native.MISS_DTYPE)

    def call(misses, cap, workspace_bytes=1):
        return lib.metis_het_search_outputs(C.byref(p), C.byref(sp), C.byref(shard), C.c_void_p(rec.ctypes.data),
                                            C.c_int64(len(rec)), None, C.c_int32(0), None, misses, C.c_int64(cap),
                                            C.c_void_p(rec.ctypes.data), C.c_int64(workspace_bytes), C.byref(summary),
                                            None)
    for misses, cap in ((None, 5), (C.c_void_p(dummy.ctypes.data), -1), (None, -1)):
        assert call(misses, cap) == -2                        # METIS_E_ARG
        assert b'misses/miss_capacity mismatch' in lib.metis_last_error()
    # the miss arguments pass; the search then stops at the (deliberately) too small workspace, still on the host
    assert call(None, 0) == -3 and b'workspace too small' in lib.metis_last_error()


WORKER = r'''
import os, sys
sys.path.insert(0, os.environ['REPO'])
import numpy as np
import torch, torch.distributed as dist
dist.init_process_group('gloo', init_method='tcp://127.0.0.1:' + os.environ['PORT'],
                        rank=int(os.environ['RANK']), world_size=2)
from metis_b200 import native, search
rank = dist.get_rank()
rng = np.random.default_rng(11)
merge = search.WindowMerge(3, with_misses=True)
for w, base in enumerate([0, 100, 250]):
    ords = np.sort(rng.choice(np.arange(rank, 100, 2), size=4 if w != 1 else 0, replace=False)).astype(np.uint32)
    raw = np.zeros(2 * len(ords), dtype=native.MISS_DTYPE)
    raw['ordinal'] = np.repeat(ords, 2)
    raw['key'] = np.tile([1, 2], len(ords))
    raw['deficit'] = raw['ordinal'] * 10.0 + base + raw['key']
    raw['num_stage'] = 3
    merge.add(base, dict(num_oom_attempts=len(raw)), None, None, misses=raw)
merged = merge.result()
out = search.gather_window_records(merged, 'cpu')
m = out.misses
assert len(m) == 2 * len(merged.misses)
key = list(zip(m['ordinal'].tolist(), m['call'].tolist(), m['attempt'].tolist()))
assert key == sorted(key) and len(set(key)) == len(key)
base = np.where(m['ordinal'] >= 250, 250, 0)
assert (m['deficit'] == (m['ordinal'] - base) * 10.0 + base + m['attempt']).all()
dist.barrier(); dist.destroy_process_group()
print('rank', rank, 'ok')
'''


def test_two_rank_window_gather_carries_misses(tmp_path):
    """world size 2 over gloo, synthetic per-rank windows: gather_window_records also gathers every rank's misses and
    merges them into the reference's order, each with its own values, across windows (one of them empty)."""
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


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()
    return torch


def _api_inputs(name, workload_dir, root=None, meta=None, w=None):
    """(args, cluster, profile, cfg, seqs) of a transcript or golden workload, or of a workload directory given."""
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    if root is None and name in TRANSCRIPT:
        _meta, args, cluster, profile, cfg, seqs, _api = tb._transcript_inputs(name, workload_dir)
        return args, cluster, profile, cfg, seqs
    if root is None:
        meta, _arr = load_golden(name)
        w, root, _ = workload_dir(name)
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), meta['file_order']).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                      vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
    return parse_args(w.cli_args(root)), cluster, profile, cfg, [tuple(s) for s in meta['node_sequences']]


def _run(inputs, **flags):
    from metis_b200 import api
    args, cluster, profile, cfg, seqs = inputs
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                                device='cuda:0', **flags)


def _schedule(monkeypatch, reserved):
    shard = native.MetisShard
    monkeypatch.setattr(native, 'MetisShard', lambda rank, world, tile, _r: shard(rank, world, tile, reserved))


def _result_tuples(res):
    m = res.misses
    return list(zip(m.ordinal.tolist(), m.call.tolist(), m.attempt.tolist(), _bits(m.deficit).tolist(),
                    m.stage.tolist()))


def _host_want(name, workload_dir, inputs):
    from metis_b200 import api
    args, cluster, profile, cfg, seqs = inputs
    problem, space, _ = api.het_problem(args, cluster, profile, cfg, None, seqs)
    _rec, miss, summary = _host_search(problem, space, 1)
    return _tuples(miss), summary


def _check_views(res, k=5):
    """closest_misses(k) is the numpy lexsort's first k; miss_detail's state minima are the deficits."""
    m = res.misses
    want = np.lexsort((np.arange(len(m)), m.deficit))[:k]
    assert (res._closest_order()[:k] == want).all()
    got = res.closest_misses(k)
    assert [(t[5], _bits(t[6]), t[7]) for t in got] == [(int(m.attempt[i]), _bits(m.deficit[i]), int(m.stage[i]))
                                                         for i in want]
    det = res.miss_detail(want)
    for r, i in enumerate(want.tolist()):
        S = int(m.num_stage[i])
        st = det.memory_state[r]
        assert np.isnan(st[S:]).all() and _bits(-st[:S].min()) == _bits(m.deficit[i])
        assert int(np.argmin(st[:S])) == int(m.stage[i])
        cap = det.memory_capacity[r, :S]
        assert (_bits(cap - det.memory_demand[r, :S]) == _bits(st[:S])).all()
    return got, det


@pytest.mark.gpu
@pytest.mark.parametrize('shape', ['bulk_then_chain', 'chain_only', 'replay', 'windows', 'device_listed'])
@pytest.mark.parametrize('name', TRANSCRIPT + ['het32_tight', 'rough_q10', 'rough_t3', 'lim_s128_l255'])
def test_api_misses(name, shape, workload_dir, monkeypatch):
    """misses=True: result.misses is the host build's (which equals the transcripts and the oracle) bit for bit, in
    reference order, whatever the schedule, the hand-over store (METIS_SAVE_SLOTS=40: later continuations replay their
    first attempt), windows or device listing; tuples, summary, best() and headroom are those of a search without
    misses; the counters satisfy the identity."""
    _gpu()
    from metis_b200 import api
    api.release_engines()
    _schedule(monkeypatch, 2 ** 31 - 1 if shape == 'chain_only' else 1)
    if shape == 'replay':
        monkeypatch.setenv('METIS_SAVE_SLOTS', '40')
    if shape == 'windows':
        from test_windowed_search import _force_windows
        _force_windows(monkeypatch, 3)
    if shape == 'device_listed':
        monkeypatch.setattr(api, '_DEVICE_LISTING_COMPS', 0)
    inputs = _api_inputs(name, workload_dir)
    plain = _run(inputs, headroom=True)
    got = _run(inputs, headroom=True, misses=True)
    want, host_summary = _host_want(name, workload_dir, inputs)
    assert 'misses_s' in got.timings and 'misses_s' not in plain.timings
    s = dict(got.summary)
    assert s.pop('num_oom_attempts') == len(want)
    assert s == plain.summary
    assert list(got) == list(plain) and got.best() == plain.best()
    assert (_bits(got.headroom) == _bits(plain.headroom)).all()
    assert _result_tuples(got) == want
    assert s['num_balancer_runs'] == s['num_records'] + s['num_keyerror'] + len(want)
    if shape == 'windows':
        assert s['num_windows'] > 1
    if shape == 'device_listed':
        assert s['listing'] == 'device'
    if want:
        _check_views(got)
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['c3_homo64_mpl6', 'c4_het128'])
def test_whole_space_misses(name, workload_dir):
    """Every out-of-memory attempt of C3-mpl6 and C4: the identity of the counters, deficits > 0, closest_misses(k) the
    lexsort's, and the replayed state minima equal to the recorded deficits."""
    _gpu()
    from metis_b200 import api
    api.release_engines()
    res = _run(_api_inputs(name, workload_dir), misses=True)
    s, m = res.summary, res.misses
    assert s['num_oom_attempts'] == len(m) and s['num_balancer_runs'] == s['num_records'] + s['num_keyerror'] + len(m)
    assert len(m) > 0 and (m.deficit > 0).all() and (m.stage < m.num_stage).all()
    key = list(zip(m.ordinal.tolist(), m.call.tolist(), m.attempt.tolist()))
    assert key == sorted(key) and len(set(key)) == len(key)
    order = np.lexsort((np.arange(len(m)), m.deficit))
    assert (res._closest_order() == order).all()
    _check_views(res, 100)
    api.release_engines()


@pytest.mark.gpu
def test_infeasible_cluster_on_the_gpu(workload_dir, tmp_path_factory):
    """Nothing fits: the result is empty; the misses, the closest miss and its detail are the oracle's."""
    _gpu()
    from metis_b200 import api
    api.release_engines()
    root, meta, w = infeasible_inputs(workload_dir, str(tmp_path_factory.mktemp('infeasible') / 'w'))
    res = _run(_api_inputs(None, workload_dir, root=root, meta=meta, w=w), misses=True)
    assert len(res) == 0
    _c, _counters, want = _oracle_misses(None, workload_dir, root=root, meta=meta, w=w)
    assert _result_tuples(res) == _oracle_tuples(want)
    o = want[min(range(len(want)), key=lambda i: (want[i].deficit, i))]
    (_ns, groups, strategies, _batches, part, attempt, deficit, stage), = res.closest_misses(1)
    assert (strategies, list(part), attempt, _bits(deficit), stage) == (
        [tuple(x) for x in o.strategies], list(o.partition), o.attempt, _bits(o.deficit), o.stage)
    assert [g // dp // tp for g, (dp, tp) in zip(groups, strategies)] == [1] * len(groups)
    det = res.miss_detail(res._closest_order()[:1])
    S = len(o.state)
    for f, v in (('performance', o.performance), ('memory_capacity', o.capacity), ('memory_demand', o.demand),
                 ('memory_state', o.state)):
        assert (_bits(getattr(det, f)[0, :S]) == _bits([float(x) for x in v])).all(), f
    api.release_engines()



GATHER_WORKER = r'''
import os, sys
sys.path.insert(0, os.environ['REPO'])
import numpy as np
import torch, torch.distributed as dist
dist.init_process_group('gloo', init_method='tcp://127.0.0.1:' + os.environ['PORT'],
                        rank=int(os.environ['RANK']), world_size=2)
from metis_b200 import search
rank = dist.get_rank()
n = 5 if rank == 0 else 0 if os.environ['EMPTY'] == '1' else 3
m = np.zeros(n, dtype=search.MISS_HOST_DTYPE)
m['ordinal'] = np.arange(n) * 2 + rank                   # interleaved shards of one space
m['call'] = rank
m['attempt'] = 1 + np.arange(n) % 3
m['deficit'] = m['ordinal'] + 0.5
got = search.gather_misses(m, 'cpu')
assert len(got) == (8 if os.environ['EMPTY'] != '1' else 5)
key = list(zip(got['ordinal'].tolist(), got['call'].tolist(), got['attempt'].tolist()))
assert key == sorted(key) and (got['deficit'] == got['ordinal'] + 0.5).all() and (got['call'] == got['ordinal'] % 2).all()
dist.barrier(); dist.destroy_process_group()
print('rank', rank, 'ok')
'''


@pytest.mark.parametrize('empty', [False, True], ids=['both_ranks', 'one_rank_empty'])
def test_two_rank_gather_misses(tmp_path, empty):
    """world size 2 over gloo: gather_misses (used by gather_records for one search and by gather_window_records)
    gives every rank every rank's misses in the reference's order, also when one rank has none."""
    import socket
    import sys
    script = tmp_path / 'gather.py'
    script.write_text(GATHER_WORKER)
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    repo = os.path.dirname(HERE)
    procs = [subprocess.Popen([sys.executable, str(script)],
                              env=dict(os.environ, REPO=repo, RANK=str(r), PORT=str(port), EMPTY=str(int(empty))),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=300)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), '\n'.join(outs)


@pytest.mark.gpu
@pytest.mark.parametrize('split', [False, True], ids=['one_search', 'windows'])
def test_multi_rank_gather_carries_misses(split, workload_dir, monkeypatch):
    """With torch.distributed initialised (NCCL, a world of one rank) cost_het_cluster(..., misses=True) takes the
    multi-rank path: gather_records (one search) or gather_window_records (windows).  The misses, their count and the
    views equal the single-process result's."""
    import socket
    torch = _gpu()
    import torch.distributed as dist
    from metis_b200 import api
    api.release_engines()
    inputs = _api_inputs('c2_het16', workload_dir)
    want = _run(inputs, misses=True)
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
        got = _run(inputs, misses=True)
    finally:
        dist.destroy_process_group()
        api.release_engines()
    assert (got.summary['num_windows'] > 1) == split
    if not split:
        assert got.summary['records_per_rank'] == [len(want)]   # the gather path ran
    assert got.summary['num_oom_attempts'] == want.summary['num_oom_attempts'] == len(want.misses) == 2953
    assert _result_tuples(got) == _result_tuples(want)
    assert list(got) == list(want)
    assert got.closest_misses(3) == want.closest_misses(3)
