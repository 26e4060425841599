"""Windowed het search: a plan space walked in ordinal windows, each a MetisPlanSpace of its own
(flatten.plan_windows), must give what one search of the whole space gives.

CPU: the window planner on golden-sized spaces (coverage, ordinal -> plan, rows) and the 512-GPU space, and the
windowed orchestration through the host build of the evaluator.  GPU (-m gpu): forced small windows through
api.cost_het_cluster against the one-window result and the goldens, and the 512-GPU / 1-type / variance-0 / mpl-4
space (1.5e9 plans, 10.5 GiB of rows) against the pinned oracle.
"""
import ctypes as C
import itertools
import math
import os
import random

import numpy as np
import pytest

import hostsim_util as hs
from conftest import C1_DIR, golden_rows, load_golden
from metis_b200 import flatten, native


def _lib_or_skip():
    try:
        return native.load_library()
    except native.MetisNativeError as e:
        pytest.skip(str(e))


def _space_args(w):
    """(node sequences, devices, gbs, layers, variance, mpl) of a workload's plan space."""
    return (math.factorial(len(w.device_types())), sum(n for _, n in w.nodes), w.gbs, w.num_layers, w.variance,
            w.max_permute_len)


def _host_rows(space: flatten.FlatPlanSpace) -> np.ndarray:
    """A device_rows space's row blob, written on the host by the row kernel's code (metis_rows.cuh)."""
    rows = np.zeros(max(int(space.rows_total_bytes), 16), dtype=np.uint8)
    rc = hs.hostsim().hostsim_generate_rows(C.c_void_p(space.comp_recs.ctypes.data), C.c_int64(len(space.comp_recs)),
                                            C.c_void_p(space.comp_pool.ctypes.data), C.c_void_p(rows.ctypes.data))
    assert rc == 0
    return rows


def _max_slice_plans(space):
    return int(space.comp_recs['num_rows'].max()) * len(space.batches)


def _split(space, parts):
    """Windows of about 1/parts of the plans each (the budget counts plans only); parts=0: one window per slice."""
    if parts == 0:
        return flatten.plan_windows(space, 0)
    return flatten.plan_windows(space, -(-space.num_plans // parts) + _max_slice_plans(space))


def _check_windows(space, windows, samples=200, seed=0):
    # every ordinal exactly once, in order
    base = 0
    for w in windows:
        assert w.base == base and w.space.num_plans > 0
        assert flatten.fits_one_search(w.space)
        assert (np.diff(w.space.blocks['first_ordinal']) > 0).all()
        base += w.space.num_plans
    assert base == space.num_plans
    # ordinal -> plan through the windows == through the whole space; window rows == the host enumerator's tables
    full = space.tables
    rng = random.Random(seed)
    bases = np.asarray([w.base for w in windows], dtype=np.int64)
    picks = {rng.randrange(space.num_plans) for _ in range(samples)}
    for w in windows:
        picks |= {w.base, w.base + w.space.num_plans - 1}
    rows_of = {}
    for o in sorted(picks):
        k = int(np.searchsorted(bases, o, side='right')) - 1
        if k not in rows_of:
            rows_of = {k: _host_rows(windows[k].space)}
        got = windows[k].locate(o, rows_of[k])
        want = space.locate(o)
        assert got[:4] == want[:4], (o, got, want)
        assert (got[4] == want[4]).all(), o
    for w in windows:
        rows = _host_rows(w.space)
        for b, blk in enumerate(w.space.blocks):
            S, n, at = int(blk['num_stage']), int(blk['num_rows']), int(blk['rows_offset'])
            _, table = full[S]
            r0 = int(w.row_base[b])
            assert (rows[at:at + n * S].reshape(n, S) == table[r0:r0 + n]).all(), (w.base, b)


PLANNER_SPACES = {
    'c3_mpl4': ('c3_homo64_mpl4', ()), 'c3_mpl6': ('c3_homo64_mpl6', ()), 'c4': ('c4_het128', ()),
    'c4_mpl6': ('c4_het128_mpl6', ()), 'q1_corrected': ('c4_het128', ('Q1',)), 'sweep_n32_t4': ('sweep_n32_t4', ()),
    'sweep_n256_t2_v0': ('sweep_n256_t2_v0', ()),
}


@pytest.mark.parametrize('parts', [2, 7, 0], ids=['two', 'seven', 'per_slice'])
@pytest.mark.parametrize('key', list(PLANNER_SPACES))
def test_window_planner_covers_the_space(key, parts):
    """Windows cover every ordinal once, in order; ordinal -> plan and rows through the windows equal the whole space's
    (the Q1 blocks of later node sequences and shared stage counts included)."""
    from metis_b200.workloads import WORKLOADS
    _lib_or_skip()
    name, corrected = PLANNER_SPACES[key]
    space = flatten.build_device_plan_space(*_space_args(WORKLOADS[name]), corrected=corrected)
    if parts == 0 and len(space.comp_recs) > 20000:
        pytest.skip('one window per slice: kept to the smaller spaces')
    windows = _split(space, parts)
    if parts:
        assert len(windows) == parts
    else:
        assert len(windows) == sum(int((space.comp_recs['stages'] == b['num_stage']).sum()) for b in space.blocks)
    _check_windows(space, windows)


def test_window_planner_shares_rows_between_node_sequences():
    """A window that covers a stage count for several node sequences holds its rows once."""
    from metis_b200.workloads import WORKLOADS
    _lib_or_skip()
    space = flatten.build_device_plan_space(*_space_args(WORKLOADS['c4_het128']))
    (w,) = flatten.plan_windows(space, space.num_plans)
    assert len(space.blocks) > len(np.unique(space.blocks['num_stage']))
    assert w.space.rows_total_bytes == sum(int(n) * int(s) for s, n in
                                           {int(b['num_stage']): int(b['num_rows']) for b in space.blocks}.items())
    assert len(w.space.comp_recs) == int(np.isin(space.comp_recs['stages'], space.blocks['num_stage']).sum())


def test_window_planner_512_gpus():
    """BASELINE configs[4], 512 GPUs / 1 type / variance 0 / mpl 4: 1.5e9 plans over 10.5 GiB of rows (beyond one
    search).  With an 80 GB-class budget every window stays below 2^32 plans and 4 GiB of rows, and one arena sized
    for all windows fits the budget.  Ordinal -> plan through the windows (every window's first and last plan and
    seeded samples, rows past 4 GiB of the whole space included) equals the whole space's block list and the host
    enumerator's table of the stage count (metis_enum_device_groups)."""
    _lib_or_skip()
    space = flatten.build_device_plan_space(1, 512, 512, 96, 0, 4)
    assert space.num_plans == 1473825430 and space.rows_total_bytes > 0xFFFFFFFF
    assert not flatten.fits_one_search(space)
    with pytest.raises(NotImplementedError):
        flatten.build_plan_space(1, 512, 512, 96, 0, 4, device_rows=True)
    model = (56.5, 1.25, 20.0)
    budget = 60e9
    windows = flatten.plan_windows(space, budget, *model)
    assert len(windows) >= 3
    assert flatten.arena_bytes(windows, *model) <= budget
    base = 0
    for w in windows:
        assert w.base == base
        assert w.space.num_plans <= flatten.MAX_SEARCH_PLANS
        assert w.space.rows_total_bytes <= flatten.MAX_SEARCH_ROW_BYTES
        assert flatten.window_bytes(w.space, *model) <= budget
        base += w.space.num_plans
    assert base == space.num_plans
    rng = random.Random(512)
    picks = {rng.randrange(space.num_plans) for _ in range(40)}
    for w in windows:
        picks |= {w.base, w.base + w.space.num_plans - 1}
    ndiv = len(space.batches)
    firsts = space.blocks['first_ordinal']
    by_stage = {}
    for o in sorted(picks):
        blk = space.blocks[int(np.searchsorted(firsts, o, side='right')) - 1]
        row, div = divmod(o - int(blk['first_ordinal']), ndiv)
        want = (int(blk['ns_idx']), int(blk['label_stage']), row, int(space.batches[div]))
        got = _window_plan(windows, o)
        assert got[:4] == want, (o, got[:4], want)
        by_stage.setdefault(int(blk['num_stage']), []).append((o, row, got[4]))
    assert max(by_stage) >= 90                                # window boundaries deep in the space (rows past 4 GiB)
    for S, items in by_stage.items():
        table = flatten.enumerate_device_groups(S, 512, 0, 4)
        for o, row, codes in items:
            assert (codes == table[row]).all(), (o, S, row)


# ---- orchestration through the host build --------------------------------------------------------------------------
ORCH = ['c1_het', 'mix32', 'het32_tight', 'fatal_gbs96', 'q10_big_first', 'q10_small_first', 'q10_small_first_t1']


def _inputs(name, workload_dir):
    if name == 'c1_het':
        meta, _ = load_golden('c1_het')
        cfg = dict(L=10, hidden=4096, seq=1024, vocab=51200, gbs=128, variance=1, mpl=4, max_tp=4, max_bs=4)
        root, sub = C1_DIR, 'profile_data_samples'
    else:
        meta, _ = load_golden(name)
        w, root, _ = workload_dir(name)
        cfg = dict(L=w.num_layers, hidden=w.hidden_size, seq=w.sequence_length, vocab=w.vocab_size, gbs=w.gbs,
                   variance=w.variance, mpl=w.max_permute_len, max_tp=w.max_tp, max_bs=w.max_bs)
        sub = 'profile'
    cluster, profile, _, mc = hs.load_inputs(root, sub, meta['file_order'], cfg['L'], cfg['hidden'], cfg['seq'],
                                             cfg['vocab'])
    seqs = [tuple(s) for s in meta['node_sequences']]
    problem = flatten.build_problem(profile, cluster, mc, cfg['gbs'], cfg['max_tp'], cfg['max_bs'], seqs)
    args = (len(seqs), cluster.get_total_num_devices(), cfg['gbs'], cfg['L'], cfg['variance'], cfg['mpl'])
    return problem, args


def _summary_dict(s):
    return dict(num_records=int(s.num_records), num_partition_calls=int(s.num_partition_calls),
                num_balancer_runs=int(s.num_balancer_runs), num_keyerror=int(s.num_keyerror),
                fatal_ordinal=int(s.fatal_ordinal), fatal_code=int(s.fatal_code), fatal_aux=int(s.fatal_aux))


def _sorted(rec, det):
    order = np.lexsort((rec['step'], rec['ordinal']))
    return rec[order], det[order]


@pytest.mark.parametrize('parts', [2, 7, 0], ids=['two', 'seven', 'per_slice'])
@pytest.mark.parametrize('name', ORCH)
def test_windowed_host_search_equals_one_search(name, parts, workload_dir):
    """Each window searched by the host build (hostsim_util.host_het_search) and merged by search.WindowMerge: records
    (with global ordinals), their order, detail rows, best, counters and the fatal plan equal one search of the whole
    space, bit for bit."""
    from metis_b200 import search
    _lib_or_skip()
    problem, args = _inputs(name, workload_dir)
    whole = flatten.build_plan_space(*args)
    rec1, det1, s1 = hs.host_het_search(problem, whole, mode=1)
    rec1, det1 = _sorted(rec1, det1)
    one = _summary_dict(s1)

    space = flatten.build_device_plan_space(*args)
    windows = _split(space, parts)
    assert len(windows) > 1 or space.num_plans <= _max_slice_plans(space)
    merge = search.WindowMerge(len(windows))
    details = []
    for w in windows:
        ws = flatten.FlatPlanSpace(w.space.num_plans, w.space.blocks, w.space.batches, _host_rows(w.space))
        rec, det, s = hs.host_het_search(problem, ws, mode=1)
        rec, det = _sorted(rec, det)
        b = s.best
        best = (float(b.cost), int(b.ordinal), int(b.step), int(b.num_repartition), int(b.num_stage)) \
            if s.num_records else None
        details.append(det)
        if merge.add(w.base, _summary_dict(s), best, rec):
            break
    out = merge.result()
    assert out.summary['fatal_ordinal'] == one['fatal_ordinal']
    if one['fatal_ordinal'] != 2 ** 64 - 1:
        assert (out.summary['fatal_code'], out.summary['fatal_aux']) == (one['fatal_code'], one['fatal_aux'])
        assert out.summary['windows_searched'] <= len(windows)
        return
    assert out.summary['windows_searched'] == len(windows) == out.summary['num_windows']
    for k in ('num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror'):
        assert out.summary[k] == one[k], k
    rec = out.records
    win = np.searchsorted(out.firsts, np.arange(len(rec)), side='right') - 1
    glob = out.bases[win] + rec['ordinal'].astype(np.int64)
    assert len(rec) == len(rec1)
    assert (glob == rec1['ordinal'].astype(np.int64)).all()
    assert (rec['step'] == rec1['step']).all() and (rec['num_repartition'] == rec1['num_repartition']).all()
    assert (rec['num_stage'] == rec1['num_stage']).all()
    assert (rec['cost'].view(np.uint64) == rec1['cost'].view(np.uint64)).all()
    assert (np.concatenate(details) == det1).all()
    b = s1.best
    if s1.num_records:
        assert out.best == (float(b.cost), int(b.ordinal), int(b.step), int(b.num_repartition), int(b.num_stage))
    else:
        assert out.best is None


WORKER = r'''
import os, sys
sys.path.insert(0, os.environ['REPO']); sys.path.insert(0, os.path.join(os.environ['REPO'], 'tests'))
import torch, torch.distributed as dist
dist.init_process_group('gloo', init_method='tcp://127.0.0.1:' + os.environ['PORT'],
                        rank=int(os.environ['RANK']), world_size=2)
import tempfile
import numpy as np
import hostsim_util as hs
from conftest import load_golden
from test_windowed_search import _host_rows
from metis_b200 import flatten, search
from metis_b200.workloads import WORKLOADS, materialize
name = os.environ['NAME']
meta, _ = load_golden(name)
w = WORKLOADS[name]
root = tempfile.mkdtemp(); materialize(w, root)
cluster, profile, _, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size)
seqs = [tuple(s) for s in meta['node_sequences']]
problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
args = (len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance, w.max_permute_len)
rank = dist.get_rank()
# the whole space in one search on one rank: what the two ranks' windowed search must give
rec1, det1, s1 = hs.host_het_search(problem, flatten.build_plan_space(*args), mode=1)
rec1 = rec1[np.lexsort((rec1['step'], rec1['ordinal']))]
space = flatten.build_device_plan_space(*args)
# the ranks see different free memory: the agreed budget (the smaller) cuts the same windows on both
local = space.num_plans // 3 if rank == 0 else space.num_plans // 7
budget = search.agree_budget(local, 'cpu')
assert budget == space.num_plans // 7
windows = flatten.plan_windows(space, budget)
assert len(windows) >= 7
merge = search.WindowMerge(len(windows))
for win in windows:                                            # the shard of each window: test shim for the GPU search
    ws = flatten.FlatPlanSpace(win.space.num_plans, win.space.blocks, win.space.batches, _host_rows(win.space))
    rec, _, s = hs.host_het_search(problem, ws, rank=rank, world=2, tile=64, mode=1)
    rec = rec[np.lexsort((rec['step'], rec['ordinal']))]
    b = s.best
    best = (float(b.cost), int(b.ordinal), int(b.step), int(b.num_repartition), int(b.num_stage)) if s.num_records else None
    merge.add(win.base, dict(num_records=int(s.num_records), num_partition_calls=int(s.num_partition_calls),
                             num_balancer_runs=int(s.num_balancer_runs), num_keyerror=int(s.num_keyerror),
                             fatal_ordinal=int(s.fatal_ordinal), fatal_code=int(s.fatal_code), fatal_aux=int(s.fatal_aux)),
              best, rec)
merged = merge.result()
summary, best = search.global_exchange(merged.summary, merged.best, 'cpu')   # the product's multi-rank steps
assert summary['global_fatal_ordinal'] == 2 ** 62
out = search.gather_window_records(merged, 'cpu')
glob = out.bases[np.searchsorted(out.firsts, np.arange(len(out.records)), side='right') - 1] + out.records['ordinal'].astype(np.int64)
assert len(out.records) == len(rec1) == int(s1.num_records)
assert (glob == rec1['ordinal'].astype(np.int64)).all() and (out.records['step'] == rec1['step']).all()
assert (out.records['cost'].view(np.uint64) == rec1['cost'].view(np.uint64)).all()
for k in ('num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror'):
    assert summary[k] == int(getattr(s1, k)), k
b = s1.best
assert best[:3] == (float(b.cost), int(b.ordinal), int(b.step)), best
dist.barrier(); dist.destroy_process_group()
print('rank', rank, 'ok')
'''


@pytest.mark.parametrize('name', ['c2_v100', 'het32_tight'])
def test_two_rank_windowed_search_gloo(name, tmp_path):
    """world_size 2 over gloo, ranks with different free memory: the agreed budget (search.agree_budget) gives both
    ranks the same windows; each rank searches its shard of every window (host build), and the product's exchange
    (search.global_exchange) and record gather (search.gather_window_records) give every rank the one-search result:
    records in order, counters and best."""
    import socket
    import subprocess
    import sys
    _lib_or_skip()
    load_golden(name)
    hs.hostsim()                                             # build the test shim once, before the ranks start
    script = tmp_path / 'worker.py'
    script.write_text(WORKER)
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(os.environ, REPO=repo, RANK=str(r), PORT=str(port),
                                                                      NAME=name),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=300)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), '\n'.join(outs)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()
    return torch


def _api_call(name, root, meta, w):
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), meta['file_order']).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                      vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
    args = parse_args(['--gbs', str(w.gbs), '--num_layers', str(w.num_layers), '--max_profiled_tp_degree',
                       str(w.max_tp), '--max_profiled_batch_size', str(w.max_bs), '--min_group_scale_variance',
                       str(w.variance), '--max_permute_len', str(w.max_permute_len)])
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    seqs = [tuple(s) for s in meta['node_sequences']]

    def run():
        return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                    api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                                    device='cuda:0')
    return run


def _force_windows(monkeypatch, parts):
    """Make cost_het_cluster window a space of any size into about ``parts`` windows (the budget is not a user
    option: it comes from the free device memory)."""
    from metis_b200 import api, search
    monkeypatch.setattr(api, '_ONE_SEARCH_BYTES', 0)
    monkeypatch.setattr(api, '_MIN_WINDOW_BYTES', 0)
    monkeypatch.setattr(api, '_engine_bytes', lambda key: 0)  # a cached engine's buffers would count as free memory
    real = flatten.plan_windows

    def plan(space, budget, plan_bytes=1.0, row_bytes=0.0, rec_bytes=0.0):
        return real(space, space.num_plans / parts * plan_bytes + space.rows_total_bytes * row_bytes
                    + len(space.comp_recs) * rec_bytes + _max_slice_plans(space) * plan_bytes, plan_bytes,
                    row_bytes, rec_bytes)
    monkeypatch.setattr(flatten, 'plan_windows', plan)
    monkeypatch.setattr(search, 'window_budget', lambda dev, fixed: 0.0)


@pytest.mark.gpu
def test_one_search_space_keeps_the_cached_engine(workload_dir, monkeypatch):
    """A space that fits one search takes the one-search path even when its size makes cost_het_cluster() ask the
    device for free memory (forced here for a small space): the cached engine and its buffers are reused, not
    dropped and allocated again."""
    _gpu()
    from metis_b200 import api
    meta, _ = load_golden('c3_homo64_mpl4')
    w, root, _ = workload_dir('c3_homo64_mpl4')
    run = _api_call('c3_homo64_mpl4', root, meta, w)
    api.release_engines()
    first = run()
    (eng,) = api._ENGINES.values()
    buffers = (eng[0]._dev.data_ptr(), eng[1].workspace.data_ptr(), eng[1].records.data_ptr())
    monkeypatch.setattr(api, '_ONE_SEARCH_BYTES', 0)
    again = run()
    assert first.summary['num_windows'] == again.summary['num_windows'] == 1
    (eng2,) = api._ENGINES.values()
    assert eng2 is eng and (eng[0]._dev.data_ptr(), eng[1].workspace.data_ptr(), eng[1].records.data_ptr()) == buffers
    assert (again.costs.view(np.uint64) == first.costs.view(np.uint64)).all()
    api.release_engines()


@pytest.mark.gpu
def test_forced_windows_fatal_plan(workload_dir, monkeypatch):
    """fatal_gbs96 (the reference aborts with KeyError 'tp1_bs3', quirk Q8): the windowed search reports the same
    global fatal ordinal, code and key as one search and the golden, and cost_het_cluster() raises the same KeyError."""
    _gpu()
    from metis_b200 import search
    meta, _ = load_golden('fatal_gbs96')
    w, root, _ = workload_dir('fatal_gbs96')
    run = _api_call('fatal_gbs96', root, meta, w)
    with pytest.raises(KeyError) as one:
        run()
    cluster, profile, _, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                              w.sequence_length, w.vocab_size)
    seqs = [tuple(s) for s in meta['node_sequences']]
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
    space = flatten.build_device_plan_space(*_space_args(w))
    whole = search.HetSearcher(search.DeviceProblem(problem, space, 'cuda:0')).run().summary
    windows = flatten.plan_windows(space, 0)                  # one window per slice
    assert len(windows) > 1
    merged, _, _ = search.search_windows(problem, windows, 'cuda:0')
    s = merged.summary
    assert s['fatal_ordinal'] == whole['fatal_ordinal'] == meta['fatal'][0]
    assert (s['fatal_code'], s['fatal_aux']) == (whole['fatal_code'], whole['fatal_aux']) == (1, 0 << 16 | 3)
    _force_windows(monkeypatch, 4)
    with pytest.raises(KeyError) as win:
        run()
    assert str(win.value) == str(one.value)


@pytest.mark.gpu
@pytest.mark.parametrize('name,factor', [('c3_homo64_mpl4', 1), ('c3_homo64_mpl4', 2 ** 31 - 1), ('c4_het128', 0)],
                         ids=['c3_bulk_round_then_chains', 'c3_chain_kernel_only', 'c4_default'])
def test_forced_windows_through_the_api(name, factor, workload_dir, monkeypatch):
    """cost_het_cluster() with forced small windows equals the one-window result in the same schedule (c3: both
    schedules forced in turn through MetisShard.reserved): len, every tuple, ranked(), best(), counters; and the
    goldens (c4_het128: every candidate of its reference-sampled ordinals)."""
    _gpu()
    from metis_b200 import api
    meta, arr = load_golden(name)
    w, root, _ = workload_dir(name)
    run = _api_call(name, root, meta, w)
    shard = native.MetisShard
    monkeypatch.setattr(native, 'MetisShard', lambda rank, world, tile, _r: shard(rank, world, tile, factor))
    api.release_engines()                                     # a cached engine would keep its own schedule
    ref = run()
    assert ref.summary['num_windows'] == 1
    _force_windows(monkeypatch, 5)
    got = run()
    monkeypatch.undo()                                        # the ranking below sizes its sort from the real budget
    api.release_engines()
    assert got.summary['num_windows'] >= 3 and got.summary['windows_searched'] == got.summary['num_windows']
    for k in ('num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror'):
        assert got.summary[k] == ref.summary[k], k
    assert len(got) == len(ref)
    assert (got.costs.view(np.uint64) == ref.costs.view(np.uint64)).all()
    assert got.best() == ref.best()
    assert got.ranked(50) == ref.ranked(50)
    assert got.summary['ranking'] == 'device'
    if 'sample' not in arr:
        assert list(got) == list(ref)
        assert got.ranked() == ref.ranked()
        gold = [(tuple(meta['node_sequences'][g[2]]), g[3], g[4], g[5], g[6], g[7], g[8]) for g in golden_rows(arr)]
        assert got == gold
    else:
        idx = np.linspace(0, len(ref) - 1, 3000).astype(np.int64)
        assert got.candidates.tuples(idx) == ref.candidates.tuples(idx)
        assert got[-3:] == ref[-3:] and got[0] == ref[0]
        cand = got.candidates
        rec = cand.records
        glob = cand.bases[np.searchsorted(cand.firsts, np.arange(len(rec)), side='right') - 1] + \
            rec['ordinal'].astype(np.int64)
        pick = np.nonzero(np.isin(glob, arr['sample']))[0]        # (ordinal, step) order, like the golden rows
        gold = golden_rows(arr)
        assert len(pick) == len(gold) == meta['counters']['C']
        assert glob[pick].tolist() == [g[0] for g in gold] and rec['step'][pick].tolist() == [g[1] for g in gold]
        mine = cand.tuples(pick)
        assert [m[1:] for m in mine] == [tuple(g[3:]) for g in gold]
        assert [m[0] for m in mine] == [tuple(meta['node_sequences'][g[2]]) for g in gold]


def _oracle_check(workload, root, order, space, windows, records, bases, firsts, cand, picks):
    """Every picked global ordinal: the windowed result's candidates equal the pinned oracle's, bit for bit."""
    from oracle import metis_oracle as orc
    w = workload
    ocl = orc.OracleCluster(root + '/hostfile', root + '/clusterfile.json')
    oprof, _ = orc.load_profile_dir(root + '/profile', order)
    omodel = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size, oprof['model']['parameters'])
    norm = orc.norm_layer_duration(oprof)
    win = np.searchsorted(firsts, np.arange(len(records)), side='right') - 1
    glob = bases[win] + records['ordinal'].astype(np.int64)
    seqs = list(itertools.permutations(w.device_types()))
    bad = []
    for o in picks:
        ns, label, rowi, batches, codes = _window_plan(windows, o)
        plan = {'ns_idx': ns, 'node_sequence': seqs[ns], 'dg_idx': rowi, 'device_groups': [1 << int(c) for c in codes],
                'num_stage': label, 'batches': batches, 'gbs': w.gbs}
        want, counters = [], {'A': 0, 'B': 0, 'C': 0, 'runs': 0, 'keyerr': 0}
        orc.het_evaluate_plan(oprof, ocl, omodel, norm, plan, o, w.num_layers, w.max_tp, w.max_bs, counters, want)
        idx = np.nonzero(glob == o)[0]
        mine = cand.tuples(idx) if len(idx) else []
        same = len(mine) == len(want) and all(
            (m[1], m[2], m[3], m[4], m[5]) == (x[3], x[4], x[5], x[6], x[7]) and m[6] == x[8] for m, x in zip(mine, want))
        if not same:
            bad.append(o)
    return bad


def _window_plan(windows, ordinal):
    """Global ordinal -> (ns_idx, label_stage, dg_idx, batches, codes), the row written on the host from the one
    composition slice that holds it (a whole window's rows are gigabytes)."""
    k = int(np.searchsorted([x.base for x in windows], ordinal, side='right')) - 1
    sp = windows[k].space
    ns, label, dg, batches, S, at = windows[k].plan_at(ordinal)
    recs = sp.comp_recs
    r = int(np.searchsorted(recs['row_offset'], at, side='right')) - 1
    one = recs[r:r + 1].copy()
    assert int(one['stages'][0]) == S and at < int(one['row_offset'][0]) + int(one['num_rows'][0]) * S
    base = int(one['row_offset'][0])
    one['row_offset'] = 0
    rows = np.zeros(int(one['num_rows'][0]) * S, dtype=np.uint8)
    rc = hs.hostsim().hostsim_generate_rows(C.c_void_p(one.ctypes.data), C.c_int64(1),
                                            C.c_void_p(sp.comp_pool.ctypes.data), C.c_void_p(rows.ctypes.data))
    assert rc == 0
    return ns, label, dg, batches, rows[at - base:at - base + S]


@pytest.mark.gpu
def test_512_gpus_one_type_variance0_mpl4(tmp_path):
    """BASELINE configs[4] at 512 GPUs / 1 type / variance 0 / mpl 4: 1.5e9 plans and 10.5 GiB of rows, beyond one
    search, complete on one GPU in windows.  Every window's first and last plan, and a seeded stratified sample (one
    row of every (node sequence, stage count) block with every divisor of gbs, plus uniform ordinals), equal the pinned
    oracle bit for bit.  There is no reference golden: the reference's generator cannot walk 1.5e9 ordinals."""
    torch = _gpu()
    import json
    import time
    from metis_b200 import api
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    from metis_b200.workloads import materialize, profile_file_order, sweep_workload
    from metis_b200.arguments import parse_args
    w = sweep_workload(512, 1, 0, 4)
    w.bss = (1, 2, 4, 8, 16)
    root = str(tmp_path)
    materialize(w, root)
    order = profile_file_order(w)
    cluster = GPUCluster(root + '/hostfile', root + '/clusterfile.json')
    profile, _ = ProfileDataLoader(root + '/profile', order).load_profile_data_all()
    cfg = ModelConfig('SYN', w.num_layers, w.sequence_length, w.vocab_size, w.hidden_size, 32)
    args = parse_args(['--gbs', str(w.gbs), '--num_layers', str(w.num_layers), '--max_profiled_tp_degree',
                       str(w.max_tp), '--max_profiled_batch_size', str(w.max_bs), '--min_group_scale_variance',
                       str(w.variance), '--max_permute_len', str(w.max_permute_len)])
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    seqs = list(itertools.permutations(w.device_types()))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    res = api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                               api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                               device='cuda:0')
    wall = time.perf_counter() - t0
    s = res.summary
    assert s['num_plans'] == 1473825430 and s['num_windows'] >= 3 and s['windows_searched'] == s['num_windows']
    assert s['fatal_ordinal'] == 2 ** 64 - 1
    best = res.best()
    cand = res.candidates
    space = flatten.build_device_plan_space(1, 512, w.gbs, w.num_layers, w.variance, w.max_permute_len)
    windows = cand.windows
    assert sum(x.space.num_plans for x in windows) == space.num_plans
    rng = random.Random(512)
    picks = set()
    for x in windows:
        picks |= {x.base, x.base + x.space.num_plans - 1}
    ndiv = len(space.batches)
    for blk in space.blocks:
        first, n = int(blk['first_ordinal']), int(blk['num_rows'])
        row = rng.randrange(n)
        picks |= {first + row * ndiv + d for d in range(ndiv)}
    picks |= {rng.randrange(space.num_plans) for _ in range(200)}
    if best is not None:
        picks.add(int(res._best_key[0]))
    bad = _oracle_check(w, root, order, space, windows, cand.records, cand.bases, cand.firsts, cand, sorted(picks))
    report = {'gpu': torch.cuda.get_device_name(0), 'wall_s': wall, 'num_windows': s['num_windows'],
              'peak_allocated_bytes': int(torch.cuda.max_memory_allocated()),
              'peak_reserved_bytes': int(torch.cuda.max_memory_reserved()),
              'counters': {k: s[k] for k in ('num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror')},
              'best': [best[6], best[3]] if best else None, 'best_key': list(res._best_key) if res._best_key else None,
              'checked_plans': len(picks), 'mismatches': bad[:20], 'timings': res.timings}
    out = os.environ.get('METIS_WINDOWED_REPORT')
    if out:
        with open(out, 'w') as fh:
            json.dump(report, fh, indent=1)
    print(json.dumps(report))
    assert not bad
