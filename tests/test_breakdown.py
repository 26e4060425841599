"""Cost breakdown of searched candidates (metis_het_breakdown / metis_homo_breakdown, HetSearchResult.breakdown,
api.cost_homo_breakdown): the cost terms of HeteroCostEstimator.get_cost and the memory headroom of the accepted
partition attempt, replayed on the GPU for candidates a search returned.

CPU: the host build of the breakdown evaluator (tests/hostsim/breakdown_sim.cpp) against the reference's printed
transcripts (bit for bit) and against the oracle's breakdown twins (tests/oracle_breakdown.py) on the rough, Q10 and
limit goldens and a corrected run, and the homogeneous breakdown against oracle.homo_cost.  GPU (-m gpu): the same through the C ABI and api, as one search
and forced into windows; whole-space invariants on C3-mpl6 and C4-mpl4; a breakdown taken after a later search.
"""
import ctypes as C
import gzip
import json
import os
import re
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
import oracle_breakdown as obd
from conftest import C1_DIR, GOLDEN, load_golden
from metis_b200 import flatten, native, search
from oracle import metis_oracle as orc

TRANSCRIPTS = ['c1', 'c2_het16', 'mix32']
# rough profiles, Q10 clusters, limit spaces (S = 128 and L = 255); together they hold retried candidates
# (num_repartition 2 and 3), Q1 blocks (label_stage 1 < num_stage) and mixed-type stages
ORACLE_GOLDENS = ['rough_mix2', 'rough_t3', 'rough_q10', 'rough_long_int', 'rough_keys', 'q10_big_first', 'het32_tight', 'lim_s64_l128_t2', 'lim_s128_t2', 'lim_s128_l255']
HOMO = ['c1_homo', 'rough_homo_homo', 'lim_s97_homo']
COST_FIELDS = ('stage_time', 'dp_cost', 'update_cost', 'pp_cost')
MEMORY_FIELDS = ('performance', 'memory_capacity', 'memory_demand', 'memory_state')
C1_ARGV = ['--num_layers', '10', '--gbs', '128', '--max_profiled_tp_degree', '4', '--max_profiled_batch_size', '4',
           '--min_group_scale_variance', '1', '--max_permute_len', '4', '--hidden_size', '4096',
           '--sequence_length', '1024', '--vocab_size', '51200', '--attention_head_size', '32']


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'breakdown_sim.cpp')
SIM_DEPS = [SIM_SRC, hs.SRC] + [os.path.join(HERE, '..', 'metis_b200', 'csrc', f)
                                for f in ('metis_eval.cuh', 'metis_coop.cuh', 'metis_trace.cuh', 'metis_rows.cuh')] + \
    [os.path.join(HERE, '..', 'include', 'metis_b200.h')]
_sim = []


def sim():
    """The g++ build of the breakdown (tests/hostsim/breakdown_sim.cpp) at the compiled limits, with hostsim.cpp's
    flags; one shared object, rebuilt when its sources change."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'libbreakdown_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', tmp,
                                   SIM_SRC])
            os.replace(tmp, out)                             # atomic: concurrent test processes may race
        lib = C.CDLL(out)
        lib.breakdown_sim_het.restype = C.c_int
        lib.breakdown_sim_homo.restype = C.c_int
        _sim.append(lib)
    return _sim[0]


def _host_breakdown(problem, space, records):
    """breakdown_sim_het of ``records`` (any order), like search.het_breakdown drives the device."""
    lib = sim()
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.host_rows())
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    sp = space.as_struct(lambda n: keep[n].ctypes.data)
    n = len(records)
    order = np.lexsort((records['step'], records['ordinal']))
    picks = np.ascontiguousarray(records[order])
    width = max(int(picks['num_stage'].max()), 1)
    raw = np.zeros(n, dtype=native.BREAKDOWN_DTYPE)
    st = np.full((n, native.BD_FIELDS, width), np.nan)
    assert lib.breakdown_sim_het(C.byref(p), C.byref(sp), C.c_void_p(picks.ctypes.data), C.c_int64(n),
                                 C.c_void_p(raw.ctypes.data), C.c_void_p(st.ctypes.data), C.c_int32(width)) == 0
    back = np.empty(n, dtype=np.int64)
    back[order] = np.arange(n)
    return search.Breakdown.from_raw(raw[back], st[back])


def _check_sum(bd, costs):
    """exec + fb_sync + update + dp + pp + batch generate, left to right, is the record's cost bit for bit."""
    t = bd.terms
    total = t[:, 0] + t[:, 1] + t[:, 2] + t[:, 3] + t[:, 4] + t[:, 5]
    assert (_bits(total) == _bits(costs)).all()


def _check_oracle(bd, want):
    """bd rows against obd.het_breakdowns entries, same order: every term and stage value bit for bit, NaN after."""
    assert len(bd) == len(want)
    for k, (_o, _s, _nrep, cost, terms, stages) in enumerate(want):
        assert (_bits(bd.terms[k]) == _bits(terms)).all(), (k, bd.terms[k], terms)
        S, costed = len(stages['memory_state']), len(stages['stage_time'])
        assert (bd.num_stage[k], bd.costed_stages[k]) == (S, costed)
        state = stages['memory_state']
        assert bd.min_headroom[k] == min(state) and bd.min_headroom_stage[k] == state.index(min(state))
        for f in MEMORY_FIELDS + COST_FIELDS:
            got = getattr(bd, f)[k]
            v = stages[f]
            assert (_bits(got[:len(v)]) == _bits([float(x) for x in v])).all(), (k, f, got[:len(v)], v)
            assert np.isnan(got[len(v):]).all(), (k, f)
    _check_sum(bd, [w[3] for w in want])


def _records(pairs):
    """(ordinal, step, num_stage, cost) tuples -> MetisRecord rows."""
    rec = np.zeros(len(pairs), dtype=native.RECORD_DTYPE)
    for i, (o, s, S, c) in enumerate(pairs):
        rec[i] = (c, o, s, 0, S)
    return rec


# ---- transcripts ----------------------------------------------------------------------------------------------------
def _transcript_inputs(name, workload_dir):
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.utils import DeviceType
    meta = json.load(open(os.path.join(GOLDEN, f'transcript_{name}.json')))
    if name == 'c1':
        root, sub, argv = C1_DIR, 'profile_data_samples', C1_ARGV
    else:
        w, root, digest = workload_dir(name)
        assert digest == meta['inputs_sha256']
        sub, argv = 'profile', w.cli_args(root)
    args = parse_args(argv)
    cluster, profile, _types, cfg = hs.load_inputs(root, sub, meta['file_order'], args.num_layers, args.hidden_size,
                                                   args.sequence_length, args.vocab_size)
    seqs = [tuple(DeviceType[t] for t in seq) for seq in meta['node_sequences']]
    return meta, args, cluster, profile, cfg, seqs, api


def _printed(name):
    """Per candidate of the reference's transcript: the printed cost terms and the stage_memory_capacity,
    stage_memory_demand and memory_state of the accepted attempt, as the text the reference printed."""
    text = gzip.open(os.path.join(GOLDEN, f'transcript_{name}.txt.gz'), 'rt').read().split('\n')
    out, cap, mem = [], None, None
    for line in text:
        if line.startswith('stage_memory_capacity: '):
            cap = line[len('stage_memory_capacity: '):]
        m = re.match(r'stage_memory_demand: (\[.*\]), memory_state: (\[.*\])$', line)
        if m:
            mem = m.groups()
        if line.startswith('execution_cost: '):
            terms = [kv.split(': ')[1] for kv in line.split(', ')]
            out.append((terms, cap, mem[0], mem[1]))
    return out


def _same_printed(values, printed_list):
    """repr of every value equals the printed token (an int token: the value is that integer)."""
    toks = [t.strip() for t in printed_list.strip('[]').split(',')] if isinstance(printed_list, str) else printed_list
    assert len(toks) == len(values)
    for v, t in zip(values, toks):
        if re.fullmatch(r'-?\d+', t):
            assert float(v).is_integer() and int(v) == int(t), (v, t)
        else:
            assert repr(float(v)) == t, (v, t)


def _check_transcript(name, bd):
    printed = _printed(name)
    assert len(bd) == len(printed) > 0
    for k, (terms, cap, demand, state) in enumerate(printed):
        _same_printed(bd.terms[k, :5], terms)
        S = int(bd.num_stage[k])
        _same_printed(bd.memory_capacity[k, :S], cap)
        _same_printed(bd.memory_demand[k, :S], demand)
        _same_printed(bd.memory_state[k, :S], state)


@pytest.mark.parametrize('name', TRANSCRIPTS)
def test_transcript_values_on_host(name, workload_dir):
    """Every candidate of the reference's transcript (output of the unmodified reference): the five printed cost terms
    and the capacity, demand and state of the accepted attempt are the host build's breakdown, repr for repr."""
    meta, args, cluster, profile, cfg, seqs, api = _transcript_inputs(name, workload_dir)
    problem, space, _ = api.het_problem(args, cluster, profile, cfg, None, seqs)
    rec, _det, _summary = hs.host_het_search(problem, space, mode=0, want_detail=False)
    rec = rec[np.lexsort((rec['step'], rec['ordinal']))]
    bd = _host_breakdown(problem, space, rec)
    _check_transcript(name, bd)
    _check_sum(bd, rec['cost'])


# ---- oracle, heterogeneous ------------------------------------------------------------------------------------------
def _golden_inputs(name, workload_dir, corrected=()):
    meta, arr = load_golden(name)
    w, root, digest = workload_dir(name)
    assert digest == meta['inputs_sha256']
    cluster, profile, _types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                   w.sequence_length, w.vocab_size)
    seqs = [tuple(s) for s in meta['node_sequences']]
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs, corrected=corrected)
    space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance,
                                     w.max_permute_len, corrected=corrected)
    return meta, arr, w, root, seqs, problem, space


def _sample_ordinals(arr, n=60):
    """Golden ordinals for the oracle: evenly spaced ones, and those of retried candidates and Q1 blocks."""
    o = arr['ordinal']
    pick = set(o[np.linspace(0, len(o) - 1, min(n, len(o))).astype(np.int64)].tolist())
    for mask in (arr['nrep'] == 2, arr['nrep'] == 3, arr['label_stage'] < arr['nstage']):
        pick |= set(o[mask][:15].tolist())
    return pick


def _oracle_want(w, root, meta, seqs, sample, corrected=()):
    ocl = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'), corrected=corrected)
    oprof, _ = orc.load_profile_dir(os.path.join(root, 'profile'), meta['file_order'])
    omodel = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size, oprof['model']['parameters'])
    return obd.het_breakdowns(oprof, ocl, omodel, seqs, w.gbs, w.num_layers, w.variance, w.max_permute_len, w.max_tp,
                              w.max_bs, plan_filter=sample.__contains__, corrected=corrected)


def test_oracle_twins_give_the_oracles_costs(workload_dir):
    """The breakdown twins walk the oracle's chain and split its cost: same candidates, same cost bits."""
    meta, arr, w, root, seqs, *_ = _golden_inputs('rough_t3', workload_dir)
    want = _oracle_want(w, root, meta, seqs, set(arr['ordinal'].tolist()))
    assert [(o, s, n) for o, s, n, *_ in want] == list(zip(arr['ordinal'].tolist(), arr['step'].tolist(),
                                                           arr['nrep'].tolist()))
    assert _bits([x[3] for x in want]).tolist() == _bits(arr['cost']).tolist()


@pytest.mark.parametrize('name', ORACLE_GOLDENS)
def test_host_breakdown_vs_oracle(name, workload_dir):
    """Sampled golden candidates: every term, every stage value, the minimum headroom and the stage counts of the host
    build's breakdown equal the oracle twins', at the compiled limits the breakdown kernel is built for."""
    meta, arr, w, root, seqs, problem, space = _golden_inputs(name, workload_dir)
    sample = _sample_ordinals(arr)
    want = _oracle_want(w, root, meta, seqs, sample)
    keep = np.isin(arr['ordinal'], list(sample))
    rec = _records(list(zip(arr['ordinal'][keep].tolist(), arr['step'][keep].tolist(), arr['nstage'][keep].tolist(),
                            arr['cost'][keep].tolist())))
    assert [(o, s) for o, s, *_ in want] == list(zip(rec['ordinal'].tolist(), rec['step'].tolist()))
    _check_oracle(_host_breakdown(problem, space, rec), want)
    # reversed picks: the breakdown sorts and groups them, and gives each row back in the order asked for
    _check_oracle(_host_breakdown(problem, space, rec[::-1].copy()), want[::-1])


def test_host_breakdown_covers_the_traps(workload_dir):
    """The goldens above reach what the breakdown must get right: retried candidates (2 and 3 attempts), Q1 blocks
    whose memory fields outnumber their cost fields, and Q10 clusters."""
    seen = set()
    for name in ORACLE_GOLDENS:
        _meta, arr = load_golden(name)
        seen |= {f'nrep{n}' for n in set(arr['nrep'].tolist())}
        if (arr['label_stage'] < arr['nstage']).any():
            seen.add('q1')
    assert {'nrep2', 'nrep3', 'q1'} <= seen


def test_host_breakdown_corrected_vs_oracle(workload_dir):
    """With corrected=('Q5', 'Q6') the demand and state follow MetisProblem.corrected: every candidate of a corrected
    host search against the corrected oracle twins."""
    fix = ('Q5', 'Q6')
    meta, _arr, w, root, seqs, problem, space = _golden_inputs('rough_q10', workload_dir, corrected=fix)
    rec, _det, _summary = hs.host_het_search(problem, space, mode=0, want_detail=False)
    rec = rec[np.lexsort((rec['step'], rec['ordinal']))]
    sample = set(rec['ordinal'][np.linspace(0, len(rec) - 1, 80).astype(np.int64)].tolist())
    rec = rec[np.isin(rec['ordinal'], list(sample))]
    want = _oracle_want(w, root, meta, seqs, sample, corrected=fix)
    assert [(o, s) for o, s, *_ in want] == list(zip(rec['ordinal'].tolist(), rec['step'].tolist()))
    _check_oracle(_host_breakdown(problem, space, rec), want)


# ---- oracle, homogeneous --------------------------------------------------------------------------------------------
def _homo_inputs(name, workload_dir):
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    meta, _arr = load_golden(name)
    if name == 'c1_homo':
        root, sub, argv = C1_DIR, 'profile_data_samples', C1_ARGV
    else:
        w, root, digest = workload_dir(name[:-len('_homo')])
        assert digest == meta['inputs_sha256']
        sub, argv = 'profile', w.cli_args(root)
    args = parse_args(argv)
    cluster, profile, types, cfg = hs.load_inputs(root, sub, meta['file_order'], args.num_layers, args.hidden_size,
                                                  args.sequence_length, args.vocab_size)
    ocl = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    oprof, otypes = orc.load_profile_dir(os.path.join(root, sub), meta['file_order'])
    omodel = orc.OracleModel(args.num_layers, args.hidden_size, args.sequence_length, args.vocab_size,
                             oprof['model']['parameters'])
    return args, cluster, profile, types, cfg, (oprof, ocl, omodel, otypes[0]), api


def _homo_want(oracle, plans):
    oprof, ocl, omodel, dev = oracle
    out = []
    for p in plans:
        try:
            out.append(obd.homo_breakdown(oprof, ocl, omodel, tuple(int(x) for x in p), dev))
        except KeyError:
            out.append(None)
    return out


@pytest.mark.parametrize('name', HOMO)
def test_homo_breakdown_on_host_vs_oracle(name, workload_dir):
    """HomoCostEstimator.get_cost's terms (summed to the cost bit for bit), per-stage memory and OOM flag."""
    args, cluster, profile, types, cfg, oracle, api = _homo_inputs(name, workload_dir)
    est = api.HomoCostEstimator(profile, cfg, None, cluster)
    plans, problem, table, type_id = api._homo_inputs(args, cluster, est, types[0])
    lib = sim()
    keep = dict(problem.arrays)
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    width = int(table[:, 1].max())
    terms = np.zeros((len(table), 6))
    mem = np.zeros((len(table), width))
    status = np.zeros(len(table), dtype=np.int32)
    assert lib.breakdown_sim_homo(C.byref(p), C.c_int32(type_id), C.c_void_p(table.ctypes.data),
                                  C.c_int64(len(table)), C.c_void_p(terms.ctypes.data), C.c_void_p(mem.ctypes.data),
                                  C.c_int32(width), C.c_void_p(status.ctypes.data)) == 0
    want = _homo_want(oracle, table)
    for k, x in enumerate(want):
        if x is None:
            assert status[k] == 1
            continue
        cost, smem, oom, _strs = x
        assert status[k] == (2 if oom else 0)
        t = terms[k]
        assert _bits(t[0] + t[1] + t[2] + t[3] + t[4] + t[5]) == _bits(cost)
        pp = int(table[k, 1])
        assert (_bits(mem[k, :pp]) == _bits([float(m) for m in smem])).all()
        assert np.isnan(mem[k, pp:]).all()


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()
    return torch


def _windows(monkeypatch, split):
    if split:
        from test_windowed_search import _force_windows
        _force_windows(monkeypatch, 3)


@pytest.mark.gpu
@pytest.mark.parametrize('split', [False, True], ids=['one_search', 'windows'])
@pytest.mark.parametrize('name', TRANSCRIPTS)
def test_transcript_values_through_the_api(name, split, workload_dir, monkeypatch):
    """Item 1 through api.cost_het_cluster + HetSearchResult.breakdown, as one search and forced into windows."""
    _gpu()
    meta, args, cluster, profile, cfg, seqs, api = _transcript_inputs(name, workload_dir)
    api.release_engines()
    _windows(monkeypatch, split)
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    res = api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                               api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                               device='cuda:0')
    assert (res.summary['num_windows'] > 1) == split
    bd = res.breakdown(slice(None))
    _check_transcript(name, bd)
    _check_sum(bd, res.costs)
    # an int, a reversed index array and ranked positions give the same rows
    one = res.breakdown(-1)
    assert len(one) == 1 and (_bits(one.terms[0]) == _bits(bd.terms[-1])).all()
    rev = np.arange(len(res))[::-1]
    back = res.breakdown(rev, per_stage=False)
    assert back.performance is None and (_bits(back.terms) == _bits(bd.terms[rev])).all()
    res.ranked(3)
    top = res.breakdown(res.rank_order[:3])
    assert (_bits(top.terms) == _bits(bd.terms[res.rank_order[:3]])).all()
    with pytest.raises(IndexError):
        res.breakdown([len(res)])
    api.release_engines()


def _api_run(name, workload_dir, corrected=()):
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    meta, arr = load_golden(name)
    w, root, _ = workload_dir(name)
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), meta['file_order']).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                      vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
    args = parse_args(w.cli_args(root))
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    seqs = [tuple(s) for s in meta['node_sequences']]
    return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                                device='cuda:0', corrected=corrected)


_WANT = {}


def _result_positions(res, want):
    """Positions of the oracle's (global ordinal, step) pairs in a result."""
    return np.array([res.candidates.index_of(o, s) for o, s, *_ in want], dtype=np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize('split', [False, True], ids=['one_search', 'windows'])
@pytest.mark.parametrize('name', ['rough_t3', 'rough_q10', 'q10_big_first', 'lim_s128_l255'])
def test_api_breakdown_vs_oracle(name, split, workload_dir, monkeypatch):
    """Item 2 through the api: sampled golden candidates against the oracle twins, one search and windows."""
    _gpu()
    from metis_b200 import api
    meta, arr, w, root, seqs, *_ = _golden_inputs(name, workload_dir)
    if name not in _WANT:                                     # the oracle once for both splits
        _WANT[name] = _oracle_want(w, root, meta, seqs, _sample_ordinals(arr, 12 if name.startswith('lim') else 40))
    want = _WANT[name]
    api.release_engines()
    _windows(monkeypatch, split)
    res = _api_run(name, workload_dir)
    assert (res.summary['num_windows'] > 1) == split
    _check_oracle(res.breakdown(_result_positions(res, want)), want)
    api.release_engines()


@pytest.mark.gpu
def test_api_breakdown_corrected_vs_oracle(workload_dir):
    """A corrected search's breakdown follows the corrected demand and state."""
    _gpu()
    from metis_b200 import api
    fix = ('Q5', 'Q6')
    meta, _arr, w, root, seqs, *_ = _golden_inputs('rough_q10', workload_dir)
    res = _api_run('rough_q10', workload_dir, corrected=fix)
    sample = set(res.candidates.records['ordinal'][np.linspace(0, len(res) - 1, 60).astype(np.int64)].tolist())
    want = _oracle_want(w, root, meta, seqs, sample, corrected=fix)
    _check_oracle(res.breakdown(_result_positions(res, want)), want)
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('name', HOMO)
def test_api_homo_breakdown_vs_oracle(name, workload_dir):
    """api.cost_homo_breakdown: the plans of cost_homo_cluster in its order, terms summing to its costs, per-stage
    memory, the reference's formatted strings and the OOM flag of oracle.homo_cost."""
    _gpu()
    args, cluster, profile, types, cfg, oracle, api = _homo_inputs(name, workload_dir)
    est = api.HomoCostEstimator(profile, cfg, None, cluster)
    costs = api.cost_homo_cluster(args, cluster, est, types[0], device='cuda:0')
    bd = api.cost_homo_breakdown(args, cluster, est, types[0], device='cuda:0')
    assert [p for p, _ in costs] == bd.plans
    want = _homo_want(oracle, [(p.dp, p.pp, p.tp, p.mbs, p.gbs) for p in bd.plans])
    t = bd.terms
    assert (_bits(t[:, 0] + t[:, 1] + t[:, 2] + t[:, 3] + t[:, 4] + t[:, 5]) == _bits([c for _, c in costs])).all()
    for k, (cost, smem, oom, strs) in enumerate(want):
        assert bd.oom[k] == oom and bd.stage_memory_str[k] == strs
        assert (_bits(bd.stage_memory[k, :len(smem)]) == _bits([float(m) for m in smem])).all()
        assert np.isnan(bd.stage_memory[k, len(smem):]).all()


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['c3_homo64_mpl6', 'c4_het128'])
def test_whole_space_invariants(name, workload_dir):
    """Every candidate of C3-mpl6 (273 688) and C4-mpl4: the terms summed left to right are the record's cost bit for
    bit, and the accepted attempt's headroom is never negative."""
    _gpu()
    from metis_b200 import api
    res = _api_run(name, workload_dir)
    bd = res.breakdown(slice(None), per_stage=False)
    _check_sum(bd, res.costs)
    assert (bd.min_headroom >= 0).all()
    assert (bd.num_stage > 0).all() and (bd.costed_stages <= bd.num_stage).all()
    if name == 'c3_homo64_mpl6':
        assert len(res) == 273688
    api.release_engines()


@pytest.mark.gpu
def test_breakdown_survives_a_later_search(workload_dir):
    """A result keeps its own problem tables and plan space: its breakdown is unchanged after cost_het_cluster() ran
    again on different inputs in the same cached engine."""
    _gpu()
    from metis_b200 import api
    api.release_engines()
    first = _api_run('rough_t3', workload_dir)
    before = first.breakdown(slice(None))
    other = _api_run('mix32', workload_dir)
    assert len(other) != len(first)
    after = first.breakdown(slice(None))
    for f in ('terms', 'min_headroom') + MEMORY_FIELDS + COST_FIELDS:
        a, b = getattr(before, f), getattr(after, f)
        assert ((_bits(a) == _bits(b)) | (np.isnan(a) & np.isnan(b))).all(), f
    _check_sum(after, first.costs)
    api.release_engines()
