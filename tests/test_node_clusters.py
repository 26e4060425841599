"""The search on clusters whose nodes of one device type differ in bandwidth and memory.

The reference reads a cluster's per-node values in four ways: the bandwidth inside one node is the type's first
hostfile node's (model/cluster_bandwidth.py:49-54, MetisProblem.type_bw_first), the bandwidth across nodes the smallest
of the type's nodes' (:56-68, type_bw_min), a stage's memory capacity the first clusterfile entry of the raw
instance_type string, whether the hostfile names it or not (gpu_cluster.py:47-50, type_memory), and the homogeneous
path hostfile node 0's values (node0_memory, node0_bandwidth).  Clusters with one clusterfile entry per type cannot tell
these apart; the node_* workloads (Workload.hosts / cluster_entries) can, and their goldens come from the unmodified
reference (tests/golden/make_golden.py).

CPU: the inputs discriminate (each per-node table, altered, changes the host build's records), the oracle and the
host build against the goldens, recost of mix32's candidates into node_bw_mix32's costs, breakdowns against the oracle
twins, every existing golden's input digest, and a seeded 60-cluster per-node fuzz against the oracle.  GPU (-m gpu):
the goldens through the C ABI and the api, recost, headroom and a 30-cluster fuzz.
"""
import glob
import json
import os
import random

import numpy as np
import pytest

import hostsim_util as hs
import test_breakdown as tb
import test_recost as trc
import test_rough_profiles as trp
from conftest import GOLDEN, golden_rows, load_golden
from metis_b200 import flatten
from metis_b200.workloads import WORKLOADS, node_entry, per_node
from oracle import metis_oracle as orc

# golden -> the instantiation the GPU picks
NODE = {
    'node_bw_mix32': (64, 128, False),
    'node_bw_t1': (64, 128, True),
    'node_mem_order': (64, 128, False),
    'node_q10': (64, 128, False),
    'node_homo': (64, 128, True),
}
MODES, MODE_IDS, NO_PLAN = trp.MODES, trp.MODE_IDS, trp.NO_PLAN


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def _host_candidates(problem, space, tier=None, mode=0):
    rec, det, summary = hs.host_het_search(problem, space, mode=mode, tier=tier or hs.LIMITS,
                                           capacity=max(1024, space.num_plans * 4))
    return hs.unpack_candidates(rec, det, space), summary


def _first_host_node_memory(cluster, name):
    """The memory of the type's first hostfile node: what type_memory would be if it were read by node."""
    first = next(i for i, n in cluster.nodes.items() if n.device_type.name == name)
    return float(cluster.get_device_memory(first))


# ---------------------------------------------------------------------------------------------------------------
# the generator
# ---------------------------------------------------------------------------------------------------------------
def _digested_goldens():
    """(golden file, workload) of every golden whose metadata holds the sha256 of its generated inputs."""
    out = []
    for path in sorted(glob.glob(os.path.join(GOLDEN, '*.npz'))):
        with np.load(path, allow_pickle=False) as z:
            meta = json.loads(str(z['meta']))
        if meta.get('inputs_sha256'):
            out.append((os.path.basename(path), meta['workload'], meta['inputs_sha256']))
    for path in sorted(glob.glob(os.path.join(GOLDEN, 'transcript_*.json'))):
        meta = json.load(open(path))
        if meta.get('inputs_sha256'):
            out.append((os.path.basename(path), meta['workload'], meta['inputs_sha256']))
    return out


def test_every_golden_digest_matches_its_inputs(workload_dir):
    """materialize writes, byte for byte, the inputs every golden was made from: clusters given per type are written
    as before the per-node fields existed."""
    seen = _digested_goldens()
    assert len(seen) >= 50 and {'mix32.npz', 'node_bw_mix32.npz', 'transcript_mix32.json'} <= {f for f, *_ in seen}
    for fname, name, digest in seen:
        assert workload_dir(name)[2] == digest, fname


def test_per_node_files(workload_dir):
    """A per-node workload's hostfile keeps the slot count at character 6 of its second field and its clusterfile the
    given entry order, unused entries included; a host without a matching entry is refused."""
    w, root, _ = workload_dir('node_mem_order')
    lines = open(os.path.join(root, 'hostfile')).read().splitlines()
    assert [ln.split(' ')[0] for ln in lines] == ['N1', 'N2', 'N3', 'N4']
    assert [int(ln.split(' ')[1][6:7]) for ln in lines] == [n for _, n in w.nodes]
    info = json.load(open(os.path.join(root, 'clusterfile.json')))
    assert list(info) == ['N4', 'X1', 'N2', 'N3', 'N1']
    from metis_b200.workloads import materialize
    bad = per_node(w, 'bad', [('N1', 'A100', 4)], [('N1', node_entry('H100'))])
    with pytest.raises(ValueError, match='N1'):
        materialize(bad, os.path.join(root, 'bad'))


def _problem(name, workload_dir):
    return trp._problem(name, workload_dir)


@pytest.mark.parametrize('name', list(NODE))
def test_node_inputs_discriminate(name, workload_dir):
    """Each workload's per-node readings differ where it is meant to exercise them (bw_first != bw_min for a type, a
    non-uniform bandwidth table, a type memory that is not the type's first hostfile node's, node 0's memory not the
    type's), and the host build's records change when a table is read the other way: bw_first and bw_min exchanged,
    the derived tables of a uniform cluster, or each type's memory from its first hostfile node.  So a golden
    comparison catches each of these mistakes."""
    meta, arr, w, _root, _seqs, problem, space = _problem(name, workload_dir)
    cluster = hs.load_inputs(_root, 'profile', meta['file_order'], w.num_layers, w.hidden_size, w.sequence_length,
                             w.vocab_size)[0]
    a, s = problem.arrays, problem.scalars
    gold = golden_rows(arr)
    got, _ = _host_candidates(problem, space)
    trp._same_candidates(got, gold, name)
    assert (a['type_bw_first'] != a['type_bw_min']).any() and s['uniform_bw'] == 0
    changed = []
    swapped = flatten.FlatProblem(dict(s), dict(a, type_bw_first=a['type_bw_min'], type_bw_min=a['type_bw_first']),
                                  problem.type_names, problem.key_names, problem.node_sequences)
    changed.append(('swapped_bw', _host_candidates(swapped, space)[0]))
    uniform = flatten.FlatProblem(dict(s, uniform_bw=1), dict(a), problem.type_names, problem.key_names,
                                  problem.node_sequences)
    changed.append(('uniform_bw', _host_candidates(uniform, space)[0]))
    by_node = np.array([_first_host_node_memory(cluster, t) for t in problem.type_names])
    if name in ('node_mem_order', 'node_homo'):
        assert (by_node != a['type_memory']).any()
        moved = flatten.FlatProblem(dict(s), dict(a, type_memory=by_node), problem.type_names, problem.key_names,
                                    problem.node_sequences)
        changed.append(('memory_by_host', _host_candidates(moved, space)[0]))
    if name == 'node_homo':
        assert s['node0_memory'] != a['type_memory'][0] and s['node0_bandwidth'] != a['type_bw_min'][0]
    for what, cands in changed:
        assert [c[:8] + (c[8].hex(),) for c in cands] != [g[:8] + (g[8].hex(),) for g in gold], (name, what)
    if name == 'node_bw_mix32':                          # only the costs differ from mix32's
        base = golden_rows(load_golden('mix32')[1])
        assert [g[:8] for g in gold] == [b[:8] for b in base]
        assert any(g[8] != b[8] for g, b in zip(gold, base))
    if name == 'node_mem_order':                          # the memory is tight enough to retry partitions
        assert set(arr['nrep'].tolist()) >= {1, 2, 3}


# ---------------------------------------------------------------------------------------------------------------
# CPU: oracle and host build against the goldens
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(NODE))
def test_oracle_vs_node_golden(name, workload_dir):
    """The oracle's per-node reading, bit for bit with the reference: every candidate, strategy, partition,
    num_repartition and cost, and the A/B/C counters."""
    meta, arr = load_golden(name)
    w, root, digest = workload_dir(name)
    assert digest == meta['inputs_sha256'] and meta['fatal'] is None
    want, counters = trp._oracle_search(w, root, meta['file_order'], [tuple(s) for s in meta['node_sequences']])
    for k in ('A', 'B', 'runs', 'C', 'keyerr'):
        assert counters[k] == meta['counters'][k], k
    trp._same_candidates(want, golden_rows(arr), name)


def test_lower_case_instance_type(workload_dir):
    """An instance_type in lower case names a known type whose memory the raw-string lookup does not find: the
    reference raises TypeError before it costs any candidate, and so do the oracle and build_problem."""
    meta, arr = load_golden('node_lower_case')
    w, root, digest = workload_dir('node_lower_case')
    assert digest == meta['inputs_sha256']
    assert meta['fatal'][1] == 'TypeError' and meta['counters']['C'] == 0 and len(arr['cost']) == 0
    seqs = [tuple(s) for s in meta['node_sequences']]
    with pytest.raises(TypeError) as err:
        trp._oracle_search(w, root, meta['file_order'], seqs)
    assert str(err.value) == meta['fatal'][2]
    cluster, profile, _types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                   w.sequence_length, w.vocab_size)
    with pytest.raises(TypeError) as err:
        flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
    assert str(err.value) == meta['fatal'][2]


@pytest.mark.parametrize('mode', MODES, ids=MODE_IDS)
@pytest.mark.parametrize('where', ['gpu_tier', 'limits'])
@pytest.mark.parametrize('name', list(NODE))
def test_host_build_vs_node_golden(name, where, mode, workload_dir):
    """The host build of the device evaluator in every schedule, in the instantiation the GPU picks and in the
    compiled limits <128, 256>: every golden candidate and the counters."""
    meta, arr, w, _root, _seqs, problem, space = _problem(name, workload_dir)
    tier = hs.gpu_tier(int(space.blocks['num_stage'].max()), w.num_layers, len(w.device_types()))
    assert tier == NODE[name]
    if where == 'limits':
        tier = hs.LIMITS
    got, summary = _host_candidates(problem, space, tier, mode)
    assert summary.reserved[2] == hs.tier_code(tier)
    trp._same_candidates(got, golden_rows(arr), name)
    c = meta['counters']
    assert summary.fatal_ordinal == NO_PLAN
    assert (summary.num_partition_calls, summary.num_balancer_runs, summary.num_records, summary.num_keyerror) == \
        (c['B'], c['runs'], c['C'], c['keyerr'])


def test_homo_node_golden_on_host_and_oracle(workload_dir):
    """The homogeneous path reads hostfile node 0's bandwidth, not the type's first clusterfile entry: the host build
    of HomoCostEstimator.get_cost and the oracle equal the reference's costs, and costing with the type's smallest
    bandwidth instead changes them."""
    meta, arr = load_golden('node_homo_homo')
    w, root, digest = workload_dir('node_homo')
    assert digest == meta['inputs_sha256']
    cluster, profile, types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                  w.sequence_length, w.vocab_size)
    plans = trp._homo_plans(cluster, w)
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, int(plans[:, 2].max()), int(plans[:, 3].max()),
                                    [tuple(dict.fromkeys(t.name for t in cluster.get_device_types()))])
    tid = problem.type_names.index(types[0])
    cost, status = hs.host_homo_cost(problem, tid, plans)
    keep = status != 1
    assert plans[keep].tolist() == arr['plan'].tolist()
    assert _bits(cost[keep]).tolist() == _bits(arr['cost']).tolist()
    slow = flatten.FlatProblem(dict(problem.scalars, node0_bandwidth=float(problem.arrays['type_bw_min'][tid])),
                               problem.arrays, problem.type_names, problem.key_names, problem.node_sequences)
    assert (hs.host_homo_cost(slow, tid, plans)[0][keep] != arr['cost']).any()
    ocl, oprof, otypes, omodel = trp._oracle_inputs(w, root, meta['file_order'])
    out, counters = orc.homo_search(oprof, ocl, omodel, otypes[0], w.gbs, w.max_tp)
    assert counters['yielded'] == meta['yielded'] and counters['costed'] == meta['costed'] == len(arr['cost'])
    assert [list(p) for p, _ in out] == arr['plan'].tolist()
    assert _bits([c for _, c in out]).tolist() == _bits(arr['cost']).tolist()


def test_recost_mix32_into_node_bw_mix32(workload_dir):
    """Bandwidth enters only the cost model: mix32's host-search candidates re-costed under the per-node tables of
    node_bw_mix32 (flatten.cluster_bandwidths) are the reference's node_bw_mix32 costs, bit for bit."""
    base, node = trc.Spec('mix32', workload_dir), trc.Spec('node_bw_mix32', workload_dir)
    problem, space = base.problem(base.root)
    rec, det = trc.host_search(problem, space)
    assert list(zip(rec['ordinal'].tolist(), rec['step'].tolist())) == \
        list(zip(node.arr['ordinal'].tolist(), node.arr['step'].tolist()))
    bw = trc.bandwidths([node.cluster(node.root)], problem.type_names)
    assert (bw[0, 0] != bw[0, 1]).any()
    got = trc.host_recost(problem, space, rec, det, bw)
    assert (_bits(got[0]) == _bits(node.arr['cost'])).all()
    assert (got[0] != rec['cost']).any()


@pytest.mark.parametrize('name', list(NODE))
def test_host_breakdown_vs_oracle_on_node_goldens(name, workload_dir):
    """Sampled golden candidates (retried ones included): the host breakdown's terms sum to the cost, and every term -
    the pp and dp terms that read the per-node bandwidths among them - and stage value equals the oracle twins'."""
    meta, arr, w, root, seqs, problem, space = tb._golden_inputs(name, workload_dir)
    sample = tb._sample_ordinals(arr, 40)
    want = tb._oracle_want(w, root, meta, seqs, sample)
    keep = np.isin(arr['ordinal'], list(sample))
    rec = tb._records(list(zip(arr['ordinal'][keep].tolist(), arr['step'][keep].tolist(), arr['nstage'][keep].tolist(),
                               arr['cost'][keep].tolist())))
    assert [(o, s) for o, s, *_ in want] == list(zip(rec['ordinal'].tolist(), rec['step'].tolist()))
    bd = tb._host_breakdown(problem, space, rec)
    tb._check_oracle(bd, want)
    assert (bd.terms[:, 3] > 0).any() and (bd.terms[:, 4] > 0).any()


# ---------------------------------------------------------------------------------------------------------------
# seeded fuzz: per-node cluster files
# ---------------------------------------------------------------------------------------------------------------
BANDWIDTHS = [1.25e9, 2.5e9, 5312500000.0, 9.0e9, 4.0e10, 9.0e10]
MEMORIES = [10, 16, 24, 40, 80]


def node_workload(rng, idx):
    """A random rough problem (test_rough_profiles.rough_workload) on per-node cluster files: nodes of a type under an
    IP each or sharing one, per-IP bandwidth and memory, the clusterfile in hostfile or shuffled order, with or
    without an entry no hostfile line names."""
    w = trp.rough_workload(rng, idx)
    hosts, entries = [], []
    for k, (dev, n) in enumerate(w.nodes):
        if hosts and hosts[-1][1] == dev and rng.random() < 0.3:
            ip = hosts[-1][0]
        else:
            ip = f'N{k}'
            entries.append((ip, node_entry(dev, rng.choice(BANDWIDTHS), rng.choice(MEMORIES))))
        hosts.append((ip, dev, n))
    if rng.random() < 0.5:
        rng.shuffle(entries)
    if rng.random() < 0.4:
        entries.insert(rng.randrange(len(entries) + 1),
                       ('X0', node_entry(rng.choice(w.device_types()), rng.choice(BANDWIDTHS), rng.choice(MEMORIES))))
    return per_node(w, f'node{idx}', hosts, entries)


class NodeTally(trp.FuzzTally):
    def note(self, w, problem):
        super().note(w, problem)
        a = problem.arrays
        if (a['type_bw_first'] != a['type_bw_min']).any():
            self.features.add('bw_first_ne_min')
        if len({ip for ip, _, _ in w.hosts}) < len(w.hosts):
            self.features.add('shared_ip')
        used = [ip for ip, _ in w.cluster_entries if ip != 'X0']
        if used != list(dict.fromkeys(ip for ip, _, _ in w.hosts)):
            self.features.add('reordered')
        entries = dict(w.cluster_entries)
        for t, mem in zip(problem.type_names, a['type_memory']):
            first_ip = next(ip for ip, dev, _ in w.hosts if dev == t)
            if mem != entries[first_ip]['memory'] * 1024:
                self.features.add('memory_not_first_host')
        if 'X0' in entries:
            self.features.add('unused_entry')


NODE_FEATURES = {'types1', 'types2', 'types3', 'unequal_nodes', 'bw_first_ne_min', 'shared_ip', 'reordered',
                 'memory_not_first_host', 'unused_entry'}


def test_node_random_clusters_vs_oracle(tmp_path):
    """Seeded fuzz: 60 random per-node clusters searched by the device code (host build, the schedules in turn) and
    by the oracle; every candidate, counter and fp64 cost bit agrees, and an aborted search reports a fatal plan of
    the oracle's kind."""
    rng = random.Random(20261018)
    tally = NodeTally()
    idx = 0
    while tally.done < 60 and idx < 1000:
        idx += 1
        w = node_workload(rng, idx)
        case = trp._fuzz_case(w, tmp_path, 6000)
        if case is None:
            continue
        root, order, seqs, problem, space = case
        rec, det, s = hs.host_het_search(problem, space, mode=tally.done % 4)
        summary = {k: getattr(s, k) for k in ('fatal_ordinal', 'fatal_code', 'num_partition_calls',
                                              'num_balancer_runs', 'num_records', 'num_keyerror')}
        trp._check_against_oracle(w, root, order, seqs, space, summary,
                                  lambda: hs.unpack_candidates(rec, det, space), tally)
        tally.note(w, problem)
        tally.done += 1
    print(f'node fuzz: {tally.done} clusters, {tally.candidates} candidates, fatal {tally.fatal}')
    assert tally.done == 60 and tally.candidates > 1000, vars(tally)
    assert tally.features >= NODE_FEATURES, tally.features


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('env', ['smem', 'global'], ids=['tables_in_shared_memory', 'tables_in_global_memory'])
@pytest.mark.parametrize('rows', ['host', 'gpu'], ids=['host_rows', 'gpu_rows'])
@pytest.mark.parametrize('factor', [1, 2 ** 31 - 1], ids=['bulk_round_then_chains', 'chain_kernel_only'])
@pytest.mark.parametrize('name', list(NODE))
def test_node_goldens_on_gpu(name, factor, rows, env, workload_dir, monkeypatch):
    """Every node golden through the C ABI: both schedules, device-group rows from the host enumerator or written by
    the GPU, profile tables in shared or global memory.  Records, detail rows and counters bit for bit."""
    trp._gpu()
    from metis_b200 import search
    if env == 'global':
        monkeypatch.setenv('METIS_SMEM_BLOB_MAX', '0')
    meta, arr, w, _root, seqs, problem, host_space = _problem(name, workload_dir)
    space = host_space if rows == 'host' else flatten.build_plan_space(
        len(seqs), sum(n for _, n in w.nodes), w.gbs, w.num_layers, w.variance, w.max_permute_len, device_rows=True)
    s = search.HetSearcher(search.DeviceProblem(problem, space, 'cuda:0'), want_records=True, want_detail=True)
    s.shard.reserved = factor
    out = s.run()
    sm = trp._gpu_summary(out)
    assert out.summary['instantiation'] == NODE[name]
    trp._same_candidates(hs.unpack_candidates(out.records, out.detail, host_space), golden_rows(arr), name)
    c = meta['counters']
    assert sm['fatal_ordinal'] == NO_PLAN
    assert (sm['num_partition_calls'], sm['num_balancer_runs'], sm['num_records'], sm['num_keyerror']) == \
        (c['B'], c['runs'], c['C'], c['keyerr'])


def _api_args(w, root, meta):
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    args = parse_args(w.cli_args(root))
    cluster, profile, types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                  w.sequence_length, w.vocab_size)
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    return api, args, cluster, profile, types, cfg, volume


@pytest.mark.gpu
def test_node_goldens_through_the_api(workload_dir):
    """api.cost_het_cluster on every node golden (7-tuples, costs bit for bit, ranked()), api.cost_homo_cluster on
    node_homo's homogeneous golden, and the TypeError of a lower-case instance_type."""
    trp._gpu()
    for name in list(NODE) + ['node_lower_case']:
        meta, arr = load_golden(name)
        w, root, _ = workload_dir(name)
        api, args, cluster, profile, _types, cfg, volume = _api_args(w, root, meta)
        seqs = [tuple(s) for s in meta['node_sequences']]

        def run():
            return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume,
                                                                                             cluster),
                                        api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                                        device='cuda:0')
        if meta['fatal'] is not None:
            with pytest.raises(TypeError) as err:
                run()
            assert str(err.value) == meta['fatal'][2]
            continue
        res = run()
        gold = [(tuple(meta['node_sequences'][g[2]]), g[3], g[4], g[5], g[6], g[7], g[8]) for g in golden_rows(arr)]
        got = list(res)
        assert got == gold, name
        assert _bits([g[6] for g in got]).tolist() == _bits(arr['cost']).tolist(), name
        assert res.ranked() == sorted(gold, key=lambda kv: kv[6]), name
    meta, arr = load_golden('node_homo_homo')
    w, root, _ = workload_dir('node_homo')
    api, args, cluster, profile, types, cfg, volume = _api_args(w, root, meta)
    hom = api.cost_homo_cluster(args, cluster, api.HomoCostEstimator(profile, cfg, volume, cluster), types[0],
                                'cuda:0')
    assert [[p.dp, p.pp, p.tp, p.mbs, p.gbs] for p, _ in hom] == arr['plan'].tolist()
    assert _bits([c for _, c in hom]).tolist() == _bits(arr['cost']).tolist()


@pytest.mark.gpu
def test_recost_mix32_search_under_node_bw_mix32(workload_dir, tmp_path):
    """HetSearchResult.recost of a mix32 search (mix32's problem on node_bw_mix32's hostfile, every node at mix32's
    bandwidth) under the node_bw_mix32 cluster: the reference's node_bw_mix32 costs, bit for bit."""
    trp._gpu()
    from metis_b200 import api
    from metis_b200.workloads import materialize
    node = trc.Spec('node_bw_mix32', workload_dir)
    w = WORKLOADS['node_bw_mix32']
    base = per_node(WORKLOADS['mix32'], 'node_mix32', w.hosts,
                    [(ip, dict(e, intra_bandwidth=5312500000.0)) for ip, e in w.cluster_entries])
    root = str(tmp_path / 'base')
    materialize(base, root)
    api.release_engines()
    res = trc._run(node, root)
    mix = load_golden('mix32')[1]
    pos = [res.candidates.index_of(o, s) for o, s in zip(node.arr['ordinal'].tolist(), node.arr['step'].tolist())]
    assert len(res) == len(pos) and (_bits(res.costs[pos]) == _bits(mix['cost'])).all()
    rc = res.recost([node.cluster(node.root)])
    assert (_bits(rc.costs[0][pos]) == _bits(node.arr['cost'])).all()
    assert (rc.costs[0] != res.costs).any()
    api.release_engines()


@pytest.mark.gpu
@pytest.mark.parametrize('reserved', [1, 2 ** 31 - 1], ids=['bulk_then_chain', 'chain_only'])
def test_headroom_on_node_mem_order(reserved, workload_dir, monkeypatch):
    """headroom=True on node_mem_order (memory from a clusterfile entry the hostfile never names): every candidate's
    headroom is the host breakdown's min_headroom, bit for bit."""
    trp._gpu()
    import test_headroom as th
    from metis_b200 import api
    api.release_engines()
    th._schedule(monkeypatch, reserved)
    res = th._run('node_mem_order', workload_dir, True)
    meta, arr, _w, _root, _seqs, problem, space = tb._golden_inputs('node_mem_order', workload_dir)
    assert list(res) == [(tuple(meta['node_sequences'][g[2]]), g[3], g[4], g[5], g[6], g[7], g[8])
                         for g in golden_rows(arr)]
    rec = tb._records(list(zip(arr['ordinal'].tolist(), arr['step'].tolist(), arr['nstage'].tolist(),
                               arr['cost'].tolist())))
    bd = tb._host_breakdown(problem, space, rec)
    assert (_bits(res.headroom) == _bits(bd.min_headroom)).all()
    api.release_engines()


@pytest.mark.gpu
def test_node_random_clusters_on_gpu_vs_oracle(tmp_path):
    """Seeded fuzz through the C ABI: 30 random per-node clusters (the host-build fuzz's generator, another seed) -
    bulk round forced / chain kernel only, rows from the host enumerator / written by the GPU, in turn - against the
    oracle, every candidate, counter and cost bit."""
    trp._gpu()
    from metis_b200 import search
    rng = random.Random(20261019)
    tally = NodeTally()
    idx = 0
    while tally.done < 30 and idx < 600:
        idx += 1
        w = node_workload(rng, idx)
        case = trp._fuzz_case(w, tmp_path, 4000, device_rows=bool(tally.done & 2))
        if case is None:
            continue
        root, order, seqs, problem, space = case
        s = search.HetSearcher(search.DeviceProblem(problem, space, 'cuda:0'), want_records=True, want_detail=True)
        s.shard.reserved = 1 if tally.done & 1 else 2 ** 31 - 1
        out = s.run()
        host_space = space if space.rows.size else flatten.build_plan_space(
            len(seqs), sum(n for _, n in w.nodes), w.gbs, w.num_layers, w.variance, w.max_permute_len)
        trp._check_against_oracle(w, root, order, seqs, space, trp._gpu_summary(out),
                                  lambda: hs.unpack_candidates(out.records, out.detail, host_space), tally)
        tally.note(w, problem)
        tally.done += 1
    print(f'node GPU fuzz: {tally.done} clusters, {tally.candidates} candidates, fatal {tally.fatal}')
    assert tally.done == 30 and tally.candidates > 300, vars(tally)
    assert {'bw_first_ne_min', 'memory_not_first_host', 'unused_entry'} <= tally.features, tally.features
