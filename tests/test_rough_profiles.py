"""The search on rough profiles: values that differ by device type, key and layer.

The default generator (metis_b200/workloads.py) writes one layer shape for every key, scaled by type, tp and bs, and
the same memory profile for every type.  On such inputs several wrong table lookups give the right bits: which type's
memory the memory model reads (quirk Q6), which key normalises the layer weights (Q3), how a mixed stage splits its
data.  The rough_* workloads (profile_style='rough') make them observable: per-type compute and memory shapes,
per-key noise, int memory lists, memory lists one entry short, fb_sync == 0.0 (Q9), keys only one type has, unequal
nodes (Q10).  Their goldens come from the unmodified reference (tests/golden/make_golden.py).

CPU: the oracle and the host build of the device evaluator against every golden, a seeded 160-cluster fuzz against
the oracle, and checks that each input discriminates (a Q6 correction, exchanged memory rows and a different
normalisation key each change the result).  GPU (-m gpu): the goldens through the C ABI and api, a 60-cluster fuzz,
random max_permute_len 1 workloads in the larger instantiations and the homogeneous path.
"""
import copy
import itertools
import os
import random

import numpy as np
import pytest

import hostsim_util as hs
from conftest import golden_rows, load_golden
from metis_b200 import flatten, native
from oracle import metis_oracle as orc

# golden -> (instantiation the GPU picks, whether the reference aborted)
ROUGH = {
    'rough_mix2': (64, 128, False),
    'rough_t3': (64, 128, False),
    'rough_q10': (64, 128, False),
    'rough_long_int': (64, 128, False),
    'rough_keys': (64, 128, False),
    'rough_keys_fatal': (64, 128, False),
    'rough_s66_t2': (96, 128, False),
    'rough_l130_t2': (128, 256, False),
}
FATAL = {'rough_keys_fatal'}
COMPLETE = [n for n in ROUGH if n not in FATAL]
NO_PLAN = 2 ** 64 - 1
MODES = [0, 1, 2, 3, 4]
MODE_IDS = ['sequential_run', 'first_task_then_chain', 'chain_only', 'chain_only_reversed_par_sections',
            'first_task_then_replay']


def _lib_or_skip():
    try:
        return native.load_library()
    except native.MetisNativeError as e:
        pytest.skip(str(e))


def _oracle_inputs(w, root, file_order, profile=None):
    cluster = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    prof, types = orc.load_profile_dir(os.path.join(root, 'profile'), file_order)
    prof = profile if profile is not None else prof
    model = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size, prof['model']['parameters'])
    return cluster, prof, types, model


def _oracle_search(w, root, file_order, seqs, profile=None, **kw):
    cluster, prof, _types, model = _oracle_inputs(w, root, file_order, profile)
    return orc.het_search(prof, cluster, model, seqs, w.gbs, w.num_layers, w.variance, w.max_permute_len,
                          w.max_tp, w.max_bs, **kw)


def _problem(name, workload_dir, corrected=()):
    lib = _lib_or_skip()
    meta, arr = load_golden(name)
    w, root, digest = workload_dir(name)
    assert digest == meta['inputs_sha256']
    cluster, profile, _types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                   w.sequence_length, w.vocab_size)
    seqs = [tuple(s) for s in meta['node_sequences']]
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs, corrected=corrected)
    space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance,
                                     w.max_permute_len, lib)
    return meta, arr, w, root, seqs, problem, space


def _same_candidates(got, want, w=None):
    """got / want: (ordinal, step, ns, groups, strategies, batches, partition, nrep, cost) lists."""
    assert len(got) == len(want), w
    for g, x in zip(got, want):
        assert (g[0], g[1], g[3], g[4], g[5], g[6], g[7]) == (x[0], x[1], x[3], x[4], x[5], x[6], x[7]), (w, g, x)
        assert g[8] == x[8], (w, g[0], g[1], g[8].hex(), x[8].hex())


def _fatal_cut(meta, cands):
    """The reference stops at its first failing plan: only what precedes it is compared."""
    if meta['fatal'] is None:
        return cands
    return [c for c in cands if c[0] < meta['fatal'][0]]


# ---------------------------------------------------------------------------------------------------------------
# the generator
# ---------------------------------------------------------------------------------------------------------------
def test_rough_inputs_have_the_planted_features(workload_dir):
    """What the rough goldens are meant to contain is in their inputs: int and float memory lists, a memory list one
    entry short of 15 profiled layers, fb_sync == 0.0 and negative fb_sync, a key one type lacks, a compute row two
    types share bit for bit while their other rows differ, and runs of equal layers."""
    seen = set()
    for name in ROUGH:
        w, root, _ = workload_dir(name)
        meta, _ = load_golden(name)
        prof, types = orc.load_profile_dir(os.path.join(root, 'profile'), meta['file_order'])
        nl = w.profile_layers or w.num_layers
        keys = {t: prof[f'DeviceType.{t}'] for t in types}
        for t, rows in keys.items():
            for key, e in rows.items():
                kinds = {type(v) for v in e['memory']}
                assert len(kinds) == 1 and len(e['time']['layer-computes']) == nl
                seen.add('int' if kinds == {int} else 'float')
                if len(e['memory']) == nl - 1:
                    seen.add('short')
                fb = e['time']['fb_sync']
                seen.add('zero_fb' if fb == 0.0 else 'negative_fb' if fb < 0 else 'positive_fb')
                lc = e['time']['layer-computes']
                if any(a == b for a, b in zip(lc[1:], lc[2:-1])):
                    seen.add('runs')
        if len(types) > 1:
            a, b = keys[types[0]], keys[types[1]]
            same = [k for k in a if k in b and a[k]['time']['layer-computes'] == b[k]['time']['layer-computes']]
            assert len(same) == 1, name
            if set(a) != set(b):
                seen.add('missing')
        if w.profile_layers > w.num_layers:
            seen.add('norm_len')
        if len({n for _, n in w.nodes}) > 1:
            seen.add('unequal_nodes')
    assert seen == {'int', 'float', 'short', 'zero_fb', 'negative_fb', 'positive_fb', 'runs', 'missing', 'norm_len',
                    'unequal_nodes'}, seen


# ---------------------------------------------------------------------------------------------------------------
# CPU: oracle and host build against the goldens
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(ROUGH))
def test_oracle_vs_rough_golden(name, workload_dir):
    """The oracle on the rough inputs, bit for bit with the reference: every candidate and counter, and for the
    aborted search the same exception at the same plan."""
    meta, arr = load_golden(name)
    w, root, digest = workload_dir(name)
    assert digest == meta['inputs_sha256']
    seqs = [tuple(s) for s in meta['node_sequences']]
    gold = golden_rows(arr)
    if meta['fatal'] is not None:
        stop = meta['fatal'][0]
        with pytest.raises(KeyError) as err:
            _oracle_search(w, root, meta['file_order'], seqs)
        assert str(err.value) == meta['fatal'][2]
        want, counters = _oracle_search(w, root, meta['file_order'], seqs, plan_filter=lambda o: o < stop)
        assert counters['C'] == meta['counters']['C']      # the other counters include work past the fatal plan
    elif meta['counters']['A'] > 5000:                  # minutes for the oracle: its largest block and seeded plans
        from test_limits import _oracle_sample
        *_, space = _problem(name, workload_dir)
        sample = set(_oracle_sample(space, arr, n_random=200))
        want, counters = _oracle_search(w, root, meta['file_order'], seqs, plan_filter=sample.__contains__)
        gold = [g for g in gold if g[0] in sample]
        assert counters['A'] == meta['counters']['A'] and len(gold) > 200
    else:
        want, counters = _oracle_search(w, root, meta['file_order'], seqs)
        for k in ('A', 'B', 'runs', 'C', 'keyerr'):
            assert counters[k] == meta['counters'][k], k
    _same_candidates(want, gold, name)


@pytest.mark.parametrize('mode', MODES, ids=MODE_IDS)
@pytest.mark.parametrize('where', ['gpu_tier', 'limits'])
@pytest.mark.parametrize('name', list(ROUGH))
def test_host_build_vs_rough_golden(name, where, mode, workload_dir):
    """The host build of the device evaluator in every schedule, in the instantiation the GPU picks and in the
    compiled limits <128, 256>: every golden candidate, the counters, and the fatal plan with its KeyError."""
    from metis_b200 import search
    meta, arr, w, _root, _seqs, problem, space = _problem(name, workload_dir)
    tier = hs.gpu_tier(int(space.blocks['num_stage'].max()), w.num_layers, len(w.device_types()))
    assert tier == ROUGH[name]
    if where == 'limits':
        if tier == hs.LIMITS:
            pytest.skip('the GPU picks the compiled limits already')
        tier = hs.LIMITS
    rec, det, summary = hs.host_het_search(problem, space, mode=mode, tier=tier,
                                           capacity=max(1024, space.num_plans * 4))
    assert summary.reserved[2] == hs.tier_code(tier)
    got = _fatal_cut(meta, hs.unpack_candidates(rec, det, space))
    _same_candidates(got, golden_rows(arr), name)
    c = meta['counters']
    if meta['fatal'] is None:
        assert summary.fatal_ordinal == NO_PLAN
        assert (summary.num_partition_calls, summary.num_balancer_runs, summary.num_records, summary.num_keyerror) == \
            (c['B'], c['runs'], c['C'], c['keyerr'])
    else:
        assert summary.fatal_ordinal == meta['fatal'][0]
        with pytest.raises(KeyError) as err:
            search.raise_fatal({'fatal_ordinal': summary.fatal_ordinal, 'fatal_code': summary.fatal_code,
                                'fatal_aux': summary.fatal_aux}, problem)
        assert str(err.value) == meta['fatal'][2]


def _homo_plans(cluster, w):
    from metis_b200 import api
    return np.array([[p.dp, p.pp, p.tp, p.mbs, p.gbs] for p in api.UniformPlanGenerator(
        cluster.get_total_num_devices(), w.max_tp, w.gbs) if p.gbs == w.gbs], dtype=np.int32)


def test_homo_rough_golden_on_host_and_oracle(workload_dir):
    """HomoCostEstimator.get_cost (device code, host build) and the oracle against the reference on a rough
    single-type workload: int memory, a zero fb_sync and an unprofiled key skip plans by KeyError."""
    _lib_or_skip()
    meta, arr = load_golden('rough_homo_homo')
    w, root, digest = workload_dir('rough_homo')
    assert digest == meta['inputs_sha256']
    cluster, profile, types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                  w.sequence_length, w.vocab_size)
    plans = _homo_plans(cluster, w)
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, int(plans[:, 2].max()), int(plans[:, 3].max()),
                                    [tuple(dict.fromkeys(t.name for t in cluster.get_device_types()))])
    cost, status = hs.host_homo_cost(problem, problem.type_names.index(types[0]), plans)
    keep = status != 1
    assert (~keep).sum() > 0
    assert plans[keep].tolist() == arr['plan'].tolist()
    assert cost[keep].tolist() == arr['cost'].tolist()
    ocl, oprof, otypes, omodel = _oracle_inputs(w, root, meta['file_order'])
    out, counters = orc.homo_search(oprof, ocl, omodel, otypes[0], w.gbs, w.max_tp)
    assert counters['yielded'] == meta['yielded'] and counters['costed'] == meta['costed'] == len(arr['cost'])
    assert [list(p) for p, _ in out] == arr['plan'].tolist()
    assert [c for _, c in out] == arr['cost'].tolist()


# ---------------------------------------------------------------------------------------------------------------
# CPU: each input discriminates
# ---------------------------------------------------------------------------------------------------------------
def _single_type(cluster, cand):
    types = orc.rank_types_by_devices(cluster, cand[2])
    a = 0
    for g in cand[3]:
        if len(set(types[a:a + g])) > 1:
            return False
        a += g
    return True


def _sens_filter(meta, arr):
    """The plans the sensitivity checks evaluate: all of them, or the first 400 costed ones of a large space."""
    if meta['fatal'] is not None:
        stop = meta['fatal'][0]
        return lambda o: o < stop
    if meta['counters']['A'] <= 5000:
        return None
    keep = set(np.unique(arr['ordinal'])[:400].tolist())
    return keep.__contains__


@pytest.mark.parametrize('name', COMPLETE)        # rough_keys_fatal shares rough_keys' inputs but one file
def test_rough_inputs_discriminate(name, workload_dir):
    """On each golden's inputs the oracle's result changes when (a) the memory demand comes from the stage's own type
    (correction 'Q6') - on plans whose stages are all single-type, (b) the memory rows of a node sequence's first type
    are exchanged with another type's; and (c) the layer weights (Q3: the first-listed type's tp1_bs1, normalised)
    differ bitwise from the normalised compute of other keys.  A wrong table lookup therefore cannot pass the
    golden comparisons by accident."""
    meta, arr = load_golden(name)
    w, root, _ = workload_dir(name)
    seqs = [tuple(s) for s in meta['node_sequences']]
    cluster, prof, types, _model = _oracle_inputs(w, root, meta['file_order'])
    flt = _sens_filter(meta, arr)
    base, _ = _oracle_search(w, root, meta['file_order'], seqs, plan_filter=flt)
    # (a)
    fixed, _ = _oracle_search(w, root, meta['file_order'], seqs, plan_filter=flt, corrected=('Q6',))
    pure = [c for c in base if _single_type(cluster, c)]
    pure_fixed = [c for c in fixed if _single_type(cluster, c)]
    assert pure and pure != pure_fixed, name
    # (b) for every type that starts a node sequence
    for first in sorted({s[0] for s in seqs}):
        other = next(t for t in types if t != first)
        p2 = copy.deepcopy(prof)
        a, b = p2[f'DeviceType.{first}'], p2[f'DeviceType.{other}']
        for key in set(a) & set(b):
            a[key]['memory'], b[key]['memory'] = b[key]['memory'], a[key]['memory']
        try:
            swapped, _ = _oracle_search(w, root, meta['file_order'], seqs, profile=p2, plan_filter=flt)
        except (KeyError, IndexError):
            swapped = None
        assert swapped != base, (name, first, other)
    # (c)
    norm = orc.norm_layer_duration(prof)
    differ = 0
    for t in types:
        for key, e in prof[f'DeviceType.{t}'].items():
            lc = e['time']['layer-computes']
            total = orc.fsum(lc)
            differ += [x / total for x in lc] != norm
    assert differ >= len(types) * 6, (name, differ)


# ---------------------------------------------------------------------------------------------------------------
# seeded fuzz with the rough generator
# ---------------------------------------------------------------------------------------------------------------
# node sizes in hostfile order, power-of-two totals; the last three put a smaller node first (Q10 IndexError)
LAYOUTS = [[8], [4, 4], [2, 2], [8, 8], [8, 4, 4], [8, 4, 2, 2], [4, 2, 2], [4, 2, 1, 1], [8, 8, 8, 8], [8, 8, 4, 4],
           [4, 4, 4, 4], [2, 4, 2], [4, 8, 4], [2, 2, 4]]


def rough_workload(rng, idx, mpl=None, layouts=LAYOUTS):
    """A random small cluster with rough profiles: 1-3 types, unequal nodes, more profiled than searched layers, int
    memory, short memory lists, zero fb_sync keys and keys one type lacks."""
    from metis_b200.workloads import Workload
    ntypes = rng.choice([1, 2, 2, 3, 3])
    layout = rng.choice([lay for lay in layouts if len(lay) >= ntypes])
    types = rng.sample(['A100', 'H100', 'B200', 'V100'], ntypes)
    nodes = [(types[(i * ntypes) // len(layout)], n) for i, n in enumerate(layout)]
    layers = rng.randint(6, 28)
    profile_layers = layers + rng.choice([0, 0, 0, 1, 4])
    tps, bss = (1, 2, 4), (1, 2, 4, 8, 16)
    keys = [(t, tp, bs) for t in types for tp in tps for bs in bss]
    zero = tuple(k for k in keys if rng.random() < 0.12)
    missing = ()
    if ntypes > 1 and rng.random() < 0.4:
        t = rng.choice(types[1:])                       # never the first-listed type's tp1_bs1 (norm_layer_duration)
        missing = ((t, rng.choice(tps), rng.choice(bss if rng.random() < 0.3 else (8, 16))),)
    return Workload(f'rough{idx}', nodes, layers, rng.choice([8, 12, 16, 24, 32, 48, 64]),
                    rng.choice([1024, 4096, 8192]), rng.choice([512, 2048]), rng.choice([30522, 51200]),
                    variance=rng.choice([0, 0.5, 1, 1]), max_permute_len=mpl or rng.choice([2, 3, 4, 6]),
                    max_tp=rng.choice([1, 2, 4]), max_bs=rng.choice([1, 2, 4]), bss=bss, seed=idx,
                    memory_gb={t: rng.choice([6, 10, 16, 24, 40, 80]) for t in types},
                    intra_bw={t: rng.choice([5312500000.0, 2.5e9, 9.0e10]) for t in types},
                    profile_layers=profile_layers, profile_style='rough',
                    int_memory=tuple(t for t in types if rng.random() < 0.5), short_memory=rng.random() < 0.3,
                    zero_fb_sync=zero, missing=missing)


def _fuzz_case(w, tmp_path, max_plans, device_rows=False):
    """Materialise w; -> (root, order, seqs, problem, space) or None when the space is empty / too large."""
    from metis_b200.workloads import materialize, profile_file_order
    root = str(tmp_path / w.name)
    materialize(w, root)
    order = profile_file_order(w)
    cluster, profile, _types, cfg = hs.load_inputs(root, 'profile', order, w.num_layers, w.hidden_size,
                                                   w.sequence_length, w.vocab_size)
    seqs = list(itertools.permutations(w.device_types()))
    try:
        space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers,
                                         w.variance, w.max_permute_len, device_rows=device_rows)
    except IndexError:
        return None                                    # no stage-1 rows: the reference raises before searching
    if not 1 <= space.num_plans <= max_plans:
        return None
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
    return root, order, seqs, problem, space


class FuzzTally:
    """What a fuzz run reached, so that it can assert that it reached it."""

    def __init__(self):
        self.done = self.candidates = self.keyerr = 0
        self.fatal = {'key': 0, 'index': 0}
        self.features = set()

    def note(self, w, problem):
        self.features.add(f'types{len(w.device_types())}')
        if len({n for _, n in w.nodes}) > 1:
            self.features.add('unequal_nodes')
        if int(problem.scalars['norm_len']) != w.num_layers:
            self.features.add('norm_len')
        if w.missing:
            self.features.add('missing_key')
        if w.zero_fb_sync:
            self.features.add('zero_fb_sync')
        if w.int_memory:
            self.features.add('int_memory')
        if w.short_memory:
            self.features.add('short_memory')


def _check_against_oracle(w, root, order, seqs, space, summary, got, tally):
    """The oracle on the same inputs; ``summary`` is a dict of the device summary, ``got`` its candidates."""
    try:
        want, counters = _oracle_search(w, root, order, seqs)
    except KeyError:
        assert summary['fatal_ordinal'] != NO_PLAN and summary['fatal_code'] in (1, 2), w
        tally.fatal['key'] += 1
        return
    except IndexError:
        assert summary['fatal_ordinal'] != NO_PLAN and summary['fatal_code'] == 3, w
        tally.fatal['index'] += 1
        return
    assert summary['fatal_ordinal'] == NO_PLAN, w
    assert (space.num_plans, summary['num_partition_calls'], summary['num_balancer_runs'], summary['num_records'],
            summary['num_keyerror']) == (counters['A'], counters['B'], counters['runs'], counters['C'],
                                         counters['keyerr']), w
    _same_candidates(got(), want, w)
    tally.candidates += len(want)
    tally.keyerr += counters['keyerr']


FEATURES = {'types1', 'types2', 'types3', 'unequal_nodes', 'norm_len', 'missing_key', 'zero_fb_sync', 'int_memory',
            'short_memory'}


def test_rough_random_clusters_vs_oracle(tmp_path):
    """Seeded fuzz: 160 random small clusters with rough profiles searched by the device code (host build, all four
    scheduling modes in turn) and by the oracle; every candidate, counter and fp64 cost bit must agree, and a search
    the oracle aborts (KeyError, or IndexError when node 0 is the smallest) must report a fatal plan of that kind."""
    rng = random.Random(20261016)
    tally = FuzzTally()
    idx = 0
    while tally.done < 160 and idx < 2000:
        idx += 1
        w = rough_workload(rng, idx)
        case = _fuzz_case(w, tmp_path, 6000)
        if case is None:
            continue
        root, order, seqs, problem, space = case
        rec, det, s = hs.host_het_search(problem, space, mode=tally.done % 4)
        summary = {k: getattr(s, k) for k in ('fatal_ordinal', 'fatal_code', 'num_partition_calls',
                                              'num_balancer_runs', 'num_records', 'num_keyerror')}
        _check_against_oracle(w, root, order, seqs, space, summary, lambda: hs.unpack_candidates(rec, det, space),
                              tally)
        tally.note(w, problem)
        tally.done += 1
    print(f'rough fuzz: {tally.done} clusters, {tally.candidates} candidates, {tally.keyerr} per-candidate KeyErrors, '
          f'fatal {tally.fatal}')
    assert tally.done == 160 and tally.candidates > 2000 and tally.keyerr > 0, vars(tally)
    assert tally.features == FEATURES, tally.features
    assert 0 < tally.fatal['key'] < 60 and 0 < tally.fatal['index'] < 60, tally.fatal


def rough_homo_workload(rng, idx):
    from metis_b200.workloads import Workload
    dev = rng.choice(['A100', 'H100', 'B200', 'V100'])
    per = rng.choice([2, 4, 8])
    nn = rng.choice([1, 2, 4]) if per == 8 else rng.choice([1, 2, 3, 4])
    layers = rng.randint(6, 40)
    bss = rng.choice([(1, 2, 4), (1, 2, 4, 8), (1, 2)])
    keys = [(dev, tp, bs) for tp in (1, 2, 4) for bs in bss]
    return Workload(f'rough_homo{idx}', [(dev, per)] * nn, layers, rng.choice([8, 16, 24, 32, 64, 96]),
                    rng.choice([1024, 4096]), rng.choice([512, 2048]), 51200, max_tp=rng.choice([1, 2, 4]),
                    tps=(1, 2, 4), bss=bss, seed=3000 + idx, memory_gb={dev: rng.choice([8, 16, 40, 80])},
                    profile_layers=layers + rng.choice([0, 0, 3]), profile_style='rough',
                    int_memory=(dev,) if rng.random() < 0.5 else (), short_memory=rng.random() < 0.3,
                    zero_fb_sync=tuple(k for k in keys if rng.random() < 0.15),
                    missing=tuple(k for k in keys[1:] if rng.random() < 0.08))


def _homo_case(w, tmp_path):
    from metis_b200.workloads import materialize, profile_file_order
    root = str(tmp_path / w.name)
    materialize(w, root)
    order = profile_file_order(w)
    cluster, profile, types, cfg = hs.load_inputs(root, 'profile', order, w.num_layers, w.hidden_size,
                                                  w.sequence_length, w.vocab_size)
    plans = _homo_plans(cluster, w)
    if not len(plans):
        return None
    ocl, oprof, otypes, omodel = _oracle_inputs(w, root, order)
    want, counters = orc.homo_search(oprof, ocl, omodel, otypes[0], w.gbs, w.max_tp)
    return root, order, cluster, profile, types, cfg, plans, want, counters


def test_rough_random_homo_clusters_vs_oracle_on_host(tmp_path):
    """The homogeneous path on 60 rough single-type clusters (host build) against the oracle: plans kept, plans
    skipped by KeyError (unprofiled keys, fb_sync == 0.0) and every fp64 cost."""
    _lib_or_skip()
    rng = random.Random(1016)
    costed = skipped = 0
    for idx in range(60):
        w = rough_homo_workload(rng, idx)
        case = _homo_case(w, tmp_path)
        if case is None:
            continue
        _root, _order, cluster, profile, types, cfg, plans, want, counters = case
        problem = flatten.build_problem(profile, cluster, cfg, w.gbs, int(plans[:, 2].max()), int(plans[:, 3].max()),
                                        [tuple(dict.fromkeys(t.name for t in cluster.get_device_types()))])
        cost, status = hs.host_homo_cost(problem, problem.type_names.index(types[0]), plans)
        keep = status != 1
        assert counters['matched'] == len(plans) and counters['keyerr'] == int((~keep).sum()), w
        assert plans[keep].tolist() == [list(p) for p, _ in want], w
        assert cost[keep].tolist() == [c for _, c in want], w
        costed += len(want)
        skipped += counters['keyerr']
    assert costed > 300 and skipped > 20, (costed, skipped)


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()          # raises (test error, not skip) when the extension is missing
    return torch


def _gpu_summary(out):
    return {k: out.summary[k] for k in ('fatal_ordinal', 'fatal_code', 'fatal_aux', 'num_partition_calls',
                                        'num_balancer_runs', 'num_records', 'num_keyerror')}


@pytest.mark.gpu
@pytest.mark.parametrize('env', ['smem', 'global'], ids=['tables_in_shared_memory', 'tables_in_global_memory'])
@pytest.mark.parametrize('rows', ['host', 'gpu'], ids=['host_rows', 'gpu_rows'])
@pytest.mark.parametrize('factor', [1, 2 ** 31 - 1], ids=['bulk_round_then_chains', 'chain_kernel_only'])
@pytest.mark.parametrize('name', list(ROUGH))
def test_rough_goldens_on_gpu(name, factor, rows, env, workload_dir, monkeypatch):
    """Every rough golden through the C ABI: both schedules, device-group rows from the host enumerator or written by
    the GPU, profile tables in the kernels' shared-memory copy or read from global memory.  Every candidate bit for
    bit, the counters, the instantiation, and for the aborted search the plan and its KeyError."""
    _gpu()
    from metis_b200 import search
    if env == 'global':
        monkeypatch.setenv('METIS_SMEM_BLOB_MAX', '0')
    meta, arr, w, _root, seqs, problem, host_space = _problem(name, workload_dir)
    space = host_space if rows == 'host' else flatten.build_plan_space(
        len(seqs), sum(n for _, n in w.nodes), w.gbs, w.num_layers, w.variance, w.max_permute_len, device_rows=True)
    s = search.HetSearcher(search.DeviceProblem(problem, space, 'cuda:0'), want_records=True, want_detail=True)
    s.shard.reserved = factor
    out = s.run()
    sm = _gpu_summary(out)
    assert out.summary['instantiation'] == ROUGH[name]
    got = _fatal_cut(meta, hs.unpack_candidates(out.records, out.detail, host_space))
    _same_candidates(got, golden_rows(arr), name)
    c = meta['counters']
    if meta['fatal'] is None:
        assert sm['fatal_ordinal'] == NO_PLAN
        assert (sm['num_partition_calls'], sm['num_balancer_runs'], sm['num_records'], sm['num_keyerror']) == \
            (c['B'], c['runs'], c['C'], c['keyerr'])
    else:
        assert sm['fatal_ordinal'] == meta['fatal'][0]
        with pytest.raises(KeyError) as err:
            search.raise_fatal(sm, problem)
        assert str(err.value) == meta['fatal'][2]


@pytest.mark.gpu
def test_rough_goldens_through_the_api(workload_dir):
    """api.cost_het_cluster on every complete rough golden, back to back through the cached engine: the 7-tuples
    equal the golden rows, ranked() is Python's stable sort."""
    _gpu()
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    for name in COMPLETE:
        meta, arr = load_golden(name)
        w, root, _ = workload_dir(name)
        args = parse_args(w.cli_args(root))
        cluster, profile, _types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers,
                                                       w.hidden_size, w.sequence_length, w.vocab_size)
        volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
        est = api.HeteroCostEstimator(profile, cfg, volume, cluster)
        llb = api.LayerLoadBalancer(cluster, profile, cfg, args.gbs)
        seqs = [tuple(s) for s in meta['node_sequences']]
        res = api.cost_het_cluster(args, cluster, profile, cfg, est, llb, node_sequences=seqs, device='cuda:0')
        gold = [(tuple(meta['node_sequences'][g[2]]), g[3], g[4], g[5], g[6], g[7], g[8]) for g in golden_rows(arr)]
        got = list(res)
        assert len(got) == len(gold), name
        assert got == gold, name
        assert res.ranked() == sorted(gold, key=lambda kv: kv[6]), name


@pytest.mark.gpu
def test_rough_random_clusters_on_gpu_vs_oracle(tmp_path):
    """Seeded fuzz through the C ABI: 60 random rough clusters (the generator of the host-build fuzz, another seed)
    on the GPU - bulk round forced / chain kernel only, rows from the host enumerator / written by the GPU, in turn -
    against the oracle, every candidate, counter and cost bit."""
    _gpu()
    from metis_b200 import search
    rng = random.Random(20261017)
    tally = FuzzTally()
    idx = 0
    while tally.done < 60 and idx < 900:
        idx += 1
        w = rough_workload(rng, idx)
        case = _fuzz_case(w, tmp_path, 6000, device_rows=bool(tally.done & 2))
        if case is None:
            continue
        root, order, seqs, problem, space = case
        s = search.HetSearcher(search.DeviceProblem(problem, space, 'cuda:0'), want_records=True, want_detail=True)
        s.shard.reserved = 1 if tally.done & 1 else 2 ** 31 - 1
        out = s.run()
        host_space = space if space.rows.size else flatten.build_plan_space(
            len(seqs), sum(n for _, n in w.nodes), w.gbs, w.num_layers, w.variance, w.max_permute_len)
        _check_against_oracle(w, root, order, seqs, space, _gpu_summary(out),
                              lambda: hs.unpack_candidates(out.records, out.detail, host_space), tally)
        tally.note(w, problem)
        tally.done += 1
    print(f'rough GPU fuzz: {tally.done} clusters, {tally.candidates} candidates, fatal {tally.fatal}')
    assert tally.done == 60 and tally.candidates > 500, vars(tally)
    assert {'types2', 'types3', 'unequal_nodes', 'norm_len'} <= tally.features, tally.features


@pytest.mark.gpu
def test_rough_mpl1_workloads_in_the_larger_instantiations(tmp_path):
    """Random max_permute_len 1 rough workloads whose plans have 65-128 stages or more than 128 layers, so that the
    search runs in the <96, 128> and <128, 256> instantiations: every candidate against the oracle."""
    _gpu()
    from metis_b200 import search
    from metis_b200.workloads import Workload, _nodes
    rng = random.Random(66)
    tiers = set()
    cands = 0
    # 128 GPUs and 65 / 66 layers: 65-66 stages (<96, 128>); 16 / 32 GPUs and 130-200 layers (<128, 256>)
    specs = [(('A100', 8), ('H100', 8), 65), (('V100', 8), ('B200', 8), 66), (('A100', 1), ('V100', 1), 140),
             (('H100', 1), ('B200', 1), 200), (('A100', 2), ('H100', 2), 130), (('B200', 2), ('A100', 2), 140)]
    for i, (a, b, layers) in enumerate(specs):
        w = Workload(f'rough_mpl1_{i}', _nodes(a, b), layers, 8, 4096, 1024, 51200, max_permute_len=1,
                     bss=(1, 2, 4, 8), seed=500 + i, profile_style='rough',
                     memory_gb={a[0]: rng.choice([40, 64, 240]), b[0]: rng.choice([40, 64, 240])},
                     int_memory=(b[0],), short_memory=bool(i & 1), profile_layers=layers + (i % 3))
        case = _fuzz_case(w, tmp_path, 20000)
        assert case is not None, w
        root, order, seqs, problem, space = case
        tier = hs.gpu_tier(int(space.blocks['num_stage'].max()), w.num_layers, 2)
        s = search.HetSearcher(search.DeviceProblem(problem, space, 'cuda:0'), want_records=True, want_detail=True)
        s.shard.reserved = 1 if i & 1 else 2 ** 31 - 1
        out = s.run()
        assert out.summary['instantiation'] == tier
        tiers.add(tier)
        sm = _gpu_summary(out)
        assert sm['fatal_ordinal'] == NO_PLAN
        got = hs.unpack_candidates(out.records, out.detail, space)
        if space.num_plans <= 1000:
            want, counters = _oracle_search(w, root, order, seqs)
            assert (sm['num_partition_calls'], sm['num_balancer_runs'], sm['num_records']) == \
                (counters['B'], counters['runs'], counters['C']), w
        else:                                           # the oracle needs minutes here: the largest blocks' first
            ndiv = len(space.batches)                   # rows and seeded plans
            top = int(space.blocks['num_stage'].max())
            sample = set(rng.sample(range(space.num_plans), 120))
            for blk in space.blocks[space.blocks['num_stage'] >= top - 1]:
                sample.update(range(int(blk['first_ordinal']), int(blk['first_ordinal']) + ndiv))
            want, _ = _oracle_search(w, root, order, seqs, plan_filter=sample.__contains__)
            got = [g for g in got if g[0] in sample]
        _same_candidates(got, want, w)
        cands += len(want)
    assert tiers == {(96, 128, False), (128, 256, False)} and cands > 0, (tiers, cands)


@pytest.mark.gpu
def test_rough_homo_on_gpu(workload_dir, tmp_path):
    """api.cost_homo_cluster (homo_cost_kernel) on the rough homo golden, and on 60 rough single-type clusters
    against the oracle's homo_search."""
    _gpu()
    from metis_b200 import api
    from metis_b200.arguments import parse_args

    def run(w, root, order):
        cluster, profile, types, cfg = hs.load_inputs(root, 'profile', order, w.num_layers, w.hidden_size,
                                                      w.sequence_length, w.vocab_size)
        args = parse_args(['--gbs', str(w.gbs), '--max_profiled_tp_degree', str(w.max_tp),
                           '--num_layers', str(w.num_layers)])
        volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
        return api.cost_homo_cluster(args, cluster, api.HomoCostEstimator(profile, cfg, volume, cluster), types[0],
                                     'cuda:0')

    meta, arr = load_golden('rough_homo_homo')
    w, root, _ = workload_dir('rough_homo')
    hom = run(w, root, meta['file_order'])
    assert [[p.dp, p.pp, p.tp, p.mbs, p.gbs] for p, _ in hom] == arr['plan'].tolist()
    assert [c for _, c in hom] == arr['cost'].tolist()
    rng = random.Random(1017)
    costed = 0
    for idx in range(60):
        w = rough_homo_workload(rng, idx)
        case = _homo_case(w, tmp_path)
        if case is None:
            continue
        root, order, *_rest, want, _counters = case
        hom = run(w, root, order)
        assert [[p.dp, p.pp, p.tp, p.mbs, p.gbs] for p, _ in hom] == [list(p) for p, _ in want], w
        assert [c for _, c in hom] == [c for _, c in want], w
        costed += len(want)
    assert costed > 300, costed
