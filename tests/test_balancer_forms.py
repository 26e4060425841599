"""The three forms of LayerComputeBalancer.run against the oracle, on inputs built to take their rarely taken paths
(tests/balancer_cases.py), and the WarpCoop lane primitives against numpy.

  Serial    balance_run, one plan per thread          replay / trace kernels, metis_layer_balance
  Lockstep  balance_run, 32 plans per warp re-joined  bulk round (het_first_kernel)
  Coop      CoopEvaluator::balance_coop on WarpCoop   chain kernel (het_chain_kernel)

On the CPU the host build runs Serial and Coop on one lane (forward and reverse); on the GPU tests/devsim runs all
three in each scratch tier.  Every partition (or fatal code) must equal the oracle's, and every family must reach the
path it is built for (BalancerPath notes), so a generator that stops reaching its path fails.
"""
import collections
import functools
import math
import os

import numpy as np
import pytest

import balancer_cases as bc
import devsim_util as ds

KNIFE_SHARE = 0.5          # knife-edge rows whose forward prediction must fail to verify under Coop


@functools.lru_cache(maxsize=None)
def expected(tier):
    """(cases, knife-edge statistics, oracle result per row of every case) for one scratch tier."""
    cases, stats = bc.all_cases(tier)
    return cases, stats, [[bc.oracle(L, lc, capa) for capa in rows] for _f, L, lc, rows, _t in cases]


def check_forms(tier, run, policies, noted):
    """Runs every case through `run(policy, rows, lc, L)` for each policy; asserts oracle parity and returns, for the
    policy `noted`, per family: Counter of rows and of each path taken, and the longest middle block."""
    cases, _stats, wants = expected(tier)
    seen = collections.defaultdict(collections.Counter)
    longest = 0
    for (family, L, lc, rows, _target), want in zip(cases, wants):
        for policy in policies:
            got = run(policy, rows, lc, L)
            for i, (part, rc) in enumerate(want):
                assert (got.part[i], got.rc[i]) == (part, rc), \
                    (policy, tier, family, L, len(rows[i]), [x.hex() for x in rows[i]])
            if policy == noted:
                seen[family]['rows'] += len(rows)
                for path in ds.PATHS:
                    seen[family][path] += sum(got.took(path))
                longest = max([longest] + got.block)
    return seen, longest


def assert_paths(tier, seen, longest):
    cases, stats, _ = expected(tier)
    for family, _L, _lc, _rows, target in cases:
        if target:
            assert seen[family][target] > 0, (family, target, dict(seen[family]))
    knife = seen['knife']
    assert knife['verify_failed'] >= KNIFE_SHARE * knife['rows'], dict(knife)
    total = sum(seen.values(), collections.Counter())
    assert all(total[p] > 0 for p in ds.PATHS), dict(total)
    # both sides of the strict compare that closes a stage, and the exact tie
    assert stats['at'] > 0 and stats['late'] > 0 and stats['eq'] > 0, stats
    # a middle block longer than the fixed buffer (MAXS + 64 sub-layers) the balancer used to refuse
    assert longest > tier[0] + 64, longest
    print(f'tier {tier}: longest middle block {longest} sub-layers; paths taken {dict(total)}')


@pytest.mark.parametrize('tier', ds.TIERS)
def test_balancer_families_on_host(tier):
    """Serial and Coop (one lane, PAR iterations forward and reverse) on the host build against the oracle."""
    seen, longest = check_forms(tier, lambda pol, rows, lc, L: ds.host_balance(pol, tier, rows, lc, L),
                                ('serial', 'coop', 'coop_reverse'), 'coop')
    assert_paths(tier, seen, longest)


def test_devsim_cross_compiles_for_sm90a(tmp_path):
    """The device test build compiles with the library's flags on a machine without a GPU."""
    out = ds.compile_devsim(str(tmp_path / 'libdevsim.so'))
    assert os.path.getsize(out) > 0


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return ds.devsim()


@pytest.mark.gpu
@pytest.mark.parametrize('tier', ds.TIERS)
def test_balancer_families_on_gpu(tier):
    """Serial, Lockstep and Coop (WarpCoop) in scratch tier `tier` against the oracle, bit for bit; each family
    reaches its path under Coop, and the bulk round's form takes the middle block, empty stages and the reserved tail
    inside mixed warps."""
    _gpu()
    seen, longest = check_forms(tier, lambda pol, rows, lc, L: ds.device_balance(pol, tier, rows, lc, L),
                                ('serial', 'lockstep', 'coop'), 'coop')
    assert_paths(tier, seen, longest)
    cases, _, _ = expected(tier)
    for family, L, lc, rows, _t in cases:
        if family == 'lockstep_mix':
            got = ds.device_balance('lockstep', tier, rows, lc, L)
            for path in ('middle', 'irregular', 'tail'):
                assert any(got.took(path)), path


# ---- lane primitives ----
SPECIAL = [0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, 1.0, -1.0, 0.5]
NONE = 0x7FFFFFFF          # index of a lane that holds no candidate


def _lane_sets(rng):
    """Per-lane (values, indices) for the reductions: ties everywhere, +-0.0, +-inf, subnormals, lanes without a
    candidate (index NONE, value -inf for a max / +inf for a min)."""
    sets = [([1.0] * 32, list(range(32))), ([0.0, -0.0] * 16, list(range(32))),
            ([-0.0] * 31 + [0.0], list(range(32))), ([-math.inf] * 32, [NONE] * 32)]
    for _ in range(60):
        v = [rng.choice(SPECIAL + [float(rng.randint(-3, 3))]) for _ in range(32)]
        idx = list(range(32))
        rng.shuffle(idx)
        if rng.random() < 0.5:
            idx = [i if rng.random() < 0.7 else NONE for i in idx]
        sets.append((v, idx))
    return sets


@pytest.mark.gpu
def test_warp_reductions_vs_numpy():
    """argmax_first / argmin_first / max_all on doubles and imax_first / imin_first on ints: the extreme value and
    the lowest index among the lanes that hold it, identical in every lane."""
    _gpu()
    rng = np.random.default_rng(5)
    import random
    sets = _lane_sets(random.Random(5))
    for op, pick in (('argmax_first', max), ('argmin_first', min)):
        queries = []
        for v, idx in sets:
            empty = -math.inf if op == 'argmax_first' else math.inf
            queries.append({'dv': [x if i != NONE else empty for x, i in zip(v, idx)], 'iv': idx})
        od, oi = ds.device_lanes(op, queries)
        for q, o_v, o_i in zip(queries, od, oi):
            m = pick(q['dv'])
            want_i = min(i for x, i in zip(q['dv'], q['iv']) if x == m)
            assert (o_i == want_i).all(), (op, q, o_i)
            assert all(x == m for x in o_v), (op, q, o_v)
    od, _ = ds.device_lanes('max_all', [{'dv': v} for v, _ in sets])
    for (v, _), o in zip(sets, od):
        assert all(x == max(v) for x in o)
    for op, pick in (('imax_first', np.max), ('imin_first', np.min)):
        queries = []
        for k in range(80):
            vals = rng.integers(-3, 4, 32) if k % 2 else rng.integers(-2**31, 2**31, 32)
            if k == 0:
                vals = np.zeros(32, dtype=np.int64)
            idx = rng.permutation(32).astype(np.int32)
            queries.append({'dv': vals.astype(np.float64), 'iv': idx, 'vals': vals})
        od, oi = ds.device_lanes(op, queries)
        for q, o_v, o_i in zip(queries, od, oi):
            m = pick(q['vals'])
            assert (o_v == m).all() and (o_i == q['iv'][q['vals'] == m].min()).all(), (op, q)


@pytest.mark.gpu
def test_warp_scan_and_broadcast_vs_numpy():
    _gpu()
    rng = np.random.default_rng(6)
    queries = [{'iv': rng.integers(0, 1 << rng.integers(1, 20), 32).astype(np.int32)} for _ in range(50)]
    queries.append({'iv': np.zeros(32, dtype=np.int32)})
    _, oi = ds.device_lanes('incl_scan', queries)
    for q, o in zip(queries, oi):
        assert (o == np.cumsum(q['iv'])).all()
    _, oi = ds.device_lanes('bcast_last', queries)
    for q, o in zip(queries, oi):
        assert (o == q['iv'][31]).all()


def _tables(rng):
    """Non-decreasing arrays P[0 .. n] like psub: n = 0, n + 1 = 31 / 32 / 33, n = 7 * 255, runs of ties, +-0.0,
    subnormals, +-inf at the ends."""
    out = []
    for n in (0, 1, 30, 31, 32, 33, 64, 100, 7 * 37, 7 * 128, 7 * 255):
        for kind in range(4):
            if kind == 0:
                P = np.cumsum(rng.random(n + 1))
            elif kind == 1:
                P = np.sort(rng.integers(0, max(1, n // 4) + 1, n + 1)).astype(np.float64)
            elif kind == 2:
                P = np.sort(rng.choice([-0.0, 0.0, 5e-324, 1e-310, 1.0], n + 1))
            else:
                P = np.concatenate([[-np.inf], np.cumsum(rng.random(n - 1)), [np.inf]])[:n + 1] if n >= 1 \
                    else np.array([-np.inf])
            out.append(P)
    return out


def _targets(rng, P):
    n = len(P) - 1
    ts = [P[0] - 1.0, P[0], P[n], P[n] + 1.0, P[rng.integers(0, n + 1)], 0.0, -0.0]
    if n >= 1:
        i = rng.integers(0, n)
        ts.append((P[i] + P[i + 1]) / 2)
    return [t for t in ts if not np.isnan(t)]


def _window_ref(P, n, i0, lo, t):
    """OneLane::first_ge_window (metis_coop.cuh)."""
    for k in range(32):
        if i0 + k > n:
            break
        if P[i0 + k] >= t:
            return i0 + k if (k > 0 or i0 <= lo) else -1
    return -1


@pytest.mark.gpu
def test_warp_searches_vs_numpy():
    """first_ge = searchsorted(side='left') over P[0 .. n] (n + 1 when every entry is below t); first_ge_window
    against its one-lane definition, for windows inside, clipped by n, and with the crossing at offset 0 when i0 == lo
    and when i0 > lo."""
    _gpu()
    rng = np.random.default_rng(7)
    queries, wq = [], []
    for P in _tables(rng):
        n = len(P) - 1
        for t in _targets(rng, P):
            queries.append({'P': P, 't': t})
            first = int(np.searchsorted(P, t, side='left'))
            for i0 in {0, max(0, first - 31), max(0, first - 5), first, min(n, first + 1), max(0, n - 3)}:
                for lo in {i0, max(0, i0 - 1)}:
                    wq.append({'P': P, 't': t, 'i0': i0, 'lo': lo})
    _, oi = ds.device_lanes('first_ge', queries)
    for q, o in zip(queries, oi):
        assert (o == np.searchsorted(q['P'], q['t'], side='left')).all(), (len(q['P']), q['t'])
    _, oi = ds.device_lanes('first_ge_window', wq)
    hits = collections.Counter()
    for q, o in zip(wq, oi):
        want = _window_ref(q['P'], len(q['P']) - 1, q['i0'], q['lo'], q['t'])
        assert (o == want).all(), (len(q['P']), q['t'], q['i0'], q['lo'], o[0], want)
        hits['inside' if want >= 0 else 'miss'] += 1
        hits['offset0_refused'] += want < 0 and q['i0'] > q['lo'] and q['i0'] <= len(q['P']) - 1 \
            and q['P'][q['i0']] >= q['t']
    assert hits['inside'] and hits['miss'] and hits['offset0_refused'], hits
