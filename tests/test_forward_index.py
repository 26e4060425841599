"""The chain kernel's forward prediction through the bucket index of psub against the window-probe walk it replaces,
on the host build (tests/hostsim/forward_index_sim.cpp): for every stage of every run, the predicted interval start
and end (w.first, w.fe), the replay's verdict and, when it verifies, the residual capacities must be identical.  The
index lookup itself is checked against np.searchsorted on random and tie-heavy running sums."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import balancer_cases as bc
import devsim_util as ds
import hostsim_util as hs
from conftest import load_golden
from metis_b200 import flatten, native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'hostsim', 'forward_index_sim.cpp')
CSRC = os.path.join(HERE, '..', 'metis_b200', 'csrc')
NAMES = ['runs', 'indexed', 'mismatch', 'steps', 'tail', 'step0', 'step1', 'window', 'far', 'first_ge_index',
         'first_ge_today', 'verified']
_libs = {}


def sim(tier):
    tier = (int(tier[0]), int(tier[1]), bool(tier[2]) if len(tier) > 2 else False)
    if tier not in _libs:
        out = os.path.join(hs.BUILD, f'libforward_index_s{tier[0]}_l{tier[1]}_one{int(tier[2])}.so')
        deps = [SRC] + [os.path.join(CSRC, f) for f in ('metis_eval.cuh', 'metis_coop.cuh')]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared',
                                   f'-DFI_MAXS={tier[0]}', f'-DFI_MAXL={tier[1]}', f'-DFI_ONE={int(tier[2])}',
                                   '-o', tmp, SRC])
            os.replace(tmp, out)
        lib = C.CDLL(out)
        lib.fi_instantiation.restype = C.c_uint64
        assert lib.fi_instantiation() == hs.tier_code(tier)
        assert lib.fi_num_counters() == len(NAMES)
        _libs[tier] = lib
    return _libs[tier]


def _counters(arr):
    return dict(zip(NAMES, (int(v) for v in arr)))


def rows_walks(tier, rows, lc, L):
    """Both walks on capacity rows; returns the counters."""
    lib = sim(tier)
    stride = max(len(r) for r in rows)
    capa = np.zeros((len(rows), stride))
    for i, r in enumerate(rows):
        capa[i, :len(r)] = r
    ns = np.array([len(r) for r in rows], dtype=np.int32)
    lc = np.ascontiguousarray(lc, dtype=np.float64)
    out = np.zeros(len(NAMES), dtype=np.int64)
    rc = lib.fi_rows(C.c_void_p(capa.ctypes.data), C.c_void_p(ns.ctypes.data), C.c_int64(len(rows)),
                     C.c_int32(stride), C.c_void_p(lc.ctypes.data), C.c_int32(len(lc)), C.c_int32(L),
                     C.c_void_p(out.ctypes.data))
    assert rc == 0
    return _counters(out)


def search_walks(problem, space, tier):
    """Both walks at every balancer run the chain kernel makes; returns the counters."""
    lib = sim(tier)
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.rows)
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    s = space.as_struct(lambda n: keep[n].ctypes.data)
    out = np.zeros(len(NAMES), dtype=np.int64)
    assert lib.fi_search(C.byref(p), C.byref(s), C.c_void_p(out.ctypes.data)) == 0
    return _counters(out)


def _golden_problem(name, workload_dir):
    lib = native.load_library()
    meta, _arr = load_golden(name)
    w, root, digest = workload_dir(name)
    assert digest == meta['inputs_sha256']
    cluster, profile, _types, cfg = hs.load_inputs(root, 'profile', meta['file_order'], w.num_layers, w.hidden_size,
                                                   w.sequence_length, w.vocab_size)
    seqs = [tuple(s) for s in meta['node_sequences']]
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
    space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance,
                                     w.max_permute_len, lib)
    tier = hs.gpu_tier(int(space.blocks['num_stage'].max()), w.num_layers, len(problem.type_names))
    return problem, space, tier


@pytest.mark.parametrize('tier', ds.TIERS)
def test_index_walk_equals_window_walk_on_balancer_cases(tier):
    """Every family and scratch tier (MAXS, MAXL) of tests/balancer_cases.py (knife-edge capacities, empty stages, ties, zero demands,
    shapes, the reserved tail)."""
    cases, _stats = bc.all_cases(tier)
    total = {}
    for family, L, lc, rows, _target in cases:
        c = rows_walks(tier, rows, lc, L)
        assert c['mismatch'] == 0, (family, L, c)
        for k, v in c.items():
            total[k] = total.get(k, 0) + v
    assert total['runs'] > 0 and total['indexed'] > 0 and total['steps'] > 0, total
    print(f'tier {tier}: {total}')


# chain-kernel runs of whole searches: a homogeneous and a heterogeneous cluster, a rough profile, 255 layers
@pytest.mark.parametrize('name', ['c3_homo64_mpl4', 'c2_het16', 'rough_t3', 'lim_s128_l255'])
def test_index_walk_equals_window_walk_on_chain_runs(name, workload_dir):
    problem, space, tier = _golden_problem(name, workload_dir)
    c = search_walks(problem, space, tier)
    assert c['runs'] > 0 and c['indexed'] == c['runs'], c
    assert c['mismatch'] == 0, c
    lookups = c['step0'] + c['step1'] + c['window'] + c['far']
    assert lookups + c['tail'] == c['steps'], c
    print(f'{name}: {c}')


def _lcs(rng):
    """Normalised layer weights: random, equal, and tie-heavy (zero-weight layers, single and in runs, first and
    last), at 1 .. 255 layers."""
    out = []
    for L in (1, 2, 3, 5, 31, 96, 128, 200, 255):
        out.append(rng.random(L) + 0.01)
        out.append(np.ones(L))
        z = rng.random(L) + 0.01
        z[rng.random(L) < 0.4] = 0.0
        z[0] = z[-1] = 0.0
        if z.sum() == 0.0:
            z[L // 2] = 1.0
        out.append(z)
        h = np.full(L, 0.3 / max(1, L - 1))
        h[L // 3] = 0.7
        out.append(h)
    return [v / v.sum() for v in out]


def test_lookup_vs_searchsorted():
    """psub_lookup = max(searchsorted(P, t, 'left'), lo) for every t <= P[lim] and 1 <= lo <= lim: the entries
    themselves, halfway between neighbours, one ulp around them, below the start of the window and at random."""
    lib = sim(hs.LIMITS)
    rng = np.random.default_rng(11)
    checked = 0
    for lc in _lcs(rng):
        L = len(lc)
        N = 7 * L
        lim = N - 1 - 7
        if lim < 1:
            continue
        lc = np.ascontiguousarray(lc)
        P = np.zeros(N + 1)
        scale = C.c_double()
        assert lib.fi_psub(C.c_void_p(lc.ctypes.data), C.c_int32(L), C.c_int32(L), C.c_void_p(P.ctypes.data),
                           C.byref(scale)) == N
        assert scale.value > 0.0 and (np.diff(P) >= 0).all()
        pts = np.concatenate([P[:lim + 1], (P[:lim] + P[1:lim + 1]) / 2, np.nextafter(P[:lim + 1], np.inf),
                              np.nextafter(P[:lim + 1], -np.inf), rng.random(200) * P[lim], [0.0, -1.0]])
        ts = pts[pts <= P[lim]]
        los = rng.integers(1, lim + 1, len(ts)).astype(np.int32)
        los[::3] = 1
        want = np.maximum(np.searchsorted(P, ts, side='left'), los)
        got = np.zeros(len(ts), dtype=np.int32)
        assert lib.fi_lookup(C.c_void_p(lc.ctypes.data), C.c_int32(L), C.c_int32(L), C.c_void_p(ts.ctypes.data),
                             C.c_void_p(los.ctypes.data), C.c_int64(len(ts)), C.c_void_p(got.ctypes.data)) == 0
        assert (got == want).all(), (L, ts[got != want][:5], got[got != want][:5], want[got != want][:5])
        checked += len(ts)
    assert checked > 10000


def test_no_index_without_a_non_decreasing_psub():
    """A negative, NaN or infinite layer weight, or all weights zero, leave the index empty (the walk probes as
    without one); the derived psub of such weights is what the walk would search."""
    lib = sim(hs.LIMITS)
    for bad in ([0.5, -0.1, 0.6], [0.5, np.nan, 0.5], [0.5, np.inf, 0.5], [0.0, 0.0, 0.0]):
        lc = np.ascontiguousarray(bad, dtype=np.float64)
        P = np.zeros(7 * len(lc) + 1)
        scale = C.c_double(1.0)
        assert lib.fi_psub(C.c_void_p(lc.ctypes.data), C.c_int32(len(lc)), C.c_int32(len(lc)),
                           C.c_void_p(P.ctypes.data), C.byref(scale)) == 7 * len(lc)
        assert scale.value == 0.0, bad
