"""Device listing of a plan space's compositions (metis_comps.cuh, metis_listing.cu, metis_b200.listing) and the
window planner that works from its per-stage row totals (flatten.plan_listed_windows).

CPU: the listing's routines, built with g++ (tests/hostsim/listing_sim.cpp), reproduce metis_enum_compositions -
rows per stage count, every record and the pool - on a grid of spaces; the planner's windows cover listed spaces
within the limits and the budget, and the rows written from their records equal the host enumerator's.  GPU (-m gpu):
the CUDA listing equals the host listing window by window, and api.cost_het_cluster through the device listing
equals the host-listed result; 512 GPUs / 1 type / variance 0 / mpl 6 end to end against the pinned oracle.
"""
import ctypes as C
import itertools
import math
import os
import random
import subprocess

import numpy as np
import pytest

import hostsim_util as hs
from conftest import load_golden
from metis_b200 import flatten, native

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, 'hostsim', 'listing_sim.cpp')
SIM_DEPS = [SIM_SRC, os.path.join(HERE, '..', 'metis_b200', 'csrc', 'metis_comps.cuh'),
            os.path.join(HERE, '..', 'include', 'metis_b200.h')]
_sim = []


def _lib_or_skip():
    try:
        return native.load_library()
    except native.MetisNativeError as e:
        pytest.skip(str(e))


def sim():
    """The g++ build of the listing routines (one shared object, rebuilt when its sources change)."""
    if not _sim:
        out = os.path.join(hs.BUILD, 'liblisting_sim.so')
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in SIM_DEPS):
            os.makedirs(hs.BUILD, exist_ok=True)
            tmp = f'{out}.{os.getpid()}.tmp'
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-o', tmp, SIM_SRC])
            os.replace(tmp, out)
        lib = C.CDLL(out)
        lib.listing_sim_stages.restype = C.c_int32
        lib.listing_sim_stages.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_void_p]
        lib.listing_sim_window.restype = C.c_int32
        lib.listing_sim_window.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_void_p]
        _sim.append(lib)
    return _sim[0]


class SimListing:
    """flatten.ListedWindow's listing, on the host build: same interface as metis_b200.listing.DeviceListing."""

    def __init__(self, gpus, cap, variance, mpl):
        self.args = (1, cap, gpus, float(variance), mpl)
        self.rows_per_stage = np.zeros(cap, dtype=np.int64)
        self.comps_per_stage = np.zeros(cap, dtype=np.int64)
        self.max_groups = sim().listing_sim_stages(*self.args, self.rows_per_stage.ctypes.data,
                                                   self.comps_per_stage.ctypes.data)

    def _window(self, ranges, write):
        ranges = np.ascontiguousarray(ranges, dtype=native.RANGE_DTYPE)
        sizes = np.zeros(2, dtype=np.int64)
        assert sim().listing_sim_window(*self.args, ranges.ctypes.data, len(ranges), None, None, sizes.ctypes.data) == 0
        if not write:
            return int(sizes[0]), int(sizes[1])
        recs = np.zeros(max(int(sizes[0]), 1), dtype=native.COMP_DTYPE)
        pool = np.zeros(max(int(sizes[1]), 16), dtype=np.uint8)
        assert sim().listing_sim_window(*self.args, ranges.ctypes.data, len(ranges), recs.ctypes.data, pool.ctypes.data,
                                        sizes.ctypes.data) == 0
        return recs[:int(sizes[0])], pool

    def size(self, ranges):
        return self._window(ranges, False)

    def emit(self, ranges):
        return self._window(ranges, True)

    def window_space(self, window):
        recs, pool = self.emit(window.ranges)
        lay = window.layout
        return flatten.FlatPlanSpace(lay.num_plans, lay.blocks, lay.batches, lay.rows,
                                     rows_total_bytes=lay.rows_total_bytes, comp_recs=recs, comp_pool=pool)


def host_window(recs, pool, ranges):
    """The records and pool of ``ranges`` cut from the host listing (metis_enum_compositions over the whole space):
    its slices clipped to each range, row offsets in the ranges' layout, one pool entry per composition and range."""
    out, parts, byte, po = [], [], 0, 0
    for S, _, r0, r1 in ranges.tolist():
        sel = recs[recs['stages'] == S]
        row0 = (sel['row_offset'] - sel['row_offset'][0]) // S        # the stage's first record holds its row 0
        keep = np.nonzero((row0 < r1) & (row0 + sel['num_rows'] > r0))[0]
        last = None
        for k in keep.tolist():
            r = sel[k].copy()
            f, e = max(int(row0[k]), r0), min(int(row0[k]) + int(r['num_rows']), r1)
            if int(r['pool_offset']) != last:
                last = int(r['pool_offset'])
                entry = po
                size = int(r['num_groups']) + S
                parts.append(pool[last:last + size])
                po += size
            r['first_row'] = int(r['first_row']) + f - int(row0[k])
            r['num_rows'] = e - f
            r['row_offset'] = byte + (f - r0) * S
            r['pool_offset'] = entry
            out.append(r)
        byte += (r1 - r0) * S
    rec = np.array(out, dtype=native.COMP_DTYPE) if out else np.zeros(0, dtype=native.COMP_DTYPE)
    return rec, (np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8))


def _rows_from(recs, pool, nbytes):
    rows = np.zeros(max(int(nbytes), 16), dtype=np.uint8)
    rc = hs.hostsim().hostsim_generate_rows(C.c_void_p(recs.ctypes.data), C.c_int64(len(recs)),
                                            C.c_void_p(pool.ctypes.data), C.c_void_p(rows.ctypes.data))
    assert rc == 0
    return rows


# ---- the listing against metis_enum_compositions ------------------------------------------------------------------
GRID_GPUS = [8, 16, 24, 48, 96, 100, 128]


def _caps(gpus):
    return sorted({min(gpus, L) for L in (1, 2, 96, 97, 128)})


def _compare_listing(gpus, cap, variance, mpl):
    counts, recs, pool, most = flatten.enumerate_compositions(1, cap + 1, gpus, variance, mpl)
    lst = SimListing(gpus, cap, variance, mpl)
    assert lst.rows_per_stage.tolist() == counts[:cap].tolist(), (gpus, cap, variance, mpl)
    assert lst.max_groups == max([0] + recs['num_groups'][recs['stages'] <= cap].tolist())
    assert flatten.count_compositions(gpus, cap, variance, mpl) == int(lst.comps_per_stage.sum())
    host = recs[recs['stages'] <= cap]
    assert int(lst.comps_per_stage.sum()) == len(np.unique(host['pool_offset']))
    if lst.max_groups > native.METIS_MAX_PERMUTE_GROUPS:
        return
    ranges = np.array([(S, 0, 0, int(n)) for S, n in enumerate(counts[:cap].tolist(), 1) if n], dtype=native.RANGE_DTYPE)
    got, gpool = lst.emit(ranges)
    assert len(got) == len(host)
    assert (got == host).all(), (gpus, cap, variance, mpl)
    pbytes = int(host['pool_offset'][-1] + host['num_groups'][-1] + host['stages'][-1]) if len(host) else 0
    assert (gpool[:pbytes] == pool[:pbytes]).all()
    # a cut at any row: the host listing's slices clipped to the range
    rng = random.Random(gpus * 1000 + cap * 10 + mpl)
    cut = []
    for S, _, _, n in ranges.tolist():
        a = rng.randrange(n)
        cut.append((S, 0, a, rng.randrange(a, n) + 1))
    cut = np.array(cut, dtype=native.RANGE_DTYPE)
    got, gpool = lst.emit(cut)
    want, wpool = host_window(recs, pool, cut)
    assert (got == want).all() and (gpool[:wpool.size] == wpool).all(), (gpus, cap, variance, mpl)


@pytest.mark.parametrize('gpus', GRID_GPUS)
def test_listing_equals_host_enumerator(gpus):
    """Unranking, merging and counting reproduce metis_enum_compositions: rows per stage count, every record's
    (stages, num_groups, first_row, num_rows, row_offset, pool_offset) and the pool bytes, for variance 0 / 0.5 / 1,
    mpl 1-6 and caps 1, 2, 96, 97 and 128 (where the GPU count allows); and the records of ranges cut at random rows
    are the host's slices clipped to them."""
    _lib_or_skip()
    for variance, mpl in itertools.product((0, 0.5, 1), range(1, 7)):
        for cap in _caps(gpus):
            _compare_listing(gpus, cap, variance, mpl)


@pytest.mark.parametrize('gpus,cap,variance,mpl', [(256, 96, 0, 4), (256, 128, 1, 6), (512, 96, 1, 4), (200, 97, 0.5, 5)])
def test_listing_equals_host_enumerator_large(gpus, cap, variance, mpl):
    _lib_or_skip()
    _compare_listing(gpus, cap, variance, mpl)


def test_listing_reports_too_many_groups():
    """A composition of more merged groups than the row kernel handles is counted and reported, never written."""
    _lib_or_skip()
    lst = SimListing(64, 64, 0, 64)
    assert lst.max_groups > native.METIS_MAX_PERMUTE_GROUPS
    S = 40                                                    # 40 stages of 1 or 2 GPUs: up to 40 groups
    sizes = np.zeros(2, dtype=np.int64)
    ranges = np.array([(S, 0, 0, int(lst.rows_per_stage[S - 1]))], dtype=native.RANGE_DTYPE)
    assert sim().listing_sim_window(*lst.args, ranges.ctypes.data, 1, None, None, sizes.ctypes.data) == -1


# ---- the planner on listed spaces ---------------------------------------------------------------------------------
def _space_args(w):
    return (math.factorial(len(w.device_types())), sum(n for _, n in w.nodes), w.gbs, w.num_layers, w.variance,
            w.max_permute_len)


def _listed(args, corrected=()):
    ns, gpus, gbs, layers, variance, mpl = args
    cap = min(gpus, layers)
    lst = SimListing(gpus, cap, variance, mpl)
    return lst, flatten.listed_plan_space(ns, gpus, gbs, layers, lst.rows_per_stage, corrected)


def _check_listed_windows(space, windows, budget, model, full_tables):
    base = 0
    for w in windows:
        lay = w.layout
        assert w.base == base and lay.num_plans > 0
        assert lay.num_plans <= flatten.MAX_SEARCH_PLANS and lay.rows_total_bytes <= flatten.MAX_SEARCH_ROW_BYTES
        assert (np.diff(lay.blocks['first_ordinal']) > 0).all()
        w.sized()
        assert w.num_recs <= w.rec_bound
        if budget is not None and w.layout.num_plans > flatten.METIS_COMP_SLICE_ROWS * len(space.batches):
            assert flatten.window_bytes(w.space, *model) <= budget
        base += lay.num_plans
    assert base == space.num_plans
    for w in windows if full_tables is not None else ():
        sp = w.space
        assert sp.num_plans == w.layout.num_plans and len(sp.comp_recs) == w.num_recs
        rows = _rows_from(sp.comp_recs, sp.comp_pool, sp.rows_total_bytes)
        for b, blk in enumerate(sp.blocks):
            S, n, at = int(blk['num_stage']), int(blk['num_rows']), int(blk['rows_offset'])
            r0 = int(w.row_base[b])
            assert (rows[at:at + n * S].reshape(n, S) == full_tables[S][1][r0:r0 + n]).all(), (w.base, b)


LISTED_SPACES = {
    'c3_mpl4': ('c3_homo64_mpl4', ()), 'c3_mpl6': ('c3_homo64_mpl6', ()), 'c4': ('c4_het128', ()),
    'c4_mpl6': ('c4_het128_mpl6', ()), 'q1_corrected': ('c4_het128', ('Q1',)), 'sweep_n32_t4': ('sweep_n32_t4', ()),
}


@pytest.mark.parametrize('parts', [1, 3, 11, 0], ids=['one', 'three', 'eleven', 'per_slice'])
@pytest.mark.parametrize('key', list(LISTED_SPACES))
def test_listed_windows_cover_the_space(key, parts):
    """The planner's windows cover a listed space in ordinal order within the limits and the budget; its block list
    equals the host-listed space's, plan_at equals the whole space's ordinal -> plan, and the rows written from each
    window's records equal the host enumerator's tables."""
    from metis_b200.workloads import WORKLOADS
    _lib_or_skip()
    name, corrected = LISTED_SPACES[key]
    args = _space_args(WORKLOADS[name])
    lst, space = _listed(args, corrected)
    ref = flatten.build_device_plan_space(*args, corrected=corrected)
    assert space.num_plans == ref.num_plans
    for f in ('first_ordinal', 'rows_offset', 'num_rows', 'ns_idx', 'label_stage', 'num_stage'):
        assert (space.blocks[f] == ref.blocks[f]).all(), f
    model = (56.5, 1.25, 20.0)
    if parts == 0:
        if space.num_plans > 2_000_000:
            pytest.skip('one window per slice: kept to the smaller spaces')
        budget = 0
    elif parts == 1:
        budget = float('inf')
    else:
        budget = flatten.window_bytes(ref, *model) / parts
    windows = flatten.plan_listed_windows(space, budget, *model, listing=lst)
    if parts == 1:
        assert len(windows) == 1
        assert (windows[0].space.comp_recs == ref.comp_recs[np.isin(ref.comp_recs['stages'],
                                                                    space.blocks['num_stage'])]).all()
    _check_listed_windows(space, windows, budget, model, ref.tables)
    rng = random.Random(7)
    picks = {rng.randrange(space.num_plans) for _ in range(300)} | {w.base for w in windows}
    picks |= {w.base + w.layout.num_plans - 1 for w in windows}
    bases = [w.base for w in windows]
    for o in sorted(picks):
        w = windows[int(np.searchsorted(bases, o, side='right')) - 1]
        ns, label, dg, batches, _codes = ref.locate(o)
        assert w.plan_at(o)[:4] == (ns, label, dg, batches), o


def _range_row(w, at):
    """Byte offset in a listed window's rows -> (stage count, row of its table), through the window's ranges."""
    byte = 0
    for S, _, r0, r1 in w.ranges.tolist():
        size = (r1 - r0) * S
        if at < byte + size:
            return S, r0 + (at - byte) // S
        byte += size
    raise AssertionError(at)


@pytest.mark.parametrize('mpl', [4, 6])
def test_listed_windows_512_gpus(mpl):
    """512 GPUs / 1 type / variance 0 (BASELINE configs[4]) at mpl 4 (1.5e9 plans) and mpl 6 (2.1e10 plans), planned from
    the listing's row totals with an 80 GB-class budget: windows within the limits, one arena for all within the budget,
    every ordinal once.  At every window's first and last plan and at seeded samples, the window's layout maps the plan
    to its row, and the row written from the emitted record equals metis_enum_device_groups (mpl 4) or the row written
    from the host listing's record of that stage count (mpl 6)."""
    _lib_or_skip()
    lst, space = _listed((1, 512, 512, 96, 0, mpl))
    if mpl == 4:
        assert space.num_plans == 1473825430
    model, budget = (56.5, 1.25, 20.0), 60e9
    windows = flatten.plan_listed_windows(space, budget, *model, listing=lst)
    assert len(windows) >= 3
    base = 0
    for w in windows:
        assert w.base == base
        assert w.layout.num_plans <= flatten.MAX_SEARCH_PLANS and w.layout.rows_total_bytes <= flatten.MAX_SEARCH_ROW_BYTES
        base += w.layout.num_plans
    assert base == space.num_plans
    peak = (max(w.layout.num_plans for w in windows) * model[0]
            + max(w.layout.rows_total_bytes for w in windows) * model[1] + max(w.rec_bound for w in windows) * model[2])
    assert peak <= budget
    rng = random.Random(512 + mpl)
    picks = {rng.randrange(space.num_plans) for _ in range(40)}
    for w in windows:
        picks |= {w.base, w.base + w.layout.num_plans - 1}
    ndiv = len(space.batches)
    firsts = space.blocks['first_ordinal']
    by_stage = {}
    bases = [w.base for w in windows]
    for o in sorted(picks):
        blk = space.blocks[int(np.searchsorted(firsts, o, side='right')) - 1]
        row, div = divmod(o - int(blk['first_ordinal']), ndiv)
        w = windows[int(np.searchsorted(bases, o, side='right')) - 1]
        ns, label, dg, batches, S, at = w.plan_at(o)
        assert (ns, label, dg, batches, S) == (int(blk['ns_idx']), int(blk['label_stage']), row,
                                               int(space.batches[div]), int(blk['num_stage'])), o
        assert _range_row(w, at) == (S, row), o
        recs, pool = lst.emit(np.array([(S, 0, row, row + 1)], dtype=native.RANGE_DTYPE))
        assert len(recs) == 1 and int(recs['num_rows'][0]) == 1
        by_stage.setdefault(S, []).append((o, row, _rows_from(recs, pool, S)[:S]))
    assert max(by_stage) >= 90
    for S, items in by_stage.items():
        if mpl == 4:
            table = flatten.enumerate_device_groups(S, 512, 0, mpl)
            for o, row, codes in items:
                assert (codes == table[row]).all(), (o, S, row)
        else:
            _, hrecs, hpool, _ = flatten.enumerate_compositions(S, S, 512, 0, mpl)
            starts = hrecs['row_offset'] // S
            for o, row, codes in items:
                k = int(np.searchsorted(starts, row, side='right')) - 1
                one = hrecs[k:k + 1].copy()
                one['row_offset'] = 0
                rows = _rows_from(one, hpool, int(one['num_rows'][0]) * S)
                at = (row - int(starts[k])) * S
                assert (codes == rows[at:at + S]).all(), (o, S, row)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    native.load_library()
    return torch


# the spaces of the row kernel's GPU test (test_gpu_parity), then 512 GPUs
ROW_SPACES = [(8, 0.5, 4), (16, 1, 6), (32, 0.5, 6), (32, 0, 4), (64, 1, 4), (64, 0.5, 6), (128, 1, 6), (128, 0, 4),
              (256, 0, 4), (512, 0, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize('gpus,variance,mpl', ROW_SPACES)
def test_device_listing_equals_host_listing(gpus, variance, mpl):
    """The CUDA listing's rows per stage count, and the records and pool of windows (the whole space, and windows cut by
    the planner at arbitrary rows) equal the host listing's for the same row ranges; the rows the GPU writes from
    them are byte-identical to the rows written from the host's records."""
    torch = _gpu()
    from metis_b200 import listing as listing_mod
    ns, gbs, layers = 1, gpus, 96
    key = (gpus, variance, mpl)
    cap = min(gpus, layers)
    counts, recs, pool, most = flatten.enumerate_compositions(1, cap + 1, gpus, variance, mpl)
    if most > native.METIS_MAX_PERMUTE_GROUPS:
        pytest.skip('a composition of more merged groups than the row kernel handles')
    space = flatten.listed_plan_space(ns, gpus, gbs, layers, counts[:cap])
    lst = listing_mod.DeviceListing(gpus, cap, variance, mpl, 'cuda:0', max_ranges=ns * cap + 1)
    assert lst.rows_per_stage.tolist() == counts[:cap].tolist()
    assert lst.max_groups == most or lst.max_groups == max(recs['num_groups'][recs['stages'] <= cap])
    whole = flatten.whole_space_ranges(space)
    windows = [whole] + [w.ranges for w in flatten.plan_listed_windows(space, space.num_plans / 5 + 1, listing=lst)]
    lib = native.load_library()
    for ranges in windows:
        got, gpool = lst.emit(ranges)
        want, wpool = host_window(recs, pool, ranges)
        assert len(got) == len(want) and (got == want).all(), key
        assert (gpool[:wpool.size] == wpool).all(), key
        if len(got) > 400_000:
            continue                                          # the rows of the big spaces: whole space only, below
        nbytes = int(((ranges['end_row'] - ranges['first_row']) * ranges['stages']).sum())
        dev = {}
        for name, arr in (('recs', got), ('pool', gpool)):
            dev[name] = torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1).copy()).to('cuda:0')
        out = torch.zeros(max(nbytes, 16), dtype=torch.uint8, device='cuda:0')
        rc = lib.metis_generate_rows(C.c_void_p(dev['recs'].data_ptr()), C.c_int64(len(got)),
                                     C.c_void_p(dev['pool'].data_ptr()), C.c_void_p(out.data_ptr()), None)
        native.check(rc, 'metis_generate_rows')
        torch.cuda.synchronize()
        assert (out.cpu().numpy()[:nbytes] == _rows_from(want, wpool, nbytes)[:nbytes]).all(), key


def _api_run(name, workload_dir):
    import test_windowed_search as tw
    meta, arr = load_golden(name)
    w, root, _ = workload_dir(name)
    return tw._api_call(name, root, meta, w), meta, arr


def _force_listed_windows(monkeypatch, parts):
    """cost_het_cluster through the device listing in about ``parts`` windows."""
    from metis_b200 import api, search
    monkeypatch.setattr(api, '_ONE_SEARCH_BYTES', 0)
    monkeypatch.setattr(api, '_MIN_WINDOW_BYTES', 0)
    monkeypatch.setattr(api, '_engine_bytes', lambda key: 0)
    monkeypatch.setattr(search, 'window_budget', lambda dev, fixed: 0.0)
    real = flatten.plan_listed_windows

    def plan(space, budget, plan_bytes=1.0, row_bytes=0.0, rec_bytes=0.0, listing=None):
        rows = sum({int(b['num_stage']): int(b['num_rows']) for b in space.blocks}.values())   # the record bound
        return real(space, space.num_plans / parts * plan_bytes + space.rows_total_bytes * row_bytes + rows * rec_bytes
                    + 64 * len(space.batches) * plan_bytes, plan_bytes, row_bytes, rec_bytes, listing=listing)
    monkeypatch.setattr(flatten, 'plan_listed_windows', plan)


@pytest.mark.gpu
@pytest.mark.parametrize('name,factor', [('c3_homo64_mpl4', 1), ('c3_homo64_mpl4', 2 ** 31 - 1), ('c4_het128', 0)],
                         ids=['c3_bulk_round_then_chains', 'c3_chain_kernel_only', 'c4_default'])
def test_api_device_listing_equals_host_listing(name, factor, workload_dir, monkeypatch):
    """cost_het_cluster() with the device listing forced (threshold 0), in one search and in forced windows, equals the
    host-listed result in the same schedule: len, every tuple (or the reference-sampled ordinals), ranked(50),
    best(), counters."""
    _gpu()
    from metis_b200 import api
    run, meta, arr = _api_run(name, workload_dir)
    shard = native.MetisShard
    monkeypatch.setattr(native, 'MetisShard', lambda rank, world, tile, _r: shard(rank, world, tile, factor))
    api.release_engines()
    ref = run()
    assert ref.summary['listing'] == 'host'
    monkeypatch.setattr(api, '_DEVICE_LISTING_COMPS', 0)
    api.release_engines()
    one = run()
    assert one.summary['listing'] == 'device' and one.summary['num_windows'] == 1
    _force_listed_windows(monkeypatch, 5)
    win = run()
    assert win.summary['listing'] == 'device' and win.summary['num_windows'] >= 3
    monkeypatch.undo()                                        # the ranking below sizes its sort from the real budget
    api.release_engines()
    for got in (one, win):
        for k in ('num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror'):
            assert got.summary[k] == ref.summary[k], k
        assert len(got) == len(ref)
        assert (got.costs.view(np.uint64) == ref.costs.view(np.uint64)).all()
        assert got.best() == ref.best()
        if 'sample' not in arr:
            assert list(got) == list(ref)
        else:
            idx = np.linspace(0, len(ref) - 1, 3000).astype(np.int64)
            assert got.candidates.tuples(idx) == ref.candidates.tuples(idx)
        assert got.ranked(50) == ref.ranked(50)


@pytest.mark.gpu
def test_api_device_listing_fatal_plan(workload_dir, monkeypatch):
    """fatal_gbs96 (the reference aborts with KeyError 'tp1_bs3'): the same KeyError through the device listing, in one
    search and in forced windows."""
    _gpu()
    from metis_b200 import api
    run, _, _ = _api_run('fatal_gbs96', workload_dir)
    with pytest.raises(KeyError) as host:
        run()
    monkeypatch.setattr(api, '_DEVICE_LISTING_COMPS', 0)
    with pytest.raises(KeyError) as one:
        run()
    _force_listed_windows(monkeypatch, 4)
    with pytest.raises(KeyError) as win:
        run()
    assert str(one.value) == str(win.value) == str(host.value)
    monkeypatch.undo()
    api.release_engines()


@pytest.mark.gpu
def test_512_gpus_one_type_variance0_mpl6(tmp_path):
    """512 GPUs / 1 type / variance 0 / mpl 6 (2.1e10 plans) end to end through the device listing: every window's
    first and last plan, one row of every block with every divisor of gbs, 200 uniform ordinals and the winner equal
    the pinned oracle bit for bit.  Writes a JSON report (METIS_LISTING_REPORT): wall time, timings, windows, peak
    device memory, host peak RSS, counters."""
    torch = _gpu()
    import json
    import resource
    import time
    import test_windowed_search as tw
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    from metis_b200.workloads import materialize, profile_file_order, sweep_workload
    w = sweep_workload(512, 1, 0, 6)
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
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
    s = res.summary
    assert s['listing'] == 'device' and s['fatal_ordinal'] == 2 ** 64 - 1
    assert s['num_windows'] >= 3 and s['windows_searched'] == s['num_windows']
    cand = res.candidates
    windows = cand.windows
    space = flatten.listed_plan_space(1, 512, w.gbs, w.num_layers, windows[0].listing.rows_per_stage)
    assert s['num_plans'] == space.num_plans == sum(x.layout.num_plans for x in windows)
    best = res.best()
    rng = random.Random(5126)
    picks = set()
    for x in windows:
        picks |= {x.base, x.base + x.layout.num_plans - 1}
    ndiv = len(space.batches)
    for blk in space.blocks:
        first, n = int(blk['first_ordinal']), int(blk['num_rows'])
        row = rng.randrange(n)
        picks |= {first + row * ndiv + d for d in range(ndiv)}
    picks |= {rng.randrange(space.num_plans) for _ in range(200)}
    if best is not None:
        picks.add(int(res._best_key[0]))
    bad = tw._oracle_check(w, root, order, space, windows, cand.records, cand.bases, cand.firsts, cand, sorted(picks))
    report = {'gpu': torch.cuda.get_device_name(0), 'wall_s': wall, 'num_plans': s['num_plans'],
              'num_windows': s['num_windows'], 'num_candidates': len(res),
              'peak_allocated_bytes': int(torch.cuda.max_memory_allocated()),
              'peak_reserved_bytes': int(torch.cuda.max_memory_reserved()), 'host_peak_rss_bytes': rss,
              'counters': {k: s[k] for k in ('num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror')},
              'best': [best[6], best[3]] if best else None, 'best_key': list(res._best_key) if res._best_key else None,
              'checked_plans': len(picks), 'mismatches': bad[:20], 'timings': res.timings}
    out = os.environ.get('METIS_LISTING_REPORT')
    if out:
        with open(out, 'w') as fh:
            json.dump(report, fh, indent=1)
    print(json.dumps(report))
    assert not bad
