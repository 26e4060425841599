"""The reference's per-candidate stdout (SURVEY.md 8(f)-2), reproduced from values recorded on the GPU.

While it searches, the reference prints every inter-stage plan, every strategy it walks through (the invalid ones
too), the stage performance, each partition attempt with its memory demand / state, the re-weighted performance, the
cost terms and the cost or KeyError of every candidate (search_space/plan.py:207-218,243,247;
model/load_balancer.py:92,132-133,143; model/cost_estimator.py:193,201-203,239-240; cost_het_cluster.py:31,43,48).
``plan_transcript`` yields exactly those lines.  Every number comes from ``metis_het_trace`` (one GPU thread replays
one plan with the search's own evaluator and records the values, metis_b200/csrc/metis_trace.cuh); this module only
walks the strategy chain like search_space/plan.py:192-268 does - integer bookkeeping plus comparisons of the
recorded memory states - to place the ``invalid_strategy`` lines, and formats text.  A debug path: the drop-in CLI
uses it when METIS_VERBOSE=1; a search never does.
"""
from __future__ import annotations

import ctypes as C
from collections import Counter
from dataclasses import dataclass, field
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import native

TAG_END, TAG_STRATEGY, TAG_PERF, TAG_ATTEMPT, TAG_ADJUST, TAG_RESULT, TAG_SPLIT, TAG_COST, TAG_KEYERROR, TAG_FATAL, \
    TAG_OVERFLOW = range(11)


def _as_float(word: int) -> float:
    return float(np.array([word], dtype=np.uint64).view(np.float64)[0])


class _Events:
    """Cursor over one plan's stream of 64-bit words (layout: metis_trace.cuh)."""

    def __init__(self, words: np.ndarray):
        self.w = words
        self.i = 0

    def peek(self) -> int:
        return int(self.w[self.i]) & 0xFF

    def head(self) -> Tuple[int, int, int]:
        v = int(self.w[self.i])
        self.i += 1
        return v & 0xFF, (v >> 8) & 0xFFFFFF, v >> 32

    def ints(self, n: int) -> List[int]:
        out = [int(x) for x in self.w[self.i:self.i + n]]
        self.i += n
        return out

    def floats(self, n: int) -> List[float]:
        out = self.w[self.i:self.i + n].view(np.float64).tolist()
        self.i += n
        return out

    def packed(self, n: int, bits: int) -> List[int]:
        per = 64 // bits
        words = self.ints((n + per - 1) // per)
        return [(words[k // per] >> (bits * (k % per))) & ((1 << bits) - 1) for k in range(n)]


def _memory_capacity(gpu_cluster, rank_types: Sequence[str], groups: Sequence[int]) -> list:
    """model/device_group.py:87-101 (values printed by plan.py:211)."""
    out = []
    for s in range(len(groups)):
        a, b = sum(groups[:s]), sum(groups[:s + 1])
        counts = dict(Counter(rank_types[a:b]))
        out.append(sum([gpu_cluster.get_device_memory_for_device_type(t) * n for t, n in counts.items()]))
    return out


def _rank_types(gpu_cluster, node_sequence) -> List[str]:
    """model/device_group.py:22-32."""
    types: List[str] = []
    for t in node_sequence:
        name = t.name if hasattr(t, 'name') else str(t)
        types += [name] * gpu_cluster.get_num_nodes_by_device_type(name)
    return types[:gpu_cluster.get_total_num_devices()]


def _key_error_text(site: int, a: int, b: int) -> str:
    if site == 1:
        return repr(f'key(tp{a}_bs{b}) not found in profile_data')
    if site == 2:
        return repr(f'tp{a}_bs1')
    if site == 3:
        return repr(f'batch_size({b}) not found in profile_data')
    if site == 4:
        return repr(f'tp{a}_bs{b}')
    if site == 5:
        return repr('key(fb_sync) not found in profile_data')
    return str(a)


def trace_plans(dp, ordinals: np.ndarray, words_per_plan: int = 0) -> np.ndarray:
    """metis_het_trace for the listed ordinals -> uint64 [n, words]."""
    import torch
    n = len(ordinals)
    smax = int(dp.s_struct.max_stage)
    words = words_per_plan or max(256, 64 * (4 * smax + 24))      # ~60 partition attempts of a chain
    with torch.cuda.device(dp.device):
        d_ord = torch.from_numpy(np.ascontiguousarray(ordinals, dtype=np.uint32).view(np.int32)).to(dp.device)
        trace = torch.zeros((max(n, 1), words), dtype=torch.int64, device=dp.device)
        ws = torch.empty(dp.workspace_bytes(0), dtype=torch.uint8, device=dp.device)
        s = torch.cuda.current_stream(dp.device)
        rc = dp.lib.metis_het_trace(C.byref(dp.p_struct), C.byref(dp.s_struct), C.c_void_p(d_ord.data_ptr()), C.c_int64(n),
                                    C.c_void_p(trace.data_ptr()), C.c_int32(words), C.c_void_p(ws.data_ptr()),
                                    C.c_int64(ws.numel()), C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_het_trace')
        s.synchronize()
        return trace[:n].cpu().numpy().view(np.uint64)


@dataclass
class TraceAttempt:
    """One partition attempt of a partition_layer call (model/load_balancer.py:127-143)."""
    attempt: int                  # 1..3
    performance: List[float]      # stage performance fed to this attempt's balancer run
    partition: List[int]          # layer_partition
    demand: List[float]           # stage_memory_demand
    state: List[float]            # memory_state


@dataclass
class TraceCall:
    """One partition_layer call: the valid strategy it was made for and what it printed, in order."""
    tpc: List[int]                # log2(tp) per stage
    performance: Optional[List[float]] = None             # stage_compute_performance (None: fatal before it)
    events: list = field(default_factory=list)            # ('attempt', TraceAttempt) / ('adjust', aux, values or None)
    accepted: int = 0             # attempt number accepted, 0 = layer_partition None
    fatal: Optional[Tuple[int, int]] = None               # (code, aux): the reference aborts inside this call

    @property
    def attempts(self) -> List[TraceAttempt]:
        return [e[1] for e in self.events if e[0] == 'attempt']


@dataclass
class TraceCost:
    """The costing of an accepted call: the data loadbalancer splits, then a KeyError or the cost terms."""
    splits: List[List[int]]
    keyerror: Optional[Tuple[int, int, int]] = None       # (site, a, b)
    terms: Optional[List[float]] = None                   # execution, fb_sync, update, dp, pp, cost


def decode_plan(words: np.ndarray) -> list:
    """One plan's event stream (metis_trace.cuh) -> its items in order: TraceCall, a TraceCost after every accepted
    call, and ('fatal', code, aux) when the reference aborts before a call's strategy is recorded."""
    ev = _Events(words)
    if ev.peek() == TAG_OVERFLOW:
        raise native.MetisNativeError('trace buffer too small for this plan; raise words_per_plan')
    items: list = []
    while True:
        tag, n, aux = ev.head()
        if tag == TAG_END:
            return items
        if tag == TAG_FATAL:
            items.append(('fatal', aux, ev.ints(1)[0]))
            return items
        assert tag == TAG_STRATEGY, tag
        call = TraceCall(ev.packed(n, 8))
        items.append(call)
        tag, n, aux = ev.head()
        if tag == TAG_FATAL:
            call.fatal = (aux, ev.ints(1)[0])
            return items
        assert tag == TAG_PERF
        call.performance = perf = ev.floats(n)
        while True:                                           # partition_layer, load_balancer.py:127-144
            tag, n, aux = ev.head()
            if tag == TAG_FATAL:
                call.fatal = (aux, ev.ints(1)[0])
                return items
            if tag == TAG_RESULT:
                call.accepted = aux
                break
            if tag == TAG_ATTEMPT:
                part = ev.packed(n + 1, 16)
                demand, state = ev.floats(n), ev.floats(n)
                call.events.append(('attempt', TraceAttempt(aux, perf, part, demand, state)))
            elif tag == TAG_ADJUST:
                values = ev.floats(n) if n else None
                call.events.append(('adjust', aux, values))
                if values is not None:
                    perf = values
            else:
                raise AssertionError(f'unexpected trace tag {tag}')
        if not call.accepted:
            continue
        cost = TraceCost([])
        items.append(cost)
        while True:
            tag, n, aux = ev.head()
            if tag == TAG_SPLIT:
                cost.splits.append(ev.ints(n))
            elif tag == TAG_KEYERROR:
                a, b = ev.ints(2)
                cost.keyerror = (aux, a, b)
                break
            elif tag == TAG_COST:
                cost.terms = ev.floats(6)
                break
            else:
                raise AssertionError(f'unexpected trace tag {tag}')


def _fatal(code: int, aux: int):
    return native.MetisNativeError(f'the reference aborts at this plan (fatal code {code}, aux {aux})')


def format_plan(words: np.ndarray, plan, gpu_cluster, max_tp: int, max_bs: int) -> Iterator[str]:
    """Lines of one inter-stage plan (the body of the loop at cost_het_cluster.py:31-48)."""
    items = iter(decode_plan(words))
    yield ''
    yield ''
    yield f'inter_stage_plan: {plan}'
    groups = list(plan.device_groups)
    rank_types = _rank_types(gpu_cluster, plan.node_sequence)
    strategies: Optional[List[Tuple[int, int]]] = None
    memory_state = None
    nrep = 0
    while True:
        if nrep == 1:                                         # plan.py:194-195
            return
        partition = None
        while True:                                           # has_next, plan.py:197-226
            if not strategies:
                strategies = [(g, 1) for g in groups]         # :231-236
            else:
                state = memory_state if memory_state else [1 / dp for dp, _ in strategies]        # :252-255
                nxt = None
                for s in sorted(range(len(state)), key=lambda i: state[i]):                       # :257-266
                    dp, tp = strategies[s]
                    if dp != 1:
                        nxt = list(strategies)
                        nxt[s] = (dp // 2, tp * 2)
                        break
                strategies = nxt
            if not strategies:
                return
            bad = None
            for dp, tp in strategies:                         # _is_valid_strategies, :238-249
                mbs = plan.gbs // dp // plan.batches
                if mbs == 0 or mbs > max_bs:
                    bad = f'invalid_strategy: dp_deg({dp}), batches({plan.batches}), mbs(0)'
                    break
                if tp > max_tp:
                    bad = f'invalid_strategy: tp_deg({tp})'
                    break
            if bad:
                yield bad
                continue
            call = next(items)
            if isinstance(call, tuple):
                raise _fatal(call[1], call[2])
            assert isinstance(call, TraceCall) and len(call.tpc) == len(groups), call
            assert [(g >> t, 1 << t) for g, t in zip(groups, call.tpc)] == strategies, 'device and host disagree on the chain'
            yield f'valid_strategies: {strategies}'
            if call.performance is None:
                raise _fatal(*call.fatal)
            yield f'stage_memory_capacity: {_memory_capacity(gpu_cluster, rank_types, groups)}'
            yield f'stage_compute_performance: {call.performance}'
            for e in call.events:
                if e[0] == 'attempt':
                    yield f'layer_partition: {e[1].partition}'
                    yield f'stage_memory_demand: {e[1].demand}, memory_state: {e[1].state}'
                    last_part, last_state = e[1].partition, e[1].state
                elif e[2] is None:
                    yield 'Even with the reallocation of layers, memory issues persist.'
                else:
                    yield f'adj_stage_compute_performance({e[1]}): {e[2]}'
            if call.fatal is not None:
                raise _fatal(*call.fatal)
            if call.accepted:                                 # success at attempt `accepted`
                partition, memory_state, nrep = last_part, last_state, call.accepted
                yield f'layer_partition: {partition}'
                break
            memory_state = None
            yield 'layer_partition: None'
        # cost_het_cluster.py:38-48
        yield (f'node_sequence: {plan.node_sequence}, device_group: {plan.device_groups}, num_stage: {plan.num_stage}, '
               f'batches: {plan.batches}, gbs: {plan.gbs}, strategies: {strategies}, layer_partition: {partition}')
        cost = next(items)
        for split in cost.splits:
            yield f'data loadbalancer: {split}'
        if cost.keyerror is not None:
            yield f'KeyError: {_key_error_text(*cost.keyerror)}'
        else:
            c = cost.terms
            yield (f'execution_cost: {c[0]}, fb_sync_cost: {c[1]}, parameter_upate_costs: {c[2]}, dp_cost: {c[3]}, '
                   f'pp_cost: {c[4]}')
            yield f'cost: {c[5]}'


def plan_transcript(args, gpu_cluster, profile_data, model_config, layer_load_balancer=None,
                    node_sequences: Optional[Sequence[Sequence]] = None, device=None, chunk: int = 2048) -> Iterator[str]:
    """Every line the reference prints inside cost_het_cluster() (cost_het_cluster.py:24-48), plan by plan."""
    from . import api, search
    from .utils import DeviceType
    if node_sequences is None:
        from itertools import permutations
        node_sequences = list(permutations(set(gpu_cluster.get_device_types())))
    problem, space, _ = api.het_problem(args, gpu_cluster, profile_data, model_config, layer_load_balancer, node_sequences)
    seq_objs = [tuple(t if isinstance(t, DeviceType) else DeviceType[str(t)] for t in seq) for seq in node_sequences]
    dp = search.DeviceProblem(problem, space, device)
    for lo in range(0, space.num_plans, chunk):
        ords = np.arange(lo, min(space.num_plans, lo + chunk), dtype=np.uint32)
        traces = trace_plans(dp, ords)
        for k, o in enumerate(ords.tolist()):
            ns, label, row, batches, codes = space.locate(o)
            plan = api.InterStagePlan(ns_idx=ns, node_sequence=seq_objs[ns], dg_idx=row,
                                      device_groups=[1 << int(c) for c in codes], num_stage=label, batches=batches,
                                      gbs=args.gbs)
            yield from format_plan(traces[k], plan, gpu_cluster, args.max_profiled_tp_degree, args.max_profiled_batch_size)
