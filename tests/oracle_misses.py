"""Out-of-memory partition attempts of the oracle's search (oracle/metis_oracle.py), for the miss tests: every pass of
the partition_layer loop (model/load_balancer.py:127-143) whose memory test fails, with the values it was tried with.
The oracle is not edited: orc.partition_layer and the pieces it calls are wrapped for the duration of one search."""
from contextlib import contextmanager
from typing import Dict, List, NamedTuple, Sequence

from oracle import metis_oracle as orc


class OracleMiss(NamedTuple):
    ordinal: int
    call: int                 # 0-based partition_layer call of the plan
    attempt: int              # 1..3
    deficit: float            # -min(memory_state)
    stage: int                # lowest stage attaining the minimum
    strategies: list          # [(dp, tp)] per stage
    partition: list           # layer_partition of the attempt
    performance: list         # stage performance fed to the attempt's balancer run
    capacity: list            # stage_memory_capacity
    demand: list              # stage_memory_demand
    state: list               # memory_state


@contextmanager
def _patched(module, **fns):
    old = {k: getattr(module, k) for k in fns}
    for k, f in fns.items():
        setattr(module, k, f)
    try:
        yield
    finally:
        for k, f in old.items():
            setattr(module, k, f)


def het_misses(profile: Dict, cluster, model, node_sequences, gbs: int, num_layers: int, variance,
               max_permute_len: int, max_tp: int, max_bs: int, plan_filter=None, corrected: Sequence[str] = ()):
    """orc.het_search recording its out-of-memory attempts: (candidates, counters, misses in reference order)."""
    misses: List[OracleMiss] = []
    cur = {'ordinal': -1, 'call': -1}
    part_layer, balance = orc.partition_layer, orc.layer_compute_balance
    demand_fns = {k: getattr(orc, k) for k in ('stage_memory_demand', 'stage_memory_demand_own_type')}

    def keep(ordinal):
        cur['ordinal'], cur['call'] = ordinal, -1
        return plan_filter is None or plan_filter(ordinal)

    def wrapped(profile_, cluster_, norm_lc, num_layers_, plan, strategies, perf, m_capa, counters=None,
                corrected_=()):
        cur['call'] += 1
        tried = []                                            # (perf, part) of each balancer run, then its demand

        def balance_(num_stage, num_layer, capa_in, *a, **k):
            part = balance(num_stage, num_layer, capa_in, *a, **k)
            tried.append([list(capa_in), list(part), None])
            return part

        def demand_of(fn):
            def f(*a, **k):
                d = fn(*a, **k)
                tried[-1][2] = list(d)
                return d
            return f

        with _patched(orc, layer_compute_balance=balance_, **{k: demand_of(f) for k, f in demand_fns.items()}):
            out = part_layer(profile_, cluster_, norm_lc, num_layers_, plan, strategies, perf, m_capa, counters,
                             corrected_)
        for attempt, (used, part, demand) in enumerate(tried, start=1):
            state = [mc - md for mc, md in zip(m_capa, demand)]
            m = min(state)
            if m < 0:
                misses.append(OracleMiss(cur['ordinal'], cur['call'], attempt, -m, state.index(m), list(strategies),
                                         part, used, list(m_capa), demand, state))
        return out

    with _patched(orc, partition_layer=wrapped):
        cands, counters = orc.het_search(profile, cluster, model, node_sequences, gbs, num_layers, variance,
                                         max_permute_len, max_tp, max_bs, plan_filter=keep, corrected=corrected)
    return cands, counters, misses
