"""Breakdown-returning twins of the oracle's cost and candidate walk (oracle/metis_oracle.py), for the cost breakdown
tests: what HeteroCostEstimator.get_cost adds up (model/cost_estimator.py:199-244) and the values of the accepted
partition attempt (model/load_balancer.py:121-144).  Built from the oracle's own pieces; the checks that these twins
give the oracle's costs and partitions bit for bit are in tests/test_breakdown.py."""
import math
from typing import Dict, List, Sequence, Tuple

from oracle import metis_oracle as orc


def het_cost_terms(profile: Dict, cluster, model, plan: dict, strategies, part, rank_types: Sequence[str],
                   max_profiled_bs: int):
    """orc.het_cost split into its terms: ([execution, fb_sync, max update, max dp, pp, batch generate], per-stage
    dict of lens / dp / update / pp over the costed stages).  Raises KeyError like the reference."""
    pp_bw, dp_bw = orc.het_bandwidths(cluster, plan)
    groups = plan['device_groups']
    lens, dp_costs, upd, pps = [], [], [], []
    pp_cost, fb_sync = 0., 0.
    for s, (dp, tp) in zip(range(plan['num_stage']), strategies):
        a, b = part[s], part[s + 1]
        types = [rank_types[r] for r in range(sum(groups[:s]), sum(groups[:s + 1]))]
        if len(set(types)) == 1:
            key = f'tp{tp}_bs{plan["gbs"] // dp // plan["batches"]}'
            if key not in profile[f'DeviceType.{types[0]}']:
                raise KeyError(f"key({key}) not found in profile_data")
            lens.append(orc.fsum(profile[f'DeviceType.{types[0]}'][key]['time']['layer-computes'][a:b]))
        else:
            hetero_bs = orc.partition_data(profile, types, (dp, tp), plan['gbs'] // plan['batches'])
            costs = []
            for r, h in enumerate(hetero_bs):
                if h == 0:
                    continue
                dev = types[(len(types) // dp) * r]
                acc = 0.
                for piece in [2 ** i for i in range(int(math.log2(h)), -1, -1) if h & 2 ** i]:
                    if piece > max_profiled_bs:
                        raise KeyError(f"batch_size({piece}) not found in profile_data")
                    acc += orc.fsum(profile[f'DeviceType.{dev}'][f'tp{tp}_bs{piece}']['time']['layer-computes'][a:b])
                costs.append(acc)
            lens.append(max(costs))
        mbs = plan['gbs'] // dp // plan['batches']
        if s == plan['num_stage'] - 1:
            vals = []
            for dev in types:
                node = profile.get(f'DeviceType.{dev}')
                node = node.get(f'tp{tp}_bs{mbs}') if node else None
                node = node.get('time') if node else None
                v = node.get('fb_sync') if node else None
                if not v:
                    raise KeyError("key(fb_sync) not found in profile_data")
                vals.append(v)
            fb_sync = max(vals) * plan['batches']
            pps.append(0.0)
        else:
            act = model.activation_size(b, mbs, tp)
            pps.append(act / (pp_bw(s) * (1024 * 1024)))
            pp_cost += pps[-1]
        params = model.stage_parameters(tp, a, b)
        bw = dp_bw((dp, tp), s) * (1024 * 1024)
        dp_costs.append(2 * (dp - 1) / (dp * bw) * max([params]))
        upd.append(profile['model']['optimizer_time'] / tp * ((b - a) / model.num_layers))
    exec_cost = ((plan['batches'] - 1) * max(lens)) + orc.fsum(lens)
    bg = profile['model']['batch_generator'] * plan['batches']
    terms = [exec_cost, fb_sync, max(upd), max(dp_costs), pp_cost, bg]
    return terms, dict(stage_time=lens, dp_cost=dp_costs, update_cost=upd, pp_cost=pps)


def partition_layer_values(profile: Dict, cluster, norm_lc, num_layers: int, plan: dict, strategies, perf, m_capa,
                           corrected: Sequence[str] = ()):
    """orc.partition_layer that also returns the accepted attempt's performance and memory demand:
    (part, attempt, state, perf, demand)."""
    device_types = orc.rank_types_by_nodes(cluster, plan['node_sequence'])
    attempt = 1
    while attempt <= 3:
        part = orc.layer_compute_balance(len(perf), num_layers, list(perf), norm_lc, plurality='Q5' in corrected)
        if 'Q6' in corrected:
            demand = orc.stage_memory_demand_own_type(profile, part, strategies, plan['device_groups'],
                                                      orc.rank_types_by_devices(cluster, plan['node_sequence']),
                                                      plan['gbs'], plan['batches'])
        else:
            demand = orc.stage_memory_demand(profile, part, strategies, plan['device_groups'], device_types,
                                             plan['gbs'], plan['batches'])
        state = [mc - md for mc, md in zip(m_capa, demand)]
        if not (min(state) < 0):
            return part, attempt, state, list(perf), demand
        perf = orc.adjust_compute_performance(perf, m_capa, demand)
        if not perf:
            return None, -1, None, None, None
        attempt += 1
    return None, -1, None, None, None


def het_breakdowns(profile: Dict, cluster, model, node_sequences, gbs: int, num_layers: int, variance,
                   max_permute_len: int, max_tp: int, max_bs: int, plan_filter=None,
                   corrected: Sequence[str] = ()) -> List[Tuple]:
    """orc.het_search recording every candidate's breakdown: a list of (ordinal, step, num_repartition, cost, terms,
    stages), where ``stages`` holds performance / memory_capacity / memory_demand / memory_state over every stage and
    the cost fields of het_cost_terms over the costed stages."""
    norm_lc = orc.norm_layer_duration(profile)
    out = []
    for ordinal, plan in enumerate(orc.inter_stage_plans(node_sequences, cluster.total_devices, gbs, num_layers,
                                                         variance, max_permute_len, corrected)):
        if plan_filter is not None and not plan_filter(ordinal):
            continue
        groups = plan['device_groups']
        rank_types = orc.rank_types_by_devices(cluster, plan['node_sequence'])
        strategies: List[Tuple[int, int]] = []
        mem_state = []
        nrep = step = 0
        while nrep != 1:                                 # the chain of orc.het_evaluate_plan
            found = False
            while True:
                if not strategies:
                    strategies = [(g, 1) for g in groups]
                else:
                    cur = list(strategies)
                    state = mem_state if mem_state else [1 / dp for dp, _ in strategies]
                    nxt = None
                    for s in sorted(range(len(state)), key=lambda i: state[i]):
                        dp, tp = cur[s]
                        if dp != 1:
                            cur[s] = (dp // 2, tp * 2)
                            nxt = cur
                            break
                    strategies = nxt
                if not strategies:
                    break
                if any(gbs // dp // plan['batches'] == 0 or gbs // dp // plan['batches'] > max_bs or tp > max_tp
                       for dp, tp in strategies):
                    continue
                m_capa = orc.stage_memory_capacity(cluster, rank_types, groups)
                perf = orc.stage_compute_performance(profile, rank_types, groups, strategies, gbs, plan['batches'])
                part, n_rep, state, used, demand = partition_layer_values(profile, cluster, norm_lc, num_layers, plan,
                                                                          strategies, perf, m_capa, corrected)
                mem_state = state
                if part:
                    nrep = n_rep
                    found = True
                    break
            if not found:
                break
            try:
                terms, costed = het_cost_terms(profile, cluster, model, plan, strategies, part, rank_types, max_bs)
                cost = orc.het_cost(profile, cluster, model, plan, strategies, part, rank_types, max_bs)
                stages = dict(costed, performance=used, memory_capacity=list(m_capa), memory_demand=list(demand),
                              memory_state=list(state))
                out.append((ordinal, step, nrep, cost, terms, stages))
            except KeyError:
                pass
            step += 1
    return out


def homo_breakdown(profile: Dict, cluster, model, plan, dev: str):
    """orc.homo_cost -> (cost, per-stage memory sums, oom, the reference's formatted strings)."""
    cost, mem, oom = orc.homo_cost(profile, cluster, model, plan, dev)
    return cost, mem, oom, [f'{round(m / 1024 / 1024 / 1024, 2)}GB' for m in mem]
