"""CPU oracle for the Metis plan-search hot path.  TEST INFRASTRUCTURE ONLY.

This module is a plain-Python restatement of the reference algorithm
(SamsungLabs/Metis @ ed41176).  It exists so the CUDA path can be checked
against something that runs anywhere (the GPU machines have no checkout of the reference).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs may import it.  The product package (metis_b200/)
must never import it and has no CPU fallback.

Parity pin: the reference ships no tests or golden vectors for this path
(SURVEY.md section 4), so the oracle is pinned against outputs of the
*unmodified reference*
(tests/golden/make_golden.py imports a checkout of it and dumps
tests/golden/*.json.gz; tests/test_oracle_vs_golden.py replays them).

All float arithmetic is IEEE binary64 in the order the reference evaluates it.
``fsum`` below restates CPython >= 3.12's builtin ``sum`` (Neumaier
compensation, Python/bltinmodule.c) because the reference calls ``sum`` on
float lists everywhere and the parity target is Python 3.12.

Every function cites the reference file:line it follows (paths relative to
the reference root).
"""
from __future__ import annotations

import itertools
import json
import math
import os
import re
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

HALLUCINATION = 7  # model/load_balancer.py:183 (default argument)
MEM_COEF = 5.0     # model/load_balancer.py:31 (default argument)


# --------------------------------------------------------------------------
# numeric primitives
# --------------------------------------------------------------------------
def fsum(values) -> float:
    """builtin ``sum`` of CPython 3.12 for a list of ints/floats.

    Leading ints are added as ints; the first float is added with an ordinary
    ``+``; from then on floats are accumulated with Neumaier compensation and
    the compensation is added once at the end if it is non-zero and finite.
    Ints met after the first float are added uncompensated.
    """
    it = iter(values)
    acc = 0
    for x in it:
        if isinstance(x, int) and not isinstance(x, bool):
            acc += x
            continue
        acc = acc + x          # int + float -> float
        break
    else:
        return acc             # all ints (or empty): exact int result
    f = float(acc)
    c = 0.0
    for x in it:
        if isinstance(x, float):
            t = f + x
            if abs(f) >= abs(x):
                c += (f - t) + x
            else:
                c += (x - t) + f
            f = t
        else:
            f += float(x)
    if c and math.isfinite(c):
        f += c
    return f


# --------------------------------------------------------------------------
# inputs (data_loader.py, gpu_cluster.py, utils.py)
# --------------------------------------------------------------------------
class OracleCluster:
    """gpu_cluster.py:8-58 + utils.py:8-31 restated on plain lists."""

    def __init__(self, hostfile_path: str, clusterfile_path: str, corrected: Sequence[str] = ()):
        """``corrected`` mirrors the product's opt-in mode (SURVEY.md 8(f)-4): with 'Q2' inter_bw() returns the
        clusterfile's inter_bandwidth.  Default = the reference."""
        self.corrected = tuple(corrected)
        self.node_ip: List[str] = []
        self.node_ndev: List[int] = []
        with open(hostfile_path, 'rt') as fh:            # utils.py:8-24
            for line in fh:
                if not line:
                    break
                tok = line.split(' ')
                self.node_ip.append(tok[0])
                self.node_ndev.append(int(tok[1][6:7]))  # utils.py:15 (Q10)
        with open(clusterfile_path, 'r') as fh:          # utils.py:27-31
            self.info = json.loads(fh.read())
        # gpu_cluster.py:16-17; DeviceType.from_string upper-cases (utils.py:52-57)
        self.node_type = [self.info[ip]['instance_type'].upper() for ip in self.node_ip]

    @property
    def num_nodes(self) -> int:                           # gpu_cluster.py:19-20
        return len(self.node_ip)

    @property
    def total_devices(self) -> int:                       # gpu_cluster.py:28-30
        return sum(self.node_ndev)

    @property
    def devices_per_node(self) -> int:                    # gpu_cluster.py:25-26 (node 0 only)
        return self.node_ndev[0]

    def devices_of_type(self, name: str) -> int:          # gpu_cluster.py:22-23
        return sum(n for n, t in zip(self.node_ndev, self.node_type) if t == name)

    def memory_of_type(self, name: str):                  # gpu_cluster.py:47-50
        for ip in self.info:
            if self.info[ip]['instance_type'] == name:
                return self.info[ip]['memory'] * 1024
        return None

    def memory_of_node(self, node_id: int):               # gpu_cluster.py:38-45
        return self.info[self.node_ip[node_id]]['memory'] * 1024

    def intra_bw(self, node_id: int):                     # gpu_cluster.py:52-54
        return self.info[self.node_ip[node_id]]['intra_bandwidth']

    def inter_bw_strict(self, node_id: int):              # gpu_cluster.py:56-58 (Q2: returns intra)
        return self.info[self.node_ip[node_id]]['intra_bandwidth']

    def inter_bw(self, node_id: int):                     # het path: the opt-in correction applies here only
        if 'Q2' in self.corrected:
            return self.info[self.node_ip[node_id]]['inter_bandwidth']
        return self.inter_bw_strict(node_id)

    def device_types_in_host_order(self) -> List[str]:    # gpu_cluster.py:32-33
        return list(self.node_type)


def load_profile_dir(profile_dir: str, file_order: Optional[Sequence[str]] = None
                     ) -> Tuple[Dict, List[str]]:
    """data_loader.py:10-61.  ``file_order`` pins the os.listdir order (Q3)."""
    names = list(file_order) if file_order is not None else \
        [f for f in os.listdir(profile_dir) if f.endswith('.json')]
    data: Dict = {}
    types: List[str] = []
    for name in names:
        dev = re.search(r"DeviceType\.(\w+?)_", name).group(1)
        key = f'DeviceType.{dev}'
        if key not in data:
            data[key] = {}
            types.append(dev)
        tp = re.search(r"tp(\d+)", name).group(1)
        bs = re.search(r"bs(\d+)", name).group(1)
        with open(os.path.join(profile_dir, name), 'r') as fh:
            raw = json.loads(fh.read())
        if 'model' not in data:                            # data_loader.py:16-24,54-56
            data['model'] = {
                'optimizer_time': raw['execution_time']['optimizer_time_ms'] * 2,
                'num_layers': len(raw['execution_time']['layer_compute_total_ms']),
                'batch_generator': raw['execution_time']['batch_generator_time_ms'],
                'parameters': raw['model']['parameters']['parameters_per_layer_bytes'],
            }
        lc = list(raw['execution_time']['layer_compute_total_ms'])   # data_loader.py:26-37
        data[key][f'tp{tp}_bs{bs}'] = {
            'time': {'layer-computes': lc,
                     'fb_sync': raw['execution_time']['forward_backward_time_ms'] - fsum(lc)},
            'memory': raw['execution_memory']['layer_memory_total_mb'],
        }
    return data, types


class OracleModel:
    """utils.py:72-79 + model/activation_parameter.py:5-51."""

    def __init__(self, num_layers: int, hidden_size: int, sequence_length: int,
                 vocab_size: int, params: Sequence):
        self.num_layers = num_layers
        self.hidden = hidden_size
        self.seq = sequence_length
        self.vocab = vocab_size
        self.input_params = float(params[0])          # activation_parameter.py:22
        self.output_params = float(params[-1])        # :23
        self.transformer_params = float(params[1])    # :24

    def activation_size(self, layer_id: int, bs: int, tp: int):   # :28-32
        if layer_id == self.num_layers - 1:
            return bs * self.seq * self.vocab / tp
        return bs * self.seq * self.hidden

    def parameter_list(self, tp: int) -> List[float]:              # :34-38
        out = [self.input_params / tp]
        out += [self.transformer_params / tp for _ in range(self.num_layers - 2)]
        out.append(self.output_params / tp)
        return out

    def stage_parameters(self, tp: int, a: int, b: int):           # :40-51
        n = b - a
        p = 0
        if a == 0:
            p += self.input_params / tp
            n -= 1
        if b == self.num_layers:
            p += self.output_params / tp
            n -= 1
        p += self.transformer_params / tp * n
        return p


# --------------------------------------------------------------------------
# search space: device groups (search_space/device_group.py, search_space/utils.py)
# --------------------------------------------------------------------------
def multiset_permutations(items: List) -> Iterator[List]:
    """search_space/utils.py:56-88 (Williams 2009 prefix-shift order).

    Restated on index arrays instead of a linked list: ``nxt[i]`` is the
    successor of node i, ``val[i]`` its value.
    """
    vals = sorted(items)                                  # utils.py:57
    n = len(vals)
    nxt = [-1] * n
    # utils.py:58-60: list built by prepending => head = max, chain is non-increasing
    head = 0
    for k in range(1, n):
        nxt[k] = head
        head = k

    def walk(h):
        out = []
        while h != -1:
            out.append(vals[h])
            h = nxt[h]
        return out

    def nth(h, k):                                        # utils.py:47-53
        while k > 0 and nxt[h] != -1:
            h = nxt[h]
            k -= 1
        return h

    i = nth(head, n - 2)
    j = nth(head, n - 1)
    yield walk(head)
    while nxt[j] != -1 or vals[j] < vals[head]:          # utils.py:76-88
        if nxt[j] != -1 and vals[i] >= vals[nxt[j]]:
            s = j
        else:
            s = i
        t = nxt[s]
        nxt[s] = nxt[t]
        nxt[t] = head
        if vals[t] < vals[head]:
            i = t
        j = nxt[i]
        head = t
        yield walk(head)


def merge_and_permute(comp: Sequence[int], max_permute_len: int) -> Iterator[List[Tuple[int, ...]]]:
    """search_space/device_group.py:7-55 (``permute``)."""
    groups: List[Tuple[int, ...]] = [(e,) for e in comp]
    num_reduce = len(groups) - max_permute_len
    while num_reduce > 0:
        first = groups[0]
        min_size = sum(first)
        # find_num_min (:8-12): index of first differing group + 1, else len
        num_min = len(groups)
        for idx, g in enumerate(groups):
            if g != first:
                num_min = idx + 1
                break
        if num_min // 2 > num_reduce:                      # :26-27
            num_reduce = num_min // 2
        merged: List[Tuple[int, ...]] = []
        for i in range(0, len(groups), 2):                 # :31-45
            if num_reduce <= i // 2:
                merged.extend(groups[i:])
                break
            if i + 1 >= len(groups):
                merged.append(groups[i])
            elif sum(groups[i]) == min_size and sum(groups[i]) == sum(groups[i + 1]):
                merged.append(tuple(groups[i] + groups[i + 1]))
            else:
                merged.append(groups[i])
                merged.append(groups[i + 1])
        groups = merged
        if num_reduce == len(groups) - max_permute_len:    # :48-50
            break
        num_reduce = len(groups) - max_permute_len
    return multiset_permutations(groups)


def compositions(num_stages: int, num_gpus: int, shapes: Sequence[int]) -> Iterator[List[int]]:
    """search_space/device_group.py:58-81 (``gen_dgroups_recursive``)."""
    if not shapes:
        return

    def rec(cur_sum, stage_idx, sol, prev_idx):
        if shapes[-1] * (num_stages - stage_idx) < num_gpus - cur_sum:
            return
        if shapes[0] * (num_stages - stage_idx) > num_gpus - cur_sum:
            return
        if stage_idx >= num_stages:
            if len(sol) == num_stages and cur_sum == num_gpus:
                yield sol
            return
        for i in range(max(0, prev_idx), len(shapes)):
            g = shapes[i]
            if g + cur_sum > num_gpus:
                break
            yield from rec(cur_sum + g, stage_idx + 1, sol + [g], i)

    for idx, g in enumerate(shapes):
        yield from rec(g, 1, [g], idx)


def group_shapes(num_gpus: int) -> List[int]:
    """search_space/device_group.py:84-90."""
    out, i = [], 0
    while 2 ** i <= num_gpus:
        out.append(2 ** i)
        i += 1
    return out


def device_group_rows(num_stages: int, num_gpus: int, variance, max_permute_len: int) -> List[List[int]]:
    """search_space/device_group.py:93-107."""
    floor_share = max(num_gpus // num_stages, num_stages // num_gpus)
    floor_share *= variance
    shapes = [s for s in group_shapes(num_gpus) if s >= floor_share]
    rows: List[List[int]] = []
    for comp in compositions(num_stages, num_gpus, shapes):
        for perm in merge_and_permute(comp, max_permute_len):
            rows.append(list(itertools.chain(*perm)))
    return rows


# --------------------------------------------------------------------------
# search space: plan generators (search_space/plan.py)
# --------------------------------------------------------------------------
def uniform_plans(num_devices: int, max_tp: int, max_gbs: int) -> Iterator[Tuple[int, int, int, int, int]]:
    """search_space/plan.py:40-97; yields (dp, pp, tp, mbs, gbs) snapshots."""
    dp, pp, tp, mbs, gbs = num_devices, 1, 1, 0, num_devices
    while True:
        mbs += 1                                            # _find_next_mbs :47-51
        while gbs % mbs > 0 and mbs <= gbs:
            mbs += 1
        if mbs * dp > gbs:                                  # :84-86
            mbs = 1
            gbs += 1                                        # _find_next_gbs :53-57
            while max_gbs % gbs > 0 and gbs <= max_gbs:
                gbs += 1
        if gbs > max_gbs:                                   # :88-95
            mbs = 1
            while True:                                     # _find_next_dp_pp_tp :59-76
                if tp == max_tp and pp == num_devices:
                    return
                elif tp == max_tp:
                    pp += 1
                    dp = num_devices // pp
                    tp = num_devices // dp // pp
                else:
                    tp += 1
                    dp = num_devices // tp // pp
                if dp * pp * tp == num_devices:
                    break
            gbs = dp
        yield (dp, pp, tp, mbs, gbs)


def inter_stage_plans(node_sequences: Sequence[Tuple[str, ...]], num_devices: int, gbs: int,
                      num_layers: int, variance, max_permute_len: int, corrected: Sequence[str] = ()) -> Iterator[dict]:
    """search_space/plan.py:100-175 including quirk Q1 (:144-148).

    ``node_sequences`` is ``list(itertools.permutations(set_of_types))`` as the
    caller saw it (Q4: set order is an input).
    """
    cap = min(num_devices, num_layers)
    rows = device_group_rows(1, num_devices, variance, max_permute_len)
    ns_idx, dg_idx, num_stage, batches = 0, 0, 1, gbs + 1
    _ = rows[0]                                             # plan.py:117-118 (IndexError if empty)

    def next_stage_rows(start):                             # plan.py:130-142
        s = start
        while True:
            r = device_group_rows(s, num_devices, variance, max_permute_len)
            if r or s > cap:
                return s, r
            s += 1

    while True:
        batches -= 1                                        # :120-124
        while batches >= 1 and gbs % batches > 0:
            batches -= 1
        if batches == 0:                                    # :156-158
            dg_idx += 1
            batches = gbs
        if dg_idx >= len(rows):                             # :160-163
            num_stage, rows = next_stage_rows(num_stage + 1)
            batches = gbs
            dg_idx = 0
        if num_stage > cap:                                 # :165-168 with :144-148
            ns_idx += 1
            num_stage = 1
            if 'Q1' in corrected:                           # opt-in: every node sequence starts at one stage
                rows = device_group_rows(1, num_devices, variance, max_permute_len)
            else:
                _, rows = next_stage_rows(2)                # returned stage count discarded (Q1)
            batches = gbs
            dg_idx = 0
        if ns_idx >= len(node_sequences):                   # :170-171
            return
        yield {'ns_idx': ns_idx, 'node_sequence': tuple(node_sequences[ns_idx]), 'dg_idx': dg_idx,
               'device_groups': rows[dg_idx], 'num_stage': num_stage, 'batches': batches, 'gbs': gbs}


# --------------------------------------------------------------------------
# evaluation model
# --------------------------------------------------------------------------
def _exec_full(profile: Dict, dev: str, key: str):
    """model/device_group.py:37-38 / load_balancer.py:152-153 (KeyError propagates)."""
    return fsum(profile[f'DeviceType.{dev}'][key]['time']['layer-computes'])


def _pow2_slices(h: int) -> List[int]:
    """model/device_group.py:46, load_balancer.py:49: binary decomposition high->low."""
    top = int(math.log2(h)) if h != 0 else 0
    return [2 ** i for i in range(top, -1, -1) if h & 2 ** i]


def partition_data(profile: Dict, device_types: Sequence[str], strategy: Tuple[int, int], bs: int) -> List[int]:
    """model/load_balancer.py:155-179."""
    dp, tp = strategy
    gsz = len(device_types) // dp
    perf = []
    for i in range(dp):
        grp = device_types[i * gsz:(i + 1) * gsz]
        perf.append(1. / _exec_full(profile, grp[0], f'tp{tp}_bs1'))
    total = fsum(perf)
    share = [p / total for p in perf]
    out = [int(bs * s) for s in share]
    remainder = bs - sum(out)
    frac = [(bs * s) - int(bs * s) for s in share]
    order = sorted(range(len(frac)), key=lambda i: frac[i], reverse=True)
    for i in range(remainder):
        out[order[i]] += 1
    return out


def rank_types_by_devices(cluster: OracleCluster, node_sequence: Sequence[str]) -> List[str]:
    """model/device_group.py:22-32 (StagePerformance._get_device_placement)."""
    out: List[str] = []
    for name in node_sequence:
        out += [name] * cluster.devices_of_type(name)
    return [out[r] for r in range(cluster.total_devices)]


def rank_types_by_nodes(cluster: OracleCluster, node_sequence: Sequence[str]) -> List[str]:
    """model/load_balancer.py:109-119 (LayerLoadBalancer._device_types_by_node_sequence)."""
    count = {}
    for t in cluster.node_type:
        count[t] = count.get(t, 0) + 1
    out: List[str] = []
    for name in node_sequence:
        out.extend([name] * count.get(name, 0) * cluster.node_ndev[0])
    return out


def stage_memory_capacity(cluster: OracleCluster, rank_types: Sequence[str], groups: Sequence[int]) -> List:
    """model/device_group.py:87-101."""
    out = []
    for s in range(len(groups)):
        a, b = sum(groups[:s]), sum(groups[:s + 1])
        counts: Dict[str, int] = {}
        for r in range(a, b):
            counts[rank_types[r]] = counts.get(rank_types[r], 0) + 1
        out.append(fsum([cluster.memory_of_type(t) * n for t, n in counts.items()]))
    return out


def stage_compute_performance(profile: Dict, rank_types: Sequence[str], groups: Sequence[int],
                              strategies: Sequence[Tuple[int, int]], gbs: int, batches: int) -> List[float]:
    """model/device_group.py:40-85."""
    perf = []
    for s, (dp, tp) in zip(range(len(groups)), strategies):
        bs = gbs // batches // dp
        a, b = sum(groups[:s]), sum(groups[:s + 1])
        types = [rank_types[r] for r in range(a, b)]
        if len(set(types)) > 1:
            hetero_bs = partition_data(profile, types, (dp, tp), gbs // batches)
            costs = []
            for r, h in enumerate(hetero_bs):                # :40-52
                dev = types[(len(types) // dp) * r]
                acc = 0.
                for piece in _pow2_slices(h):
                    acc += _exec_full(profile, dev, f'tp{tp}_bs{piece}')
                costs.append(acc)
            cur = 0
            if max(costs) != 0:
                cur = 1. / max(costs)
            perf.append(cur)
        else:
            perf.append(1. / _exec_full(profile, types[0], f'tp{tp}_bs{bs}'))
    total = fsum(perf)
    return [p / total for p in perf]


def layer_compute_balance(num_stage: int, num_layer: int, capa_in: Sequence[float],
                          lc: Sequence[float], plurality: bool = False) -> List[int]:
    """model/load_balancer.py:182-372 (LayerComputeBalancer.run) -> layer partition.
    ``plurality`` (opt-in correction Q5, not the reference): a layer goes to the stage that holds most of its
    sub-layers (lowest stage on ties) instead of only to a stage holding more than half."""
    H = HALLUCINATION
    N = num_layer * H
    bak = list(capa_in)
    capa = list(capa_in)
    d = []
    for x in lc:                                            # :189-193
        q = x / H
        d.extend([q] * H)
    alloc: Dict[int, List[int]] = {s: [] for s in range(num_stage)}
    un: List[int] = []

    # forward :216-231
    k = 0
    for s in range(num_stage - 1):
        for j in range(k, N - 1 - H):
            if capa[s] > d[j]:
                capa[s] -= d[j]
                alloc[s].append(j)
                k = j + 1
            else:
                un.append(j)
                k = j + 1
                break
    for j in range(k, N):
        un.append(j)
    un = list(set(sorted(un)))

    # backward :233-249
    last = num_stage - 1
    for j in sorted(un.copy(), reverse=True):
        if len(alloc[last]) < H:
            capa[last] -= d[j]
            alloc[last].append(j)
            un.remove(j)
            continue
        if (j + 1) != min(alloc[last]):
            continue
        if capa[last] > d[j]:
            capa[last] -= d[j]
            alloc[last].append(j)
            un.remove(j)

    # leftovers :251-287
    for j in sorted(un.copy()):
        lo, hi = min(alloc.keys()), max(alloc.keys())
        lo_val, hi_val = float('-inf'), float('inf')
        for s in alloc.keys():
            grp = alloc[s]
            if len(grp) == 0:
                continue
            g_min, g_max = min(grp), max(grp)
            if j > g_max and g_max > lo_val:
                lo, lo_val = s, g_max
            if j < g_min and g_min < hi_val:
                hi, hi_val = s, g_min
        pick, best = None, float('-inf')
        for s in range(lo, hi + 1):
            if capa[s] > best:
                best, pick = capa[s], s
        capa[pick] -= d[j]
        alloc[pick].append(j)
        un.remove(j)
    for s in alloc:
        alloc[s] = sorted(alloc[s])

    # majority vote :290-308
    real: Dict[int, List[int]] = {}
    if plurality:
        count = [[0] * num_stage for _ in range(num_layer)]
        for s in range(num_stage):
            for j in alloc[s]:
                count[int(j / H)][s] += 1
        real = {s: [] for s in range(num_stage)}
        for r in range(num_layer):
            real[max(range(num_stage), key=lambda s: (count[r][s], -s))].append(r)
    else:
        for s in range(num_stage):
            grp = [int(j / H) for j in alloc[s]]
            keep = [r for r in grp if grp.count(r) > (H / 2)]
            real[s] = sorted(list(set(keep)))
    alloc = real
    capa = []
    for s in range(num_stage):
        if len(alloc[s]):
            first, lastl = alloc[s][0], alloc[s][-1]
            capa.append(bak[s] - fsum(lc[first:lastl + 1]))
        else:
            capa.append(bak[s])

    # adjust :310-356
    def near(idx, cc):                                      # get_near_max :311-321
        pick, val = None, float('inf')
        if (idx - 1) >= 0 and cc[idx - 1] < val:
            pick, val = idx - 1, cc[idx - 1]
        if (idx + 1) < len(cc) and cc[idx + 1] < val:
            pick, val = idx + 1, cc[idx + 1]
        if pick is None or len(alloc[pick]) == 1:           # committed allocation (:319)
            pick = None
        return pick

    oc = capa.copy()
    oa = {s: list(v) for s, v in alloc.items()}
    n = 0
    while True:
        n += 1
        ranked = sorted([(i, oc[i]) for i in range(len(oc))], key=lambda kv: kv[1], reverse=True)
        top = ranked[0][0]
        nb = near(top, oc)
        if (nb is not None) and len(oa[nb]):
            if top > nb:
                layer = oa[nb].pop(-1)
            else:
                layer = oa[nb].pop(0)
            oa[top].append(layer)
            oa[top] = sorted(oa[top])
            oc[top] -= lc[layer]
            oc[nb] += lc[layer]
        if max(oc) > max(capa) or n > 3:
            break
        alloc = {s: list(v) for s, v in oa.items()}
        capa = oc.copy()

    part = [0]                                              # :358-364
    for s in alloc.keys():
        part.append(part[s] + len(alloc[s]))
    return part


def stage_memory_demand_own_type(profile: Dict, part: Sequence[int], strategies: Sequence[Tuple[int, int]],
                                 groups: Sequence[int], rank_types: Sequence[str], gbs: int, batches: int) -> List[float]:
    """Opt-in correction Q6 (NOT the reference): the stage's own devices (true rank -> type map) decide the memory
    profile; a mixed-type stage is split like its compute (partition_data over its own devices) and needs the
    memory of its largest replica."""
    out = []
    for s, (dp, tp) in enumerate(strategies):
        a, b = sum(groups[:s]), sum(groups[:s + 1])
        cur = [rank_types[r] for r in range(a, b)]
        la, lb = part[s], part[s + 1]
        demand = 0.001
        if len(set(cur)) == 1:
            bs = gbs // batches // dp
            demand += fsum(profile[f'DeviceType.{cur[0]}'][f'tp{tp}_bs{bs}']['memory'][la:lb]) * MEM_COEF
        else:
            hetero_bs = partition_data(profile, cur, (dp, tp), gbs // batches)
            worst = 0.0
            for r, h in enumerate(hetero_bs):
                dev = cur[(len(cur) // dp) * r]
                need = 0.0
                for piece in _pow2_slices(h) if h else []:
                    need += fsum(profile[f'DeviceType.{dev}'][f'tp{tp}_bs{piece}']['memory'][la:lb]) * MEM_COEF
                if need > worst:
                    worst = need
            demand += worst
        out.append(demand)
    return out


def stage_memory_demand(profile: Dict, part: Sequence[int], strategies: Sequence[Tuple[int, int]],
                        groups: Sequence[int], device_types: Sequence[str], gbs: int, batches: int) -> List[float]:
    """model/load_balancer.py:29-55 (Q6)."""
    out = []
    for s, (dp, tp) in enumerate(strategies):
        a, b = sum(groups[:s]), sum(groups[:s + 1])
        cur = [device_types[r] for r in range(a, b)]
        la, lb = part[s], part[s + 1]
        demand = 0.001
        if len(set(cur)) == 1:
            bs = gbs // batches // dp
            mem = profile[f'DeviceType.{device_types[0]}'][f'tp{tp}_bs{bs}']['memory']
            demand += fsum(mem[la:lb]) * MEM_COEF
        else:
            hetero_bs = partition_data(profile, device_types, (dp, tp), gbs // batches)
            for h in hetero_bs:
                for piece in _pow2_slices(h):
                    mem = profile[f'DeviceType.{device_types[0]}'][f'tp{tp}_bs{piece}']['memory']
                    demand += fsum(mem[la:lb]) * MEM_COEF
        out.append(demand)
    return out


def adjust_compute_performance(c_capa: Sequence[float], m_capa: Sequence, m_demand: Sequence[float]
                               ) -> Optional[List[float]]:
    """model/load_balancer.py:71-107."""
    adj, avail = [], []
    need = 0.
    for c, mc, md in zip(c_capa, m_capa, m_demand):
        if mc > md:
            adj.append(c)
            avail.append((c * mc / md) - c)
        else:
            avail.append(0)
            a = c * (mc / md) * 0.9
            adj.append(a)
            need += (c - a)
    if fsum(avail) < need:
        return None
    extra = [0. for _ in range(len(c_capa))]
    guard = 0
    while need > 0.01:
        tot = fsum([c if a > 0.001 else 0 for a, c in zip(avail, c_capa)])
        ratio = [c / tot if a > 0.001 else 0 for a, c in zip(avail, c_capa)]
        for (s, r), a in zip(enumerate(ratio), avail):
            give = a if need * r > a else need * r
            extra[s] += give
            avail[s] -= give
            need -= give
        guard += 1
        if guard > 100000:
            raise RuntimeError('reference would not terminate (load_balancer.py:96-104)')
    return [e + a for e, a in zip(extra, adj)]


def partition_layer(profile: Dict, cluster: OracleCluster, norm_lc: Sequence[float], num_layers: int,
                    plan: dict, strategies, perf, m_capa, counters: Optional[dict] = None,
                    corrected: Sequence[str] = ()):
    """model/load_balancer.py:121-144.  ``corrected``: opt-in 'Q5' / 'Q6' (see layer_compute_balance,
    stage_memory_demand_own_type); default = the reference."""
    device_types = rank_types_by_nodes(cluster, plan['node_sequence'])
    attempt = 1
    while attempt <= 3:
        if counters is not None:
            counters['runs'] = counters.get('runs', 0) + 1
        part = layer_compute_balance(len(perf), num_layers, list(perf), norm_lc, plurality='Q5' in corrected)
        if 'Q6' in corrected:
            demand = stage_memory_demand_own_type(profile, part, strategies, plan['device_groups'],
                                                  rank_types_by_devices(cluster, plan['node_sequence']),
                                                  plan['gbs'], plan['batches'])
        else:
            demand = stage_memory_demand(profile, part, strategies, plan['device_groups'], device_types,
                                         plan['gbs'], plan['batches'])
        state = [mc - md for mc, md in zip(m_capa, demand)]   # :57-63
        if not (min(state) < 0):
            return part, attempt, state
        perf = adjust_compute_performance(perf, m_capa, demand)
        if not perf:
            return None, -1, None
        attempt += 1
    return None, -1, None


def norm_layer_duration(profile: Dict) -> List[float]:
    """model/load_balancer.py:22-27 (first key of profile_data, Q3)."""
    first = next(iter(profile))
    lc = profile[first]['tp1_bs1']['time']['layer-computes']
    total = fsum(lc)
    return [x / total for x in lc]


def het_bandwidths(cluster: OracleCluster, plan: dict):
    """model/cluster_bandwidth.py:135-195 + :34-68; returns (pp_bw(stage), dp_bw(strategy, stage))."""
    per_node = cluster.devices_per_node
    rank_node = {}
    c = 0
    for node in range(cluster.num_nodes):                    # :34-47 (node 0's count for all, Q10)
        for _ in range(per_node):
            rank_node[c] = node
            c += 1
    count = {}
    for t in cluster.node_type:
        count[t] = count.get(t, 0) + 1
    sorted_types: List[str] = []                             # :158-167
    for name in plan['node_sequence']:
        sorted_types.extend([name] * count.get(name, 0))
    groups = plan['device_groups']

    def intra(dev):                                          # :49-54
        for node in range(cluster.num_nodes):
            if cluster.node_type[node] == dev:
                return cluster.intra_bw(node)
        return None

    def inter(devs):                                         # :56-68
        slow = float('inf')
        for node in range(cluster.num_nodes):
            for dev in devs:
                if cluster.node_type[node] == dev and cluster.inter_bw(node) < slow:
                    slow = cluster.inter_bw(node)
        return slow

    def bw_of_nodes(nodes):
        devs = [sorted_types[n] for n in list(set(nodes))]
        return intra(devs[0]) if len(devs) == 1 else inter(devs)

    def pp_bw(stage):                                        # :143-146,169-177
        ranks = range(sum(groups[:stage]), sum(groups[:stage + 2]))
        return bw_of_nodes([rank_node[r] for r in ranks])

    def dp_bw(strategy, stage):                              # :148-156,179-195
        ranks = list(range(sum(groups[:stage]), sum(groups[:stage + 1])))
        dp, tp = strategy
        grp = [[] for _ in range(dp)]
        for _t in range(tp):
            for dd in range(dp):
                grp[dd].append(ranks.pop(0))
        slow = float('inf')
        for g in grp:
            bw = bw_of_nodes([rank_node[r] for r in g])
            if bw < slow:
                slow = bw
        return slow

    return pp_bw, dp_bw


def het_cost(profile: Dict, cluster: OracleCluster, model: OracleModel, plan: dict, strategies, part,
             rank_types: Sequence[str], max_profiled_bs: int) -> float:
    """model/cost_estimator.py:199-244 (raises KeyError like the reference)."""
    pp_bw, dp_bw = het_bandwidths(cluster, plan)
    groups = plan['device_groups']
    lens, dp_costs, upd = [], [], []
    pp_cost, fb_sync = 0., 0.
    for s, (dp, tp) in zip(range(plan['num_stage']), strategies):
        a, b = part[s], part[s + 1]
        types = [rank_types[r] for r in range(sum(groups[:s]), sum(groups[:s + 1]))]
        # _get_execution_cost :175-197
        if len(set(types)) == 1:
            key = f'tp{tp}_bs{plan["gbs"] // dp // plan["batches"]}'
            if key not in profile[f'DeviceType.{types[0]}']:
                raise KeyError(f"key({key}) not found in profile_data")
            lens.append(fsum(profile[f'DeviceType.{types[0]}'][key]['time']['layer-computes'][a:b]))
        else:
            hetero_bs = partition_data(profile, types, (dp, tp), plan['gbs'] // plan['batches'])
            costs = []
            for r, h in enumerate(hetero_bs):                # :152-173
                if h == 0:
                    continue
                dev = types[(len(types) // dp) * r]
                acc = 0.
                for piece in [2 ** i for i in range(int(math.log2(h)), -1, -1) if h & 2 ** i]:
                    if piece > max_profiled_bs:
                        raise KeyError(f"batch_size({piece}) not found in profile_data")
                    acc += fsum(profile[f'DeviceType.{dev}'][f'tp{tp}_bs{piece}']['time']['layer-computes'][a:b])
                costs.append(acc)
            lens.append(max(costs))
        mbs = plan['gbs'] // dp // plan['batches']
        if s == plan['num_stage'] - 1:
            vals = []                                        # _get_fb_sync_cost :57-72 (Q9)
            for dev in types:
                node = profile.get(f'DeviceType.{dev}')
                node = node.get(f'tp{tp}_bs{mbs}') if node else None
                node = node.get('time') if node else None
                v = node.get('fb_sync') if node else None
                if not v:
                    raise KeyError("key(fb_sync) not found in profile_data")
                vals.append(v)
            fb_sync = max(vals) * plan['batches']
        else:
            act = model.activation_size(b, mbs, tp)
            pp_cost += act / (pp_bw(s) * (1024 * 1024))      # :45-47
        params = model.stage_parameters(tp, a, b)
        bw = dp_bw((dp, tp), s) * (1024 * 1024)              # :37-43
        dp_costs.append(2 * (dp - 1) / (dp * bw) * max([params]))
        upd.append(profile['model']['optimizer_time'] / tp * ((b - a) / model.num_layers))   # :145-147
    exec_cost = ((plan['batches'] - 1) * max(lens)) + fsum(lens)
    bg = profile['model']['batch_generator'] * plan['batches']
    return exec_cost + fb_sync + max(upd) + max(dp_costs) + pp_cost + bg


def het_evaluate_plan(profile: Dict, cluster: OracleCluster, model: OracleModel, norm_lc, plan: dict,
                      ordinal: int, num_layers: int, max_tp: int, max_bs: int, counters: dict, out: list,
                      corrected: Sequence[str] = ()) -> None:
    """Loop body of cost_het_cluster.py:31-48 for one inter-stage plan, with the
    IntraStagePlanGenerator chain (search_space/plan.py:178-268) inlined."""
    gbs = plan['gbs']
    groups = plan['device_groups']
    rank_types = rank_types_by_devices(cluster, plan['node_sequence'])
    strategies: List[Tuple[int, int]] = []
    mem_state = []
    nrep = 0
    step = 0
    while True:
        if nrep == 1:                                    # plan.py:194-195
            break
        found = False
        while True:
            if not strategies:                           # :198-201
                strategies = [(g, 1) for g in groups]
            else:
                cur = list(strategies)
                state = mem_state if mem_state else [1 / dp for dp, _ in strategies]   # :252-255
                order = sorted(range(len(state)), key=lambda i: state[i])
                nxt = None
                for s in order:                          # :262-266
                    dp, tp = cur[s]
                    if dp != 1:
                        cur[s] = (dp // 2, tp * 2)
                        nxt = cur
                        break
                strategies = nxt
            if not strategies:                           # :203-204
                break
            valid = True                                 # :238-249
            for dp, tp in strategies:
                mbs = gbs // dp // plan['batches']
                if mbs == 0 or mbs > max_bs or tp > max_tp:
                    valid = False
                    break
            if not valid:
                continue
            m_capa = stage_memory_capacity(cluster, rank_types, groups)
            perf = stage_compute_performance(profile, rank_types, groups, strategies, gbs, plan['batches'])
            counters['B'] += 1
            part, n_rep, state = partition_layer(profile, cluster, norm_lc, num_layers, plan,
                                                 strategies, perf, m_capa, counters, corrected)
            mem_state = state
            if part:                                     # :219-226
                nrep = n_rep
                found = True
                break
        if not found:
            break
        try:
            cost = het_cost(profile, cluster, model, plan, strategies, part, rank_types, max_bs)
            counters['C'] += 1
            out.append((ordinal, step, plan['node_sequence'], list(groups), list(strategies),
                        plan['batches'], list(part), nrep, cost))
        except KeyError:
            counters['keyerr'] += 1
        step += 1


def het_search(profile: Dict, cluster: OracleCluster, model: OracleModel, node_sequences, gbs: int,
               num_layers: int, variance, max_permute_len: int, max_tp: int, max_bs: int,
               plan_filter=None, corrected: Sequence[str] = ()):
    """cost_het_cluster.py:21-50.

    Returns (candidates, counters); a candidate is
    (ordinal, step, node_sequence, device_groups, strategies, batches, partition, num_repartition, cost).
    ``plan_filter(ordinal)`` lets callers evaluate a shard of the inter-stage plans.
    """
    norm_lc = norm_layer_duration(profile)
    counters = {'A': 0, 'B': 0, 'C': 0, 'runs': 0, 'keyerr': 0}
    out: list = []
    for ordinal, plan in enumerate(inter_stage_plans(node_sequences, cluster.total_devices, gbs,
                                                     num_layers, variance, max_permute_len, corrected)):
        counters['A'] += 1
        if plan_filter is not None and not plan_filter(ordinal):
            continue
        het_evaluate_plan(profile, cluster, model, norm_lc, plan, ordinal, num_layers, max_tp, max_bs,
                          counters, out, corrected)
    return out, counters


# --------------------------------------------------------------------------
# homogeneous path
# --------------------------------------------------------------------------
def uniform_layer_counts(total_layers: int, num_stages: int) -> List[int]:
    """model/utils.py:5-31."""
    base = (total_layers - 2) // num_stages
    rem = (total_layers - 2) % num_stages
    out = [base] * num_stages
    for i in range(1, rem + 1):
        out[i] += 1
    out[0] += 1
    out[-1] += 1
    return out


def homo_cost(profile: Dict, cluster: OracleCluster, model: OracleModel, plan, dev: str):
    """model/cost_estimator.py:98-138 + cluster_bandwidth.py:71-132; returns (time, stage_mem, oom)."""
    dp, pp, tp, mbs, gbs = plan
    per_node = cluster.devices_per_node
    total = cluster.total_devices
    intra, inter = cluster.intra_bw(0), cluster.inter_bw_strict(0)
    params = model.parameter_list(tp)
    counts = uniform_layer_counts(model.num_layers, pp)
    num_mbs = gbs // mbs // dp
    key = f'tp{tp}_bs{mbs}'
    lens, stage_params, stage_mem = [], [], []
    pp_cost, fb_sync = 0., 0.

    def same_node(ranks):
        return len(set(r // per_node for r in ranks)) == 1

    for s in range(len(counts)):
        a, b = sum(counts[:s]), sum(counts[:s + 1])
        if key not in profile[f'DeviceType.{dev}']:
            raise KeyError(f"key({key}) not found in profile_data")
        lens.append(fsum(profile[f'DeviceType.{dev}'][key]['time']['layer-computes'][a:b]))
        stage_params.append(fsum(params[a:b]))
        stage_mem.append(fsum(profile[f'DeviceType.{dev}'][key]['memory'][a:b]))
        if s == len(counts) - 1:
            v = profile[f'DeviceType.{dev}'][key]['time'].get('fb_sync')
            if not v:
                raise KeyError("key(fb_sync) not found in profile_data")
            fb_sync = v * num_mbs
        else:
            act = model.activation_size(b, mbs, tp)
            assert tp * dp * pp == total
            bw = intra                                       # cluster_bandwidth.py:111-123
            for d in range(dp):
                for t in range(tp):
                    r0 = s * dp * tp + d * tp + t
                    r1 = (s + 1) * dp * tp + d * tp + t
                    if not same_node([r0, r1]):
                        bw = inter
            pp_cost += act / (bw * (1024 * 1024))
    oom = cluster.memory_of_node(0) < max(stage_mem)
    exec_cost = ((num_mbs - 1) * max(lens)) + fsum(lens)
    upd = profile['model']['optimizer_time'] / pp / tp
    bw = intra                                               # :125-132
    for p in range(pp):
        if not same_node(range(p * dp * tp, (p + 1) * dp * tp)):
            bw = inter
    dp_cost = 2 * (dp - 1) / (dp * (bw * (1024 * 1024))) * max(stage_params)
    bg = profile['model']['batch_generator'] * num_mbs
    return exec_cost + fb_sync + upd + dp_cost + pp_cost + bg, stage_mem, oom


def homo_search(profile: Dict, cluster: OracleCluster, model: OracleModel, dev: str, gbs: int, max_tp: int):
    """cost_homo_cluster.py:21-37; returns (list of (plan, cost), counters)."""
    out = []
    counters = {'yielded': 0, 'matched': 0, 'costed': 0, 'keyerr': 0}
    for plan in uniform_plans(cluster.total_devices, max_tp, gbs):
        counters['yielded'] += 1
        if plan[4] != gbs:
            continue
        counters['matched'] += 1
        try:
            cost, _, _ = homo_cost(profile, cluster, model, plan, dev)
            out.append((plan, cost))
            counters['costed'] += 1
        except KeyError:
            counters['keyerr'] += 1
    return out, counters
