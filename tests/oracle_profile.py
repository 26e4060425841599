"""Profile what-if (HetSearchResult.recost_profiles) at fixed arguments: the seeded scenario profiles the tests and
tests/golden/make_profile_golden.py build from a base profile, and the oracle's restatement of what each scenario gives
a searched candidate whose device groups, strategies and layer partition are held fixed - HeteroCostEstimator.get_cost
(model/cost_estimator.py:199-244) and the smallest capacity - LayerLoadBalancer._get_stage_memory_demand
(model/load_balancer.py:29-55) over all stages, with the exception either one raises.  Built from the oracle's own
pieces (oracle/metis_oracle.py)."""
import copy
import hashlib
import json
import math
import random
from typing import Dict, List, Sequence, Tuple

import numpy as np

from oracle import metis_oracle as orc

KINDS = ('base', 'compute', 'memory', 'keys', 'model', 'noise')
# exception codes of the goldens and the oracle; the device reports METIS_FATAL_* codes (device_exceptions)
EXC = {'': 0, 'KeyError': 1, 'IndexError': 2, 'ZeroDivisionError': 3}
OTHER = 9


def exc_code(e) -> int:
    return EXC.get(type(e).__name__, OTHER) if e is not None else 0


def device_exceptions(status: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(cost, memory) exception codes (EXC) of metis_het_profile_recost's status bytes: a raising get_cost is
    METIS_FATAL_KEY_EXEC; the memory code is the METIS_FATAL_* of the first failing stage."""
    fatal = {0: 0, 1: EXC['KeyError'], 2: EXC['KeyError'], 3: EXC['IndexError'], 6: EXC['ZeroDivisionError']}
    lut = np.full(16, OTHER, dtype=np.int8)
    for k, v in fatal.items():
        lut[k] = v
    status = np.asarray(status, dtype=np.uint8)
    return lut[status & 15], lut[status >> 4]


def sha256(profile: Dict) -> str:
    return hashlib.sha256(json.dumps(profile, sort_keys=True).encode()).hexdigest()


def _types(profile: Dict) -> List[str]:
    return [k for k in profile if k.startswith('DeviceType.')]


def scenario(base: Dict, kind: str, seed: int, node_sequences: Sequence[Sequence[str]]) -> Dict:
    """One scenario profile of ``kind`` (KINDS) made from ``base`` with random.Random(seed):
      base     the profile itself
      compute  one type's layer-computes scaled per key and layer
      memory   the memory of a node sequence's first type scaled (the type whose profile gives every stage its memory
               demand, quirk Q6), so that some candidates stop fitting
      keys     one key removed (never the first type's tp1_bs1, which LayerLoadBalancer's constructor reads) and one
               fb_sync set to 0.0 (a KeyError in get_cost, quirk Q9)
      model    the 'model' section: parameters, optimizer_time and batch_generator
      noise    every value re-drawn within +-10 %"""
    rng = random.Random(seed)
    p = copy.deepcopy(base)
    types = _types(p)
    if kind == 'compute':
        t = rng.choice(types)
        for entry in p[t].values():
            entry['time']['layer-computes'] = [v * rng.uniform(0.5, 2.0) for v in entry['time']['layer-computes']]
    elif kind == 'memory':
        t = 'DeviceType.' + rng.choice(list(node_sequences))[0]
        f = rng.choice([2.0, 3.0, 4.0])
        for entry in p[t].values():
            entry['memory'] = [v * f for v in entry['memory']]
    elif kind == 'keys':
        keys = [(t, k) for t in types for k in p[t] if (t, k) != (types[0], 'tp1_bs1')]
        t, k = rng.choice(keys)
        del p[t][k]
        keys = [(t, k) for t in types for k in p[t]]
        t, k = rng.choice(keys)
        p[t][k]['time']['fb_sync'] = 0.0
    elif kind == 'model':
        m = p['model']
        m['parameters'] = [v * rng.uniform(0.25, 4.0) for v in m['parameters']]
        m['optimizer_time'] = m['optimizer_time'] * rng.uniform(0.25, 4.0)
        m['batch_generator'] = m['batch_generator'] * rng.uniform(0.25, 4.0)
    elif kind == 'noise':
        for t in types:
            for entry in p[t].values():
                tm = entry['time']
                tm['layer-computes'] = [v * rng.uniform(0.9, 1.1) for v in tm['layer-computes']]
                tm['fb_sync'] = tm['fb_sync'] * rng.uniform(0.9, 1.1)
                entry['memory'] = [v * rng.uniform(0.9, 1.1) for v in entry['memory']]
        m = p['model']
        m['parameters'] = [v * rng.uniform(0.9, 1.1) for v in m['parameters']]
        m['optimizer_time'] = m['optimizer_time'] * rng.uniform(0.9, 1.1)
        m['batch_generator'] = m['batch_generator'] * rng.uniform(0.9, 1.1)
    elif kind != 'base':
        raise ValueError(kind)
    return p


def scenarios(base: Dict, seed: int, node_sequences) -> List[Dict]:
    """One scenario of each kind (KINDS, in order), kind k from seed * 100 + k."""
    return [scenario(base, kind, seed * 100 + k, node_sequences) for k, kind in enumerate(KINDS)]


def candidate_args(arr: Dict, seqs) -> List[Tuple]:
    """(plan dict, strategies, partition) of every candidate of a golden's arrays (conftest.load_golden)."""
    out = []
    for i in range(len(arr['cost'])):
        s = int(arr['nstage'][i])
        plan = dict(node_sequence=tuple(seqs[int(arr['ns_idx'][i])]), device_groups=[int(x) for x in arr['groups'][i, :s]],
                    num_stage=int(arr['label_stage'][i]), batches=int(arr['batches'][i]), gbs=None)
        strategies = [(int(d), int(t)) for d, t in zip(arr['dp'][i, :s], arr['tp'][i, :s])]
        out.append((plan, strategies, [int(x) for x in arr['part'][i, :s + 1]]))
    return out


def profile_recost(profile: Dict, cluster: 'orc.OracleCluster', model_dims: Tuple[int, int, int, int], gbs: int,
                   max_bs: int, cands: Sequence[Tuple], corrected: Sequence[str] = ()):
    """The oracle under one scenario profile: (costs, headroom, cost exception codes, memory exception codes), one
    entry per candidate (plan, strategies, partition) of ``cands``.  ``model_dims``: (num_layers, hidden_size,
    sequence_length, vocab_size); the parameters come from the scenario's 'model' section."""
    num_layers, hidden, seq, vocab = model_dims
    model = orc.OracleModel(num_layers, hidden, seq, vocab, profile['model']['parameters'])
    n = len(cands)
    costs, head = np.full(n, np.nan), np.full(n, np.nan)
    cexc, mexc = np.zeros(n, dtype=np.int8), np.zeros(n, dtype=np.int8)
    for i, (plan, strategies, part) in enumerate(cands):
        plan = dict(plan, gbs=gbs)
        groups = plan['device_groups']
        rank_types = orc.rank_types_by_devices(cluster, plan['node_sequence'])
        try:
            costs[i] = orc.het_cost(profile, cluster, model, plan, strategies, part, rank_types, max_bs)
        except Exception as e:                                 # noqa: BLE001 - recorded as the reference raises it
            cexc[i] = exc_code(e)
        m_capa = orc.stage_memory_capacity(cluster, rank_types, groups)
        try:
            if 'Q6' in corrected:
                demand = orc.stage_memory_demand_own_type(profile, part, strategies, groups, rank_types, gbs,
                                                          plan['batches'])
            else:
                demand = orc.stage_memory_demand(profile, part, strategies, groups,
                                                 orc.rank_types_by_nodes(cluster, plan['node_sequence']), gbs,
                                                 plan['batches'])
            head[i] = min(mc - md for mc, md in zip(m_capa, demand))
        except Exception as e:                                 # noqa: BLE001
            mexc[i] = exc_code(e)
    return costs, head, cexc, mexc


def nan_bits(x) -> np.ndarray:
    """fp64 bits with every NaN as one pattern (the device's NaN and numpy's differ in sign)."""
    x = np.asarray(x, dtype=np.float64)
    return np.where(np.isnan(x), np.float64(math.nan), x).view(np.uint64)
