"""Seeded synthetic inputs for the BASELINE.json configs (SURVEY.md section 8d).

Writes a profile directory (reference JSON schema, README.md:61-112 of the
reference as read by data_loader.py:16-37), a hostfile (utils.py:8-24) and a
clusterfile (README.md:203-230).  Only IEEE +,-,*,/ on literals and a seeded
Mersenne twister are used, so the bytes are identical on every machine; the
golden files store a sha256 of what was generated.
"""
from __future__ import annotations

import hashlib
import json
import os
import random
from dataclasses import dataclass, field, replace
from typing import Dict, List, Sequence, Tuple

# relative per-layer time of each device type (A100 == 1.0)
SPEED = {'A100': 1.0, 'H100': 0.55, 'B200': 0.30, 'V100': 2.0, 'P100': 3.1, 'T4': 4.2}
# 1 / tp**0.8 as literals (libm pow is not bit-reproducible across builds)
TP_SCALE = {1: 1.0, 2: 0.5743491774985175, 4: 0.32987697769322355, 8: 0.18946457081379978}
MEMORY_GB = {'A100': 80, 'H100': 80, 'B200': 180, 'V100': 16, 'P100': 15, 'T4': 15}


@dataclass
class Workload:
    """One named search problem: cluster + model + search flags."""
    name: str
    nodes: List[Tuple[str, int]]                 # (device type, gpus on node) in hostfile order
    num_layers: int
    gbs: int
    hidden_size: int
    sequence_length: int
    vocab_size: int
    variance: int = 1
    max_permute_len: int = 4
    max_tp: int = 4
    max_bs: int = 4
    tps: Sequence[int] = (1, 2, 4)
    bss: Sequence[int] = (1, 2, 4)
    seed: int = 0
    memory_gb: Dict[str, float] = field(default_factory=dict)   # override per type
    intra_bw: Dict[str, float] = field(default_factory=dict)    # override per type
    profile_layers: int = 0                      # 0 -> num_layers
    # 'default': one layer shape for every key, scaled by type, tp and bs (the BASELINE configs);
    # 'rough': per-type shapes, per-key noise and memory, planted ties (see _rough_profiles)
    profile_style: str = 'default'
    int_memory: Sequence[str] = ()               # rough: types whose memory lists are all-int
    short_memory: bool = False                   # rough: memory lists one entry shorter than the compute lists
    zero_fb_sync: Sequence[Tuple[str, int, int]] = ()   # rough: keys with forward_backward == sum(layer computes)
    missing: Sequence[Tuple[str, int, int]] = ()        # rough: keys left unprofiled
    # cluster files written node by node (both set or neither): hostfile lines (ip, device type, gpus) in hostfile
    # order, and the clusterfile's (ip, {instance_type, intra_bandwidth, inter_bandwidth, memory}) entries in file order,
    # which may list the types in another order and IPs no hostfile line names.  Unset: one IP per device type
    hosts: Sequence[Tuple[str, str, int]] = ()
    cluster_entries: Sequence[Tuple[str, Dict[str, object]]] = ()

    def device_types(self) -> List[str]:
        seen: List[str] = []
        for t, _ in self.nodes:
            if t not in seen:
                seen.append(t)
        return seen

    def cli_args(self, root: str) -> List[str]:
        return ['--model_name', 'SYN', '--model_size', self.name, '--num_layers', str(self.num_layers),
                '--gbs', str(self.gbs), '--hidden_size', str(self.hidden_size),
                '--sequence_length', str(self.sequence_length), '--vocab_size', str(self.vocab_size),
                '--attention_head_size', '32',
                '--hostfile_path', os.path.join(root, 'hostfile'),
                '--clusterfile_path', os.path.join(root, 'clusterfile.json'),
                '--profile_data_path', os.path.join(root, 'profile'),
                '--max_profiled_tp_degree', str(self.max_tp),
                '--max_profiled_batch_size', str(self.max_bs),
                '--min_group_scale_variance', str(self.variance),
                '--max_permute_len', str(self.max_permute_len)]


def _profile_json(dev: str, tp: int, bs: int, base: List[float], num_layers: int) -> dict:
    lc = [b * SPEED[dev] * bs * TP_SCALE[tp] for b in base]
    total = 0.0
    for x in lc:
        total += x
    mem = [7820 / tp] + [4146 / tp * (1 + 0.1 * bs)] * (num_layers - 2) + [12132 / tp]
    params = [393216000] + [202383360] * (num_layers - 2) + [393220096]
    return {
        'model': {'model_name': 'SYN', 'num_layers': num_layers,
                  'parameters': {'total_parameters_bytes': sum(params),
                                 'parameters_per_layer_bytes': params}},
        'execution_time': {'total_time_ms': 1.4 * total, 'forward_backward_time_ms': 1.2 * total,
                           'batch_generator_time_ms': 0.9, 'layernorm_grads_all_reduce_time_ms': 0.02,
                           'embedding_grads_all_reduce_time_ms': 0.04, 'optimizer_time_ms': 40 / tp,
                           'layer_compute_total_ms': lc},
        'execution_memory': {'total_memory': 0, 'layer_memory_total_mb': mem},
    }


def _rough_shape(rng: random.Random, n: int, first, mid, last) -> Tuple[List[float], List[bool]]:
    """n per-layer values: first(), mid() for the middle layers with runs of equal values, last();
    ``same[j]`` marks a layer that repeats layer j - 1."""
    vals, same = [first()], [False]
    for _ in range(n - 2):
        if len(vals) > 1 and rng.random() < 0.2:
            vals.append(vals[-1])
            same.append(True)
        else:
            vals.append(mid())
            same.append(False)
    return vals + [last()], same + [False]


def _rough_profiles(w: Workload, nl: int, rng: random.Random) -> Dict[Tuple[str, int, int], dict]:
    """Profiles whose values differ by device type, key and layer (profile_style='rough').

    Per type: a compute shape log-uniform over three decades with embedding-like first and last layers, and a memory
    shape of its own.  Per key: compute and memory rows with multiplicative noise (rows of one type are not
    proportional across tp and bs), runs of equal layers kept, forward_backward_time_ms a little above or below the
    layers' sum, or equal to it for the keys in ``w.zero_fb_sync`` (fb_sync == 0.0).  Memory lists are all-int for
    ``w.int_memory`` and all-float otherwise.  The second type repeats the first type's compute row bit for bit at one
    key.  Keys in ``w.missing`` are not written."""
    from .flatten import py312_sum                  # the builtin sum of CPython >= 3.12, the reference's own
    types = w.device_types()
    tie_key = (w.tps[len(w.tps) // 2], w.bss[len(w.bss) // 2])

    def log_uniform():                              # 0.05 .. ~63: 10**(k/10) by repeated products, k in [0, 30)
        x = 0.05
        for _ in range(rng.randrange(30)):
            x *= 1.2589254117941673
        return x * (1 + 0.25 * rng.random())

    out: Dict[Tuple[str, int, int], dict] = {}
    for ti, dev in enumerate(types):
        shape, same = _rough_shape(rng, nl, lambda: 0.2 + 0.3 * rng.random(), log_uniform,
                                   lambda: 3 + 5 * rng.random())
        mshape, msame = _rough_shape(rng, nl, lambda: 6000 + 4000 * rng.random(), lambda: 1500 + 5000 * rng.random(),
                                     lambda: 9000 + 6000 * rng.random())
        speed = SPEED[dev]
        for tp in w.tps:
            for bs in w.bss:
                lc: List[float] = []
                for j in range(nl):
                    lc.append(lc[-1] if same[j] else shape[j] * speed * bs * TP_SCALE[tp] * (0.9 + 0.2 * rng.random()))
                mem: list = []
                for j in range(nl):
                    mem.append(mem[-1] if msame[j] else mshape[j] / tp * (1 + 0.1 * bs) * (0.95 + 0.1 * rng.random()))
                if dev in w.int_memory:
                    mem = [int(m) for m in mem]
                if w.short_memory:
                    mem = mem[:-1]
                if ti == 1 and (tp, bs) == tie_key:
                    lc = list(out[(types[0], tp, bs)]['execution_time']['layer_compute_total_ms'])
                total = py312_sum(lc)
                r = rng.random()
                if (dev, tp, bs) in w.zero_fb_sync:
                    fb = total
                elif r < 0.3:
                    fb = total * (1 - 0.002 * (1 + r))
                else:
                    fb = total * (1.05 + 0.1 * r)
                params = [393216000] + [202383360] * (nl - 2) + [393220096]
                out[(dev, tp, bs)] = {
                    'model': {'model_name': 'SYN', 'num_layers': nl,
                              'parameters': {'total_parameters_bytes': sum(params), 'parameters_per_layer_bytes': params}},
                    'execution_time': {'total_time_ms': 1.4 * total, 'forward_backward_time_ms': fb,
                                       'batch_generator_time_ms': 0.9, 'layernorm_grads_all_reduce_time_ms': 0.02,
                                       'embedding_grads_all_reduce_time_ms': 0.04, 'optimizer_time_ms': 40 / tp,
                                       'layer_compute_total_ms': lc},
                    'execution_memory': {'total_memory': 0, 'layer_memory_total_mb': mem},
                }
    for key in w.missing:
        del out[tuple(key)]
    return out


def materialize(w: Workload, root: str) -> str:
    """Write w's files under ``root``; returns sha256 over all generated bytes."""
    os.makedirs(os.path.join(root, 'profile'), exist_ok=True)
    rng = random.Random(w.seed)
    nl = w.profile_layers or w.num_layers
    rough = _rough_profiles(w, nl, rng) if w.profile_style == 'rough' else None
    if rough is None:
        base = [0.3] + [10 + rng.random() for _ in range(nl - 2)] + [0.4]
    digest = hashlib.sha256()
    for dev in w.device_types():
        for tp in w.tps:
            for bs in w.bss:
                if rough is not None and (dev, tp, bs) not in rough:
                    continue
                prof = rough[(dev, tp, bs)] if rough is not None else _profile_json(dev, tp, bs, base, nl)
                text = json.dumps(prof, indent=1)
                with open(os.path.join(root, 'profile', f'DeviceType.{dev}_tp{tp}_bs{bs}.json'), 'w') as fh:
                    fh.write(text)
                digest.update(text.encode())
    if w.hosts:
        host, cluster = _node_files(w)
    else:
        ips = {dev: f'IP{i + 1}' for i, dev in enumerate(w.device_types())}
        host = ''.join(f'{ips[dev]} {str(n) * 7}\n' for dev, n in w.nodes)   # utils.py:15 reads char 6
        cluster = {ips[dev]: {'instance_type': dev, 'inter_bandwidth': 312500000.0,
                              'intra_bandwidth': w.intra_bw.get(dev, 5312500000.0),
                              'memory': w.memory_gb.get(dev, MEMORY_GB[dev])}
                   for dev in w.device_types()}
    with open(os.path.join(root, 'hostfile'), 'w') as fh:
        fh.write(host)
    digest.update(host.encode())
    text = json.dumps(cluster, indent=2)
    with open(os.path.join(root, 'clusterfile.json'), 'w') as fh:
        fh.write(text)
    digest.update(text.encode())
    return digest.hexdigest()


def _node_files(w: Workload) -> Tuple[str, dict]:
    """(hostfile text, clusterfile dict) of a workload whose cluster is given node by node."""
    if [(dev, n) for _, dev, n in w.hosts] != list(w.nodes):
        raise ValueError(f'{w.name}: hosts do not match nodes')
    cluster = {}
    for ip, entry in w.cluster_entries:
        if ip in cluster:
            raise ValueError(f'{w.name}: clusterfile entry {ip!r} listed twice')
        cluster[ip] = {k: entry[k] for k in ('instance_type', 'inter_bandwidth', 'intra_bandwidth', 'memory')}
    for ip, dev, n in w.hosts:
        if not 1 <= n <= 9 or ip not in cluster or str(cluster[ip]['instance_type']).upper() != dev:
            raise ValueError(f'{w.name}: host {ip!r} ({dev}, {n} GPUs) has no matching clusterfile entry')
    return ''.join(f'{ip} slots={n}\n' for ip, _, n in w.hosts), cluster   # utils.py:15 reads char 6


def node_entry(dev: str, intra_bw: float = 5312500000.0, memory_gb: float = 0, instance_type: str = '') -> dict:
    """One clusterfile entry; memory defaults to MEMORY_GB[dev], instance_type to dev."""
    return {'instance_type': instance_type or dev, 'inter_bandwidth': 312500000.0, 'intra_bandwidth': intra_bw,
            'memory': memory_gb or MEMORY_GB[dev]}


def per_node(w: Workload, name: str, hosts: Sequence[Tuple[str, str, int]],
             entries: Sequence[Tuple[str, Dict[str, object]]], **change) -> Workload:
    """``w`` renamed, on the cluster files ``hosts`` / ``entries`` (see Workload.hosts)."""
    return replace(w, name=name, nodes=[(dev, n) for _, dev, n in hosts], hosts=tuple(hosts),
                   cluster_entries=tuple(entries), **change)


def profile_file_order(w: Workload) -> List[str]:
    """A fixed listing order for the profile directory (pins quirk Q3 in tests/bench)."""
    return [f'DeviceType.{dev}_tp{tp}_bs{bs}.json' for dev in w.device_types() for tp in w.tps for bs in w.bss
            if (dev, tp, bs) not in w.missing]


def _nodes(*spec: Tuple[str, int]) -> List[Tuple[str, int]]:
    out: List[Tuple[str, int]] = []
    for dev, count in spec:
        out += [(dev, 8)] * count
    return out


# BASELINE.json configs (C1 uses the reference's shipped sample files, see tests/golden/fixtures/c1)
WORKLOADS: Dict[str, Workload] = {w.name: w for w in [
    # configs[1]: 2-type 16-GPU, 24-layer BERT-Large shape, gbs 32
    Workload('c2_het16', _nodes(('A100', 1), ('H100', 1)), 24, 32, 1024, 512, 30522),
    # survey KAT-style stand-in with small-memory V100s (forces re-partition / OOM branches)
    Workload('c2_v100', _nodes(('A100', 1), ('V100', 1)), 24, 32, 1024, 512, 30522),
    # mixed-type stages: 1 A100 node + 3 H100 nodes, so 16-GPU groups straddle the type boundary
    Workload('mix32', _nodes(('A100', 1), ('H100', 3)), 12, 32, 1024, 512, 30522),
    # configs[2]: homo 64-GPU, 96-layer GPT-3 shape, gbs 512; mpl 4 (8.3e4 plans) and mpl 6 (7.7e5 plans)
    Workload('c3_homo64_mpl4', _nodes(('A100', 8)), 96, 512, 12288, 2048, 51200, max_permute_len=4),
    Workload('c3_homo64_mpl6', _nodes(('A100', 8)), 96, 512, 12288, 2048, 51200, max_permute_len=6),
    # configs[3]: 3-type 128-GPU, 80-layer Llama-3-70B shape, gbs 1024
    # batch sizes 8 and 16 are profiled but --max_profiled_batch_size stays 4: mixed-type stages then
    # split unevenly (B200 replicas get >4 samples) and exercise the per-candidate KeyError path
    # (cost_estimator.py:166-167) instead of aborting the whole search (quirk Q8)
    Workload('c4_het128', _nodes(('A100', 6), ('H100', 5), ('B200', 5)), 80, 1024, 8192, 8192, 128256,
             bss=(1, 2, 4, 8, 16), memory_gb={'B200': 180}),
    Workload('c4_het128_mpl6', _nodes(('A100', 6), ('H100', 5), ('B200', 5)), 80, 1024, 8192, 8192, 128256,
             bss=(1, 2, 4, 8, 16), max_permute_len=6),
    # small 2-type 32-GPU case with three stages of attempts (tight memory)
    Workload('het32_tight', _nodes(('A100', 2), ('V100', 2)), 24, 64, 2048, 1024, 51200,
             memory_gb={'A100': 40, 'V100': 16}),
    # non power-of-two gbs: the reference aborts with KeyError (bs=3 unprofiled, quirk Q8)
    Workload('fatal_gbs96', _nodes(('A100', 2)), 12, 96, 1024, 512, 30522),
    # BASELINE configs[4] sweep points small enough for the reference to finish (goldens)
    Workload('sweep_n8_t1', _nodes(('A100', 1)), 24, 64, 4096, 1024, 51200, variance=0),
    Workload('sweep_n16_t2_v0', _nodes(('A100', 1), ('H100', 1)), 24, 64, 4096, 1024, 51200, variance=0,
             bss=(1, 2, 4, 8), max_permute_len=5),
    Workload('sweep_n32_t4', [('A100', 8), ('H100', 8), ('B200', 8), ('V100', 8)], 24, 128, 4096, 1024, 51200,
             bss=(1, 2, 4, 8, 16), memory_gb={'V100': 32}),
    # BASELINE configs[4] at >= 128 GPUs with variance 0 (the variance-1 filter collapses these spaces): the
    # reference is run on a stratified sample of the ordinals (tests/golden/make_golden.py name:strat)
    Workload('sweep_n128_t1_v0', _nodes(('A100', 16)), 96, 512, 12288, 2048, 51200, variance=0),
    Workload('sweep_n256_t2_v0', _nodes(('A100', 16), ('H100', 16)), 24, 512, 12288, 2048, 51200, variance=0,
             bss=(1, 2, 4, 8, 16)),
    # nodes with different GPU counts (quirk Q10: the reference maps ranks to nodes, and builds the memory model's
    # rank list, with node 0's count): node 0 larger than the others / smaller (-> IndexError aborts the search)
    Workload('q10_big_first', [('A100', 8), ('A100', 4), ('H100', 4)], 12, 32, 1024, 512, 30522,
             bss=(1, 2, 4, 8, 16), memory_gb={'A100': 24, 'H100': 40}),
    Workload('q10_small_first', [('A100', 4), ('A100', 8), ('H100', 4)], 12, 32, 1024, 512, 30522,
             bss=(1, 2, 4, 8, 16)),
    Workload('q10_small_first_t1', [('A100', 2), ('A100', 4), ('A100', 2)], 12, 16, 1024, 512, 30522),
    # more profiled layers than --num_layers (the reference normalises over all of them, appendix A)
    Workload('long_profile', _nodes(('A100', 2)), 10, 32, 1024, 512, 30522, profile_layers=17),
    # the compiled limits (128 stages, 255 layers): each workload lands in one instantiation of the search kernels
    # <MAXS, MAXL, ONE> (metis_search.cu, metis_het_search), at or next to a boundary.  Memories are tuned so that
    # candidates are costed at (or next to) the largest stage count and re-partitioning happens
    Workload('lim_s64_l128', _nodes(('A100', 8)), 128, 8, 4096, 1024, 51200, max_permute_len=1),        # <64,128,1>
    Workload('lim_s64_l128_t2', _nodes(('A100', 4), ('H100', 4)), 128, 8, 4096, 1024, 51200, max_permute_len=1,
             bss=(1, 2, 4, 8)),                                                                        # <64,128,0>
    Workload('lim_s65', _nodes(('A100', 16)), 65, 8, 4096, 1024, 51200, max_permute_len=1,
             memory_gb={'A100': 18}),                                                                  # <96,128,1>
    Workload('lim_s96_t2', _nodes(('A100', 8), ('H100', 8)), 96, 8, 4096, 1024, 51200, max_permute_len=1,
             bss=(1, 2, 4, 8), memory_gb={'A100': 48, 'H100': 48}),                                    # <96,128,0>
    Workload('lim_s97', _nodes(('A100', 16)), 97, 8, 4096, 1024, 51200, max_permute_len=1,
             memory_gb={'A100': 64}),                                                                  # <128,256,1>
    Workload('lim_l129_t2', _nodes(('A100', 1), ('H100', 1)), 129, 8, 4096, 1024, 51200, max_permute_len=1,
             bss=(1, 2, 4, 8), memory_gb={'A100': 240, 'H100': 240}),                                  # <128,256,0> by L
    Workload('lim_s128_l255', _nodes(('A100', 16)), 255, 8, 4096, 1024, 51200, max_permute_len=1),     # <128,256,1>
    Workload('lim_s128_t2', _nodes(('A100', 8), ('H100', 8)), 129, 2, 4096, 1024, 51200, max_permute_len=1,
             bss=(1, 2, 4, 8), memory_gb={'A100': 58, 'H100': 64}),                                    # <128,256,0> by S
    # rough profiles (profile_style='rough'): memory that depends on the device type, compute rows that are not one
    # shape scaled, int memory lists, fb_sync == 0.0 and unprofiled keys, so that which type's / key's table the
    # search reads changes the result (tests/test_rough_profiles.py)
    # mixed-type stages and tight memory; the two node sequences start with different types (quirk Q6)
    Workload('rough_mix2', _nodes(('A100', 1), ('V100', 3)), 12, 32, 1024, 512, 30522, bss=(1, 2, 4, 8, 16),
             memory_gb={'A100': 40, 'V100': 16}, int_memory=('V100',), seed=101, profile_style='rough'),
    # three types, all six node sequences, nodes of 4 GPUs
    Workload('rough_t3', [('A100', 4), ('H100', 4), ('V100', 4), ('V100', 4)], 10, 16, 1024, 512, 30522,
             bss=(1, 2, 4, 8, 16), memory_gb={'A100': 24, 'H100': 32, 'V100': 16}, int_memory=('H100',), seed=102,
             profile_style='rough'),
    # unequal nodes, node 0 largest (quirk Q10 rank lists) with type-dependent memory
    Workload('rough_q10', [('A100', 8), ('H100', 4), ('V100', 4)], 12, 32, 1024, 512, 30522, bss=(1, 2, 4, 8, 16),
             memory_gb={'A100': 24, 'H100': 40, 'V100': 16}, seed=103, profile_style='rough'),
    # 15 profiled layers for 10 model layers, memory lists of 14 int entries
    Workload('rough_long_int', _nodes(('A100', 1), ('H100', 1)), 10, 32, 1024, 512, 30522, profile_layers=15,
             memory_gb={'A100': 16, 'H100': 24}, int_memory=('A100', 'H100'), short_memory=True, seed=104,
             profile_style='rough'),
    # fb_sync == 0.0 at two keys (per-candidate KeyError, quirk Q9) and a key only one type has
    Workload('rough_keys', [('A100', 4), ('H100', 4), ('H100', 4), ('H100', 4)], 12, 32, 1024, 512, 30522,
             bss=(1, 2, 4, 8, 16), memory_gb={'A100': 24, 'H100': 24}, seed=105,
             zero_fb_sync=(('H100', 2, 2), ('A100', 1, 4)), missing=(('H100', 4, 8),), profile_style='rough'),
    # the same with a searched key missing for one type: the reference aborts with KeyError at plan 11
    Workload('rough_keys_fatal', [('A100', 4), ('H100', 4), ('H100', 4), ('H100', 4)], 12, 32, 1024, 512, 30522,
             bss=(1, 2, 4, 8, 16), memory_gb={'A100': 24, 'H100': 24}, seed=105,
             zero_fb_sync=(('H100', 2, 2), ('A100', 1, 4)), missing=(('H100', 1, 4),), profile_style='rough'),
    # max_permute_len 1 in the larger instantiations: <96,128,0> by the stage count, <128,256,0> by the layer count
    Workload('rough_s66_t2', _nodes(('A100', 8), ('H100', 8)), 66, 8, 4096, 1024, 51200, max_permute_len=1,
             bss=(1, 2, 4, 8), memory_gb={'A100': 48, 'H100': 40}, seed=106, profile_style='rough'),
    Workload('rough_l130_t2', _nodes(('A100', 1), ('H100', 1)), 130, 8, 4096, 1024, 51200, max_permute_len=1,
             bss=(1, 2, 4, 8), memory_gb={'A100': 240, 'H100': 240}, seed=107, profile_style='rough'),
    # single type for the homogeneous path (cost_homo_cluster): int memory, a zero fb_sync, an unprofiled key
    Workload('rough_homo', _nodes(('H100', 2)), 20, 64, 4096, 1024, 51200, bss=(1, 2, 4, 8), memory_gb={'H100': 40},
             zero_fb_sync=(('H100', 2, 1),), missing=(('H100', 4, 8),), int_memory=('H100',), seed=108,
             profile_style='rough'),
]}

# The same problems under bandwidths that differ by device type (the clusterfile holds one intra_bandwidth per IP, and
# a Workload gives every node of a type the same IP, so a per-node difference within a type cannot be written here).
# Bandwidth enters only the cost model: these searches visit the candidates of their base workload, with other costs
# (HetSearchResult.recost, tests/test_recost.py).  They differ from the base only in intra_bw.
WORKLOADS.update({w.name: w for w in [
    replace(WORKLOADS['mix32'], name='bw_mix32', intra_bw={'A100': 2.5e9, 'H100': 9.0e10}),
    replace(WORKLOADS['rough_t3'], name='bw_rough_t3', intra_bw={'A100': 1.25e9, 'H100': 4.0e10, 'V100': 7.5e8}),
]})

# Clusters written node by node (Workload.hosts / cluster_entries), where the reference's four per-node readings part:
# a type's bandwidth on one node is its first hostfile node's (cluster_bandwidth.py:49-54), across nodes the smallest
# of its nodes' (:56-68), its memory the first clusterfile entry of that instance_type (gpu_cluster.py:47-50), and
# the homogeneous path reads hostfile node 0 (tests/test_node_clusters.py).
WORKLOADS.update({w.name: w for w in [
    # mix32's nodes under an IP each, the H100s on three bandwidths: mix32's candidates, other costs
    per_node(WORKLOADS['mix32'], 'node_bw_mix32',
             [('N0', 'A100', 8), ('N1', 'H100', 8), ('N2', 'H100', 8), ('N3', 'H100', 8)],
             [('N0', node_entry('A100')), ('N1', node_entry('H100', 9.0e10)), ('N2', node_entry('H100', 2.5e9)),
              ('N3', node_entry('H100', 4.0e10))]),
    # one type (the <.., ONE> instantiations): node 0 is neither the slowest nor the only bandwidth
    per_node(WORKLOADS['mix32'], 'node_bw_t1', [(f'N{k}', 'A100', 8) for k in range(4)],
             [('N0', node_entry('A100', 4.0e10)), ('N1', node_entry('A100', 1.25e9)),
              ('N2', node_entry('A100', 4.0e10)), ('N3', node_entry('A100', 8.0e9))]),
    # rough profiles, three types: the clusterfile lists the types in another order than the hostfile, its first A100
    # entry is a node the hostfile never names (less memory than the A100 node used), its first V100 entry the second
    # V100 node of the hostfile (more memory than the first), and the V100 nodes differ in bandwidth
    per_node(WORKLOADS['rough_t3'], 'node_mem_order',
             [('N1', 'A100', 4), ('N2', 'H100', 4), ('N3', 'V100', 4), ('N4', 'V100', 4)],
             [('N4', node_entry('V100', 1.5e9, 20)), ('X1', node_entry('A100', 2.5e9, 14)),
              ('N2', node_entry('H100', 4.0e10, 32)), ('N3', node_entry('V100', 9.0e9, 16)),
              ('N1', node_entry('A100', 2.5e9, 24))]),
    # unequal nodes, node 0 largest (quirk Q10 rank lists), the A100 nodes on different bandwidths
    per_node(WORKLOADS['q10_big_first'], 'node_q10', [('N1', 'A100', 8), ('N2', 'A100', 4), ('N3', 'H100', 4)],
             [('N1', node_entry('A100', 3.0e10, 24)), ('N2', node_entry('A100', 2.0e9, 24)),
              ('N3', node_entry('H100', 9.0e10, 40))]),
    # one type: hostfile node 0 (N2) differs in memory and bandwidth from the type's first clusterfile entry (N1)
    per_node(WORKLOADS['mix32'], 'node_homo', [('N2', 'A100', 8), ('N1', 'A100', 8)],
             [('N1', node_entry('A100', 2.5e9, 12)), ('N2', node_entry('A100', 4.0e10, 80))], gbs=64),
    # an instance_type in lower case: the type is known (DeviceType.from_string upper-cases) but its memory is not
    # found (the raw string is compared), so the reference raises TypeError (device_group.py:99-100)
    per_node(WORKLOADS['mix32'], 'node_lower_case', [('N0', 'A100', 8), ('N1', 'H100', 8)],
             [('N0', node_entry('A100', instance_type='a100')), ('N1', node_entry('H100'))]),
]})


def sweep_workload(ndev: int, ntypes: int, variance: int = 1, mpl: int = 4, num_layers: int = 96,
                   gbs: int = 512) -> Workload:
    """configs[4]: search-space sweep 8-512 GPUs x 1-4 device types."""
    order = ['A100', 'H100', 'B200', 'V100'][:ntypes]
    nnodes = max(1, ndev // 8)
    per = 8 if ndev >= 8 else ndev
    nodes = [(order[(i * ntypes) // nnodes], per) for i in range(nnodes)]
    return Workload(f'sweep_n{ndev}_t{ntypes}_v{variance}_m{mpl}', nodes, num_layers, gbs, 12288, 2048, 51200,
                    variance=variance, max_permute_len=mpl, memory_gb={'V100': 32})
