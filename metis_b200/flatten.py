"""Flatten the reference's nested inputs into the dense arrays of ``MetisProblem`` and
enumerate the candidate space into ``MetisPlanSpace`` (include/metis_b200.h).

Host-side logic only (no arithmetic of the search itself happens here, except the
load-time constants the reference also computes once on the host: ``sum(layer-computes)``
per profile key, ``norm_layer_duration`` (model/load_balancer.py:22-27) and the per-type
bandwidth/memory lookups of gpu_cluster.py).
"""
from __future__ import annotations

import ctypes as C
import math
import sys
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import native


def py312_sum(values) -> float:
    """CPython >= 3.12 ``sum`` (Neumaier-compensated for floats, Python/bltinmodule.c) so that
    load-time constants do not depend on the interpreter version running the host code."""
    if sys.version_info >= (3, 12):
        return sum(values)                                  # the interpreter's own sum IS this algorithm
    it = iter(values)
    acc = 0
    for x in it:
        if isinstance(x, int) and not isinstance(x, bool):
            acc += x
            continue
        acc = acc + x
        break
    else:
        return acc
    f, c = float(acc), 0.0
    for x in it:
        if isinstance(x, float):
            t = f + x
            c += ((f - t) + x) if abs(f) >= abs(x) else ((x - t) + f)
            f = t
        else:
            f += float(x)
    if c and math.isfinite(c):
        f += c
    return f


def _numeric_list(values, what: str) -> np.ndarray:
    kinds = {type(v) for v in values}
    if not kinds <= {int, float}:
        raise TypeError(f'{what}: only int/float entries are supported')
    if len(kinds) == 2:
        # CPython's sum() leaves ints un-compensated inside a float list; not representable here
        raise NotImplementedError(f'{what}: mixed int/float arrays are not supported')
    return np.asarray(values, dtype=np.float64)


def _type_name(t) -> str:
    return t.name if hasattr(t, 'name') else str(t)


@dataclass
class FlatProblem:
    """Numpy twin of MetisProblem; ``as_struct`` binds pointers (host or device)."""
    scalars: Dict[str, object]
    arrays: Dict[str, np.ndarray]
    type_names: List[str]
    key_names: List[Tuple[str, int, int]]            # (type, tp, bs) per key id
    node_sequences: List[Tuple[str, ...]]

    def as_struct(self, ptr_of: Callable[[str], int]) -> native.MetisProblem:
        p = native.MetisProblem()
        for k, v in self.scalars.items():
            setattr(p, k, v)
        for name in ('key_index', 'layer_compute', 'layer_memory', 'exec_full', 'fb_sync', 'norm_lc',
                     'type_memory', 'type_bw_first', 'type_bw_min', 'ns_run_type', 'ns_run_end', 'ns_q10_end'):
            setattr(p, name, ptr_of(name))
        return p


def norm_layer_duration(profile_data: Dict) -> List[float]:
    """model/load_balancer.py:22-27: weights from the first-listed type's tp1_bs1 (quirk Q3)."""
    first = next(iter(profile_data))
    durations = profile_data[first]['tp1_bs1']['time']['layer-computes']
    total = py312_sum(durations)
    return [d / total for d in durations]


def cluster_bandwidths(gpu_cluster, type_names: Sequence[str], corrected: Sequence[str] = ()
                       ) -> Tuple[List[float], List[float]]:
    """The bandwidth tables the cost model reads, one entry per device type of ``type_names``: bw_first[T] is the
    intra_bandwidth of the type's first node (cluster_bandwidth.py:49-54), bw_min[T] the smallest between-node
    bandwidth of its nodes (:56-68), which gpu_cluster.py:56-58 reads from intra_bandwidth (quirk Q2) or, with 'Q2' in
    ``corrected``, from the clusterfile's inter_bandwidth.  MetisProblem.type_bw_first / type_bw_min and the scenarios
    of HetSearchResult.recost both come from here."""
    bw_first, bw_min = [], []
    node_ids = list(gpu_cluster.nodes.keys())
    for name in type_names:
        mine = [i for i in node_ids if _type_name(gpu_cluster.nodes[i].device_type) == name]
        bw_first.append(float(gpu_cluster.get_intra_bandwidth(mine[0])))
        if 'Q2' in corrected:
            bw_min.append(float(min(gpu_cluster.nodes_info[gpu_cluster.host_entries[i]['ip']]['inter_bandwidth']
                                    for i in mine)))
        else:
            bw_min.append(float(min(gpu_cluster.get_inter_bandwidth(i) for i in mine)))
    return bw_first, bw_min


def build_problem(profile_data: Dict, gpu_cluster, model_config, gbs: int, max_tp: int, max_bs: int,
                  node_sequences: Sequence[Sequence], norm_lc: Optional[Sequence[float]] = None,
                  corrected: Sequence[str] = ()) -> FlatProblem:
    """``corrected`` (opt-in, SURVEY.md 8(f)-4): 'Q2' fills the between-node bandwidth table from the
    clusterfile's ``inter_bandwidth`` instead of reproducing gpu_cluster.py:56-58, which returns the intra value;
    'Q5' / 'Q6' set the METIS_FIX_* bits evaluated on the device (vote without dropped layers, memory demand from
    the stage's own device type)."""
    nodes = [gpu_cluster.nodes[i] for i in gpu_cluster.nodes.keys()]
    per_node = nodes[0].num_devices                         # gpu_cluster.py:25-26: node 0's count stands for all (Q10)
    type_names: List[str] = []
    for n in nodes:
        if _type_name(n.device_type) not in type_names:
            type_names.append(_type_name(n.device_type))
    if len(type_names) > native.METIS_MAX_TYPES:
        raise NotImplementedError(f'more than {native.METIS_MAX_TYPES} device types')
    if len(node_sequences) > 256:                            # ns_idx travels in 8 bits of the list entries
        raise NotImplementedError('more than 256 node sequences')
    num_layers = model_config.num_layers
    if num_layers > min(native.METIS_MAX_LAYERS, 255):       # layer_partition entries travel as one byte
        raise NotImplementedError('--num_layers > 255')

    num_tp = max(1, int(math.floor(math.log2(max_tp))) + 1) if max_tp >= 1 else 1
    profiled_bs = [1]
    for name in type_names:
        for key in profile_data.get(f'DeviceType.{name}', {}):
            profiled_bs.append(int(key.split('_bs')[1]))
    num_bs = min(max(max(profiled_bs), max_bs, 1), 4096)

    key_index = np.full((len(type_names), num_tp, num_bs), -1, dtype=np.int16)
    key_names: List[Tuple[str, int, int]] = []
    lc_rows, mem_rows, exec_full, fb_sync = [], [], [], []
    for ti, name in enumerate(type_names):
        for key, entry in profile_data.get(f'DeviceType.{name}', {}).items():
            tp = int(key[2:].split('_bs')[0])
            bs = int(key.split('_bs')[1])
            if tp < 1 or tp & (tp - 1) or tp > (1 << (num_tp - 1)) or bs < 1 or bs > num_bs:
                continue                                    # never addressed by the het search
            lc = entry['time']['layer-computes']
            key_index[ti, int(math.log2(tp)), bs - 1] = len(key_names)
            key_names.append((name, tp, bs))
            lc_rows.append(_numeric_list(lc, f'{name} {key} layer_compute_total_ms'))
            mem_rows.append(_numeric_list(entry['memory'], f'{name} {key} layer_memory_total_mb'))
            exec_full.append(float(py312_sum(lc)))
            fb = entry['time'].get('fb_sync')
            fb_sync.append(float(fb) if fb else 0.0)         # falsy -> KeyError in the reference (Q9)
    if not key_names:
        raise KeyError('no profile data for the device types of the cluster')
    if norm_lc is None:
        norm_lc = norm_layer_duration(profile_data)
    lpad = max([num_layers] + [len(r) for r in lc_rows] + [len(r) for r in mem_rows])
    lpad += lpad & 1
    layer_compute = np.zeros((len(key_names), lpad), dtype=np.float64)
    layer_memory = np.zeros((len(key_names), lpad), dtype=np.float64)
    for i, (lc, mem) in enumerate(zip(lc_rows, mem_rows)):
        layer_compute[i, :len(lc)] = lc
        layer_memory[i, :len(mem)] = mem

    type_memory = []
    for name in type_names:
        mem = gpu_cluster.get_device_memory_for_device_type(name)
        if mem is None:
            raise TypeError("unsupported operand type(s) for *: 'NoneType' and 'int'")   # device_group.py:99-100
        type_memory.append(float(mem))
    bw_first, bw_min = cluster_bandwidths(gpu_cluster, type_names, corrected)
    uniform_bw = int(len(set(bw_first + bw_min)) == 1)

    seqs = [tuple(_type_name(t) for t in seq) for seq in node_sequences]
    run_type = np.zeros((len(seqs), len(type_names)), dtype=np.uint8)
    run_end = np.zeros((len(seqs), len(type_names)), dtype=np.int32)
    q10_end = np.zeros((len(seqs), len(type_names)), dtype=np.int32)
    nodes_of = {name: sum(1 for n in nodes if _type_name(n.device_type) == name) for name in type_names}
    for si, seq in enumerate(seqs):
        if sorted(seq) != sorted(type_names):
            raise ValueError('node sequence is not a permutation of the cluster device types')
        total = total_q10 = 0
        for k, name in enumerate(seq):
            total += gpu_cluster.get_num_nodes_by_device_type(name)      # devices of the type: model/device_group.py:22-32
            total_q10 += nodes_of[name] * per_node                       # load_balancer.py:109-119 (Q10)
            run_type[si, k] = type_names.index(name)
            run_end[si, k] = total
            q10_end[si, k] = total_q10

    params = profile_data['model']['parameters']
    scalars = dict(
        num_types=len(type_names), num_tp=num_tp, num_bs=num_bs, num_keys=len(key_names), lpad=lpad,
        num_layers=num_layers, norm_len=len(norm_lc), gbs=gbs, max_tp=max_tp, max_bs=max_bs,
        num_nodes=len(nodes), devices_per_node=per_node, total_devices=int(sum(n.num_devices for n in nodes)),
        num_node_sequences=len(seqs), uniform_bw=uniform_bw, q10_devices=per_node * len(nodes),
        corrected=(1 if 'Q5' in corrected else 0) | (2 if 'Q6' in corrected else 0), reserved1=0,
        sequence_length=int(model_config.sequence_length), hidden_size=int(model_config.hidden_size),
        vocab_size=int(model_config.vocab_size),
        optimizer_time=float(profile_data['model']['optimizer_time']),
        batch_generator=float(profile_data['model']['batch_generator']),
        input_params=float(params[0]), transformer_params=float(params[1]), output_params=float(params[-1]),
        node0_bandwidth=float(gpu_cluster.get_intra_bandwidth(0)),
        node0_memory=float(gpu_cluster.get_device_memory(0)),
    )
    arrays = dict(
        key_index=np.ascontiguousarray(key_index), layer_compute=layer_compute, layer_memory=layer_memory,
        exec_full=np.asarray(exec_full, dtype=np.float64), fb_sync=np.asarray(fb_sync, dtype=np.float64),
        norm_lc=np.asarray(norm_lc, dtype=np.float64),
        type_memory=np.asarray(type_memory, dtype=np.float64),
        type_bw_first=np.asarray(bw_first, dtype=np.float64), type_bw_min=np.asarray(bw_min, dtype=np.float64),
        ns_run_type=run_type, ns_run_end=run_end, ns_q10_end=q10_end,
    )
    return FlatProblem(scalars, arrays, type_names, key_names, seqs)


# ---------------------------------------------------------------------------------------------
# candidate space
# ---------------------------------------------------------------------------------------------
def enumerate_device_groups(num_stages: int, num_gpus: int, variance, max_permute_len: int,
                            lib=None) -> np.ndarray:
    """Rows of gen_dgroups_for_stages_with_variance (search_space/device_group.py:93-107) as
    log2 codes, shape [rows, num_stages]; enumerated by the library's C++ host enumerator."""
    lib = lib or native.load_library()
    n = lib.metis_enum_device_groups(num_stages, num_gpus, float(variance), max_permute_len, None, 0)
    if n < 0:
        raise native.MetisNativeError(f'metis_enum_device_groups failed ({n})')
    out = np.empty((n, num_stages), dtype=np.uint8)
    if n:
        got = lib.metis_enum_device_groups(num_stages, num_gpus, float(variance), max_permute_len,
                                           out.ctypes.data, n)
        if got != n:
            raise native.MetisNativeError('metis_enum_device_groups: inconsistent row count')
    return out


def enumerate_device_group_tables(first_stage: int, last_stage: int, num_gpus: int, variance, max_permute_len: int,
                                  lib=None, out: Optional[np.ndarray] = None) -> Dict[int, np.ndarray]:
    """All row tables for stage counts first_stage..last_stage in one threaded library call.  ``out`` (uint8,
    e.g. the pinned staging buffer of a DeviceProblem) receives the tables when it is large enough."""
    lib = lib or native.load_library()
    n = last_stage - first_stage + 1
    counts = np.zeros(n, dtype=np.int64)
    total = lib.metis_enum_device_group_tables(first_stage, last_stage, num_gpus, float(variance), max_permute_len,
                                               counts.ctypes.data, None, 0)
    if total < 0:
        raise native.MetisNativeError(f'metis_enum_device_group_tables failed ({total})')
    padded = ((max(int(total), 1) + 15) // 16) * 16                              # 16 B multiple for the device copy
    if out is not None and out.dtype == np.uint8 and out.ndim == 1 and out.size >= padded and out.flags.c_contiguous:
        blob = out[:padded]
        blob[int(total):] = 0
    else:
        blob = np.zeros(padded, dtype=np.uint8)
    got = lib.metis_enum_device_group_tables(first_stage, last_stage, num_gpus, float(variance), max_permute_len,
                                             counts.ctypes.data, blob.ctypes.data, int(total))
    if got != total:
        raise native.MetisNativeError('metis_enum_device_group_tables: inconsistent size')
    out: Dict[int, np.ndarray] = {}
    off = 0
    for i in range(n):
        stages = first_stage + i
        size = int(counts[i]) * stages
        out[stages] = blob[off:off + size].reshape(int(counts[i]), stages)   # views into the one blob
        off += size
    out[0] = blob                                                            # the blob itself (offset 0 = first table)
    return out


@dataclass
class FlatPlanSpace:
    """Numpy twin of MetisPlanSpace."""
    num_plans: int
    blocks: np.ndarray            # structured, native.BLOCK_DTYPE
    batches: np.ndarray           # int32, divisors of gbs descending
    rows: np.ndarray              # uint8 blob of all row tables
    tables: Dict[int, Tuple[int, np.ndarray]] = field(default_factory=dict)   # S -> (byte offset, rows)
    rows_total_bytes: int = -1    # device_rows spaces: size of the row blob the GPU writes (rows stays empty)
    comp_recs: Optional[np.ndarray] = None     # native.COMP_DTYPE, device_rows spaces
    comp_pool: Optional[np.ndarray] = None

    def as_struct(self, ptr_of: Callable[[str], int]) -> native.MetisPlanSpace:
        s = native.MetisPlanSpace()
        s.num_plans = self.num_plans
        s.rows_bytes = int(self.rows_total_bytes if self.rows_total_bytes >= 0 else self.rows.size)
        s.num_blocks = len(self.blocks)
        s.num_div = len(self.batches)
        s.max_stage = int(self.blocks['num_stage'].max()) if len(self.blocks) else 1
        s.blocks = ptr_of('blocks')
        s.batches = ptr_of('batches')
        s.rows = ptr_of('rows')
        return s

    def host_rows(self) -> np.ndarray:
        """The row blob on the host; a device_rows space enumerates it on first use (debug / test paths only)."""
        if self.rows.size == 0 and self.comp_recs is not None:
            self.tables._fill()
            return self.tables.blob
        return self.rows

    def locate(self, ordinal: int) -> Tuple[int, int, int, int, np.ndarray]:
        """ordinal -> (ns_idx, label_stage, dg_idx, batches, device_groups) like InterStagePlan."""
        firsts = self.blocks['first_ordinal']
        b = int(np.searchsorted(firsts, ordinal, side='right')) - 1
        blk = self.blocks[b]
        rel = ordinal - int(blk['first_ordinal'])
        row, div = divmod(rel, len(self.batches))
        _, table = self.tables[int(blk['num_stage'])]
        return int(blk['ns_idx']), int(blk['label_stage']), row, int(self.batches[div]), table[row]


def _walk_blocks(num_node_sequences: int, cap: int, nrows_of: Callable[[int], int],
                 corrected: Sequence[str]) -> List[Tuple[int, int, int]]:
    """The (ns_idx, label, stage count) blocks in the order of InterStagePlanGenerator.__next__
    (search_space/plan.py:153-175), including the mislabelled num_stage=1 block of every later node sequence
    (quirk Q1; with 'Q1' in ``corrected`` every node sequence starts with the real one-stage rows)."""
    def next_stage(start: int) -> int:                         # plan.py:130-142
        s = start
        while nrows_of(s) == 0 and s <= cap:
            s += 1
        return s

    if nrows_of(1) == 0:
        raise IndexError('list index out of range')            # plan.py:117-118
    out: List[Tuple[int, int, int]] = []
    ns, label, stages = 0, 1, 1
    while True:
        out.append((ns, label, stages))
        s = next_stage(label + 1)
        if s > cap:
            ns += 1
            if ns >= num_node_sequences:
                break
            if 'Q1' in corrected:
                label, stages = 1, 1
            else:
                label, stages = 1, next_stage(2)               # plan.py:144-148 (Q1)
            if nrows_of(stages) == 0:
                raise IndexError('list index out of range')    # plan.py:173
        else:
            label, stages = s, s
    return out


def _blocks_array(plan_blocks, nrows_of, offset_of, ndiv: int) -> Tuple[np.ndarray, int]:
    blocks = np.zeros(len(plan_blocks), dtype=native.BLOCK_DTYPE)
    ordinal = 0
    for i, (ns_idx, label, stages) in enumerate(plan_blocks):
        blocks[i]['first_ordinal'] = ordinal
        blocks[i]['rows_offset'] = offset_of(stages)
        blocks[i]['num_rows'] = nrows_of(stages)
        blocks[i]['ns_idx'] = ns_idx
        blocks[i]['label_stage'] = label
        blocks[i]['num_stage'] = stages
        ordinal += nrows_of(stages) * ndiv
    return blocks, ordinal


def _check_stage_limit(plan_blocks) -> None:
    """The search kernels hold at most METIS_MAX_STAGES stages per plan (scratch, detail rows); refuse a larger space
    here, before its rows are uploaded or written on the GPU, like the other limits of the flattening."""
    most = max(stages for _, _, stages in plan_blocks)
    if most > native.METIS_MAX_STAGES:
        raise NotImplementedError(f'more than {native.METIS_MAX_STAGES} pipeline stages ({most})')


def build_plan_space(num_node_sequences: int, num_devices: int, gbs: int, num_layers: int, variance,
                     max_permute_len: int, lib=None, rows_out: Optional[np.ndarray] = None,
                     corrected: Sequence[str] = (), device_rows: bool = False) -> FlatPlanSpace:
    """The candidate space of one search.  ``device_rows`` (SURVEY.md 8(f)-1): the host only lists the compositions
    (``comp_recs`` / ``comp_pool``) and the GPU writes the rows (metis_generate_rows); ``rows`` stays empty and
    ``tables`` is filled by the host enumerator only if somebody asks for it."""
    cap = min(num_devices, num_layers)
    lib = lib or native.load_library()
    batches = [b for b in range(gbs, 0, -1) if gbs % b == 0]   # plan.py:120-124
    if device_rows:
        space = build_device_plan_space(num_node_sequences, num_devices, gbs, num_layers, variance, max_permute_len,
                                        lib, corrected)
        if space is not None:
            if not fits_one_search(space):
                raise NotImplementedError('device-group tables of 4 GiB or more / more than 2^32 plans are not supported')
            return space
        # a composition with more merged groups than the device kernel handles: enumerate on the host
    cache: Dict[int, np.ndarray] = enumerate_device_group_tables(1, cap + 1, num_devices, variance, max_permute_len, lib,
                                                                 rows_out)
    blob = cache.pop(0)
    base_addr = blob.__array_interface__['data'][0]
    nrows_of = lambda st: len(cache[st]) if st in cache else 0                           # noqa: E731
    offset_of = lambda st: cache[st].__array_interface__['data'][0] - base_addr         # noqa: E731
    plan_blocks = _walk_blocks(num_node_sequences, cap, nrows_of, corrected)
    _check_stage_limit(plan_blocks)
    blocks, total = _blocks_array(plan_blocks, nrows_of, offset_of, len(batches))
    tables = {st: (offset_of(st), cache[st]) for _, _, st in plan_blocks}
    if blob.size > 0xFFFFFFFF:                               # list entries address a row with 32 bits
        raise NotImplementedError('device-group tables of 4 GiB or more are not supported')
    if total > 0xFFFFFFF0:
        raise NotImplementedError('more than 2^32 inter-stage plans')
    return FlatPlanSpace(total, blocks, np.asarray(batches, dtype=np.int32), blob, tables)


class _LazyTables(dict):
    """S -> (byte offset, rows): filled by the host enumerator on first use (device_rows spaces)."""

    def __init__(self, cap, num_devices, variance, max_permute_len):
        super().__init__()
        self._args = (cap, num_devices, variance, max_permute_len)
        self._done = False
        self.blob = None

    def _fill(self):
        if not self._done:
            cap, num_devices, variance, mpl = self._args
            cache = enumerate_device_group_tables(1, cap + 1, num_devices, variance, mpl)
            blob = self.blob = cache.pop(0)
            base = blob.__array_interface__['data'][0]
            for st, rows in cache.items():
                dict.__setitem__(self, st, (rows.__array_interface__['data'][0] - base, rows))
            self._done = True

    def __getitem__(self, key):
        self._fill()
        return dict.__getitem__(self, key)

    def __contains__(self, key):
        self._fill()
        return dict.__contains__(self, key)


# One search holds at most this many plans (a list entry and a record carry the ordinal in 32 bits) and rows of
# less than 4 GiB (a list entry addresses its row with a 32-bit byte offset).
MAX_SEARCH_PLANS = 0xFFFFFFF0
MAX_SEARCH_ROW_BYTES = 0xFFFFFFFF


def fits_one_search(space: FlatPlanSpace) -> bool:
    """Whether ``space`` is within the 32-bit limits of one metis_het_search call."""
    return space.num_plans <= MAX_SEARCH_PLANS and int(space.rows_total_bytes) <= MAX_SEARCH_ROW_BYTES


def build_device_plan_space(num_node_sequences: int, num_devices: int, gbs: int, num_layers: int, variance,
                            max_permute_len: int, lib=None, corrected: Sequence[str] = ()) -> Optional[FlatPlanSpace]:
    """The whole candidate space as a device_rows space (compositions listed on the host, rows written by the GPU),
    WITHOUT the limits of one search: the input of plan_windows.  None when a composition has more merged groups than
    the row kernel handles (such spaces are enumerated on the host by build_plan_space)."""
    cap = min(num_devices, num_layers)
    lib = lib or native.load_library()
    batches = [b for b in range(gbs, 0, -1) if gbs % b == 0]   # plan.py:120-124
    counts, recs, pool, most = enumerate_compositions(1, cap + 1, num_devices, variance, max_permute_len, lib)
    if most > native.METIS_MAX_PERMUTE_GROUPS:
        return None
    offsets, off = {}, 0
    for stages in range(1, cap + 2):
        offsets[stages] = off
        off += int(counts[stages - 1]) * stages
    nrows_of = lambda st: int(counts[st - 1]) if 1 <= st <= cap + 1 else 0     # noqa: E731
    plan_blocks = _walk_blocks(num_node_sequences, cap, nrows_of, corrected)
    _check_stage_limit(plan_blocks)
    blocks, total = _blocks_array(plan_blocks, nrows_of, lambda st: offsets[st], len(batches))
    space = FlatPlanSpace(total, blocks, np.asarray(batches, dtype=np.int32), np.zeros(0, dtype=np.uint8))
    space.rows_total_bytes = off
    space.comp_recs, space.comp_pool = recs, pool
    space.tables = _LazyTables(cap, num_devices, variance, max_permute_len)
    return space


@dataclass
class PlanWindow:
    """A contiguous ordinal range of a larger space, as a space of its own: global ordinal = ``base`` + the window's
    ordinal.  Its blocks cover whole composition slices (METIS_COMP_SLICE_ROWS rows) of the parent's blocks; row r of
    window block b is row ``row_base[b] + r`` of the parent's block.  The window's rows are the union of the row ranges
    its blocks cover, per stage count (node sequences share them), written by metis_generate_rows from ``comp_recs``."""
    base: int
    space: FlatPlanSpace
    row_base: np.ndarray          # int64 per window block

    def plan_at(self, ordinal: int) -> Tuple[int, int, int, int, int, int]:
        """Global ``ordinal`` -> (ns_idx, label_stage, dg_idx, batches, num_stage, byte offset of its row in the
        window's rows); dg_idx is the row in the whole space's table of that stage count, as in InterStagePlan."""
        return _plan_at(self.base, self.space, self.row_base, ordinal)

    def locate(self, ordinal: int, rows: np.ndarray) -> Tuple[int, int, int, int, np.ndarray]:
        """Global ``ordinal`` -> (ns_idx, label_stage, dg_idx, batches, device_groups) like FlatPlanSpace.locate, with
        the codes read from ``rows`` (the window's row blob, e.g. generated on the host)."""
        ns, label, dg, batches, S, at = self.plan_at(ordinal)
        return ns, label, dg, batches, rows[at:at + S]

    def arena_sizes(self) -> Dict[str, int]:
        """Bytes of the space's tables in a DeviceProblem arena (search.search_windows sizes one arena for all)."""
        return _arena_sizes(self.space, self.space.comp_recs.nbytes, self.space.comp_pool.nbytes)


def _plan_at(base: int, sp: FlatPlanSpace, row_base: np.ndarray, ordinal: int) -> Tuple[int, int, int, int, int, int]:
    rel = ordinal - base
    if not 0 <= rel < sp.num_plans:
        raise IndexError(f'ordinal {ordinal} is not in this window')
    b = int(np.searchsorted(sp.blocks['first_ordinal'], rel, side='right')) - 1
    blk = sp.blocks[b]
    row, div = divmod(rel - int(blk['first_ordinal']), len(sp.batches))
    S = int(blk['num_stage'])
    return (int(blk['ns_idx']), int(blk['label_stage']), int(row_base[b]) + row, int(sp.batches[div]), S,
            int(blk['rows_offset']) + row * S)


def _arena_sizes(space: FlatPlanSpace, rec_bytes: int, pool_bytes: int) -> Dict[str, int]:
    return dict(blocks=space.blocks.nbytes, batches=space.batches.nbytes, comp_recs=int(rec_bytes),
                comp_pool=int(pool_bytes), rows=int(space.rows_total_bytes))


def window_bytes(space: FlatPlanSpace, plan_bytes: float, row_bytes: float, rec_bytes: float) -> float:
    """Device memory of searching ``space`` under the cost model of plan_windows."""
    return space.num_plans * plan_bytes + int(space.rows_total_bytes) * row_bytes + len(space.comp_recs) * rec_bytes


def _slices_by_stage(space: FlatPlanSpace) -> Dict[int, Tuple[int, np.ndarray]]:
    """S -> (index of the first composition record of S, row boundaries of its slices: K+1 int64 values, 0 .. rows)."""
    recs = space.comp_recs
    st = recs['stages'].astype(np.int64)
    out = {}
    for S in np.unique(space.blocks['num_stage']).tolist():
        lo, hi = int(np.searchsorted(st, S, side='left')), int(np.searchsorted(st, S, side='right'))
        first = (recs['row_offset'][lo:hi] - recs['row_offset'][lo]) // S
        nrows = int(space.blocks['num_rows'][space.blocks['num_stage'] == S][0])
        out[S] = (lo, np.append(first, nrows).astype(np.int64))
    return out


def _uncovered(k0: int, c: np.ndarray, bounds: np.ndarray, covered: List[Tuple[int, int]]):
    """For slice ranges [k0, c) (c an array): slices and rows not yet in ``covered`` (disjoint slice intervals)."""
    new_k = c - k0
    new_r = bounds[c] - bounds[k0]
    for a, b in covered:
        lo = max(k0, a)
        hi = np.minimum(c, b)
        hit = hi > lo
        new_k = new_k - np.where(hit, hi - lo, 0)
        new_r = new_r - np.where(hit, bounds[np.where(hit, hi, lo)] - bounds[lo], 0)
    return new_k, new_r


def arena_bytes(windows: Sequence[PlanWindow], plan_bytes: float, row_bytes: float, rec_bytes: float) -> float:
    """Device memory of searching ``windows`` one after the other in one arena and workspace sized for all of them:
    the most plans, the most rows and the most composition records of any window, under window_bytes' cost model."""
    return (max(w.space.num_plans for w in windows) * plan_bytes
            + max(int(w.space.rows_total_bytes) for w in windows) * row_bytes
            + max(len(w.space.comp_recs) for w in windows) * rec_bytes)


def plan_windows(space: FlatPlanSpace, budget: float, plan_bytes: float = 1.0, row_bytes: float = 0.0,
                 rec_bytes: float = 0.0) -> List[PlanWindow]:
    """Cut a device_rows space (build_device_plan_space) into windows, in ordinal order, each within the limits of one
    search (fewer than 2^32 plans, rows below 4 GiB), such that one arena and workspace sized for all of them fit
    ``budget`` bytes of device memory (arena_bytes), counted as ``plan_bytes`` per plan, ``row_bytes`` per byte of
    rows and ``rec_bytes`` per composition record.  Cuts fall on composition slices; a window holds at least one
    slice, whatever the budget."""
    target = budget
    for _ in range(8):
        windows = _cut_windows(space, target, plan_bytes, row_bytes, rec_bytes)
        peak = arena_bytes(windows, plan_bytes, row_bytes, rec_bytes)
        if peak <= budget or target <= 0:
            break
        # the window with the most plans and the one with the most rows differ: cut every window smaller
        target = min(target * budget / peak, target - 1)
    return windows


def _cut_windows(space: FlatPlanSpace, budget: float, plan_bytes: float, row_bytes: float,
                 rec_bytes: float) -> List[PlanWindow]:
    """Greedy cut of plan_windows: each window on its own within ``budget`` (window_bytes)."""
    if space.comp_recs is None:
        raise NotImplementedError('only spaces whose rows the GPU writes (device_rows) can be searched in windows')
    ndiv = len(space.batches)
    slices = _slices_by_stage(space)
    windows: List[PlanWindow] = []
    seg: List[Tuple[int, int, int]] = []                  # (parent block, first slice, end slice)
    covered: Dict[int, List[Tuple[int, int]]] = {}        # S -> disjoint slice intervals of the window's rows
    state = [0, 0, 0, 0]                                  # plans, row bytes, records, base ordinal

    def close():
        windows.append(_make_window(space, slices, seg, covered, state[3]))
        state[3] += state[0]
        state[:3] = [0, 0, 0]
        seg.clear()
        covered.clear()

    def add(b, S, k0, k1, bounds):
        nk, nr = _uncovered(k0, np.asarray([k1]), bounds, covered.get(S, []))
        state[0] += int(bounds[k1] - bounds[k0]) * ndiv
        state[1] += int(nr[0]) * S
        state[2] += int(nk[0])
        seg.append((b, k0, k1))
        ivs = sorted(covered.get(S, []) + [(k0, k1)])
        merged = [ivs[0]]
        for a, e in ivs[1:]:
            if a <= merged[-1][1]:
                merged[-1] = (merged[-1][0], max(merged[-1][1], e))
            else:
                merged.append((a, e))
        covered[S] = merged

    for b in range(len(space.blocks)):
        S = int(space.blocks['num_stage'][b])
        bounds = slices[S][1]
        K = len(bounds) - 1
        k0 = 0
        while k0 < K:
            span, fit = 256, k0
            while True:                                   # largest end slice that fits, probing a growing span
                c = np.arange(k0 + 1, min(K, k0 + span) + 1, dtype=np.int64)
                nk, nr = _uncovered(k0, c, bounds, covered.get(S, []))
                plans = state[0] + (bounds[c] - bounds[k0]) * ndiv
                rows = state[1] + nr * S
                cost = plans * plan_bytes + rows * row_bytes + (state[2] + nk) * rec_bytes
                ok = (plans <= MAX_SEARCH_PLANS) & (rows <= MAX_SEARCH_ROW_BYTES) & (cost <= budget)
                n_ok = int(np.argmin(ok)) if not ok.all() else len(ok)
                if n_ok:
                    fit = int(c[n_ok - 1])
                if n_ok < len(ok) or c[-1] == K:
                    break
                span *= 4
            if fit == k0:
                if seg:                                   # nothing more fits: the next window starts here
                    close()
                    continue
                fit = k0 + 1                              # an empty window takes one slice
            add(b, S, k0, fit, bounds)
            k0 = fit
            if k0 < K:
                close()
    if seg:
        close()
    return windows


def _make_window(space: FlatPlanSpace, slices, seg, covered, base: int) -> PlanWindow:
    ndiv = len(space.batches)
    recs = space.comp_recs
    at: Dict[Tuple[int, int], int] = {}                   # (S, interval start) -> byte offset in the window's rows
    parts, off = [], 0
    for S in sorted(covered):
        lo, bounds = slices[S]
        for a, e in covered[S]:
            at[(S, a)] = off
            part = recs[lo + a:lo + e].copy()
            part['row_offset'] = part['row_offset'] - part['row_offset'][0] + off
            parts.append(part)
            off += int(bounds[e] - bounds[a]) * S
    blocks = np.zeros(len(seg), dtype=native.BLOCK_DTYPE)
    row_base = np.zeros(len(seg), dtype=np.int64)
    ordinal = 0
    for i, (b, k0, k1) in enumerate(seg):
        src = space.blocks[b]
        S = int(src['num_stage'])
        bounds = slices[S][1]
        a = next(a for a, e in covered[S] if a <= k0 and k1 <= e)
        blocks[i] = src
        blocks[i]['first_ordinal'] = ordinal
        blocks[i]['rows_offset'] = at[(S, a)] + int(bounds[k0] - bounds[a]) * S
        blocks[i]['num_rows'] = int(bounds[k1] - bounds[k0])
        row_base[i] = bounds[k0]
        ordinal += int(bounds[k1] - bounds[k0]) * ndiv
    w = FlatPlanSpace(ordinal, blocks, space.batches, np.zeros(0, dtype=np.uint8))
    w.rows_total_bytes = off
    w.comp_recs = np.concatenate(parts) if parts else recs[:0].copy()
    w.comp_pool = space.comp_pool
    return PlanWindow(base, w, row_base)


def enumerate_compositions(first_stage: int, last_stage: int, num_gpus: int, variance, max_permute_len: int, lib=None):
    """metis_enum_compositions: (rows per stage count, MetisCompRec array, pool bytes, largest number of merged groups)."""
    import ctypes as C
    lib = lib or native.load_library()
    n = last_stage - first_stage + 1
    counts = np.zeros(n, dtype=np.int64)
    pool_bytes, most = C.c_int64(0), C.c_int32(0)
    ncomp = lib.metis_enum_compositions(first_stage, last_stage, num_gpus, float(variance), max_permute_len,
                                        counts.ctypes.data, None, 0, None, 0, C.byref(pool_bytes), C.byref(most))
    if ncomp < 0:
        raise native.MetisNativeError(f'metis_enum_compositions failed ({ncomp})')
    recs = np.zeros(max(int(ncomp), 1), dtype=native.COMP_DTYPE)
    pool = np.zeros(max(int(pool_bytes.value), 16), dtype=np.uint8)
    got = lib.metis_enum_compositions(first_stage, last_stage, num_gpus, float(variance), max_permute_len,
                                      counts.ctypes.data, recs.ctypes.data, int(ncomp), pool.ctypes.data,
                                      int(pool_bytes.value), C.byref(pool_bytes), C.byref(most))
    if got != ncomp:
        raise native.MetisNativeError('metis_enum_compositions: inconsistent count')
    return counts, recs[:int(ncomp)], pool, int(most.value)


# ---------------------------------------------------------------------------------------------
# device listing (SURVEY.md 8(f)-1): the GPU lists the compositions (metis_list_*, metis_b200.listing), the host plans
# the windows from the rows of each stage count and holds one window's records at a time
# ---------------------------------------------------------------------------------------------
def count_compositions(num_devices: int, cap: int, variance, max_permute_len: int, lib=None) -> int:
    """Compositions of stage counts 1..cap (what metis_enum_compositions would list), from the counting table of the
    device listing; host only, no listing."""
    lib = lib or native.load_library()
    listing = native.MetisListing(1, cap, num_devices, max_permute_len, float(variance), 1, 0)
    comps = np.zeros(cap, dtype=np.int64)
    n = lib.metis_list_workspace_bytes(C.byref(listing), comps.ctypes.data)
    if n < 0:
        native.check(int(n), 'metis_list_workspace_bytes')
    return int(comps.sum())


def listed_plan_space(num_node_sequences: int, num_devices: int, gbs: int, num_layers: int, rows_per_stage,
                      corrected: Sequence[str] = ()) -> FlatPlanSpace:
    """The block list of a space whose compositions the GPU lists: ``rows_per_stage[S - 1]`` = rows of stage count S.
    The space has no records (``comp_recs`` is None); plan_listed_windows cuts it into windows that get theirs."""
    cap = min(num_devices, num_layers)
    batches = [b for b in range(gbs, 0, -1) if gbs % b == 0]   # plan.py:120-124
    nrows_of = lambda st: int(rows_per_stage[st - 1]) if 1 <= st <= min(cap, len(rows_per_stage)) else 0  # noqa: E731
    offsets, off = {}, 0
    for stages in range(1, cap + 1):
        offsets[stages] = off
        off += nrows_of(stages) * stages
    plan_blocks = _walk_blocks(num_node_sequences, cap, nrows_of, corrected)
    _check_stage_limit(plan_blocks)
    blocks, total = _blocks_array(plan_blocks, nrows_of, lambda st: offsets[st], len(batches))
    space = FlatPlanSpace(total, blocks, np.asarray(batches, dtype=np.int32), np.zeros(0, dtype=np.uint8))
    space.rows_total_bytes = off
    return space


class ListedWindow:
    """A window of a listed space (plan_listed_windows), with PlanWindow's interface: ``base``, ``row_base``,
    ``plan_at`` / ``locate`` and ``space``, a FlatPlanSpace whose ``comp_recs`` / ``comp_pool`` are the window's own.
    The records are written by the device listing when ``space`` is asked for (``emit(ranges)`` -> (recs, pool)); the
    listing keeps the last window's only, so the host never holds more than one window's records."""

    def __init__(self, base: int, layout: FlatPlanSpace, row_base: np.ndarray, ranges: np.ndarray, rec_bound: int,
                 listing):
        self.base = base
        self.layout = layout          # blocks, batches, plans, rows; no records
        self.row_base = row_base
        self.ranges = ranges          # native.RANGE_DTYPE: the window's rows, range after range
        self.rec_bound = rec_bound    # at most one record per row
        self.listing = listing        # .window_space(window) -> FlatPlanSpace, .size(ranges) -> (records, pool bytes)
        self.num_recs = self.pool_bytes = None

    @property
    def space(self) -> FlatPlanSpace:
        return self.listing.window_space(self)

    def plan_at(self, ordinal: int) -> Tuple[int, int, int, int, int, int]:
        return _plan_at(self.base, self.layout, self.row_base, ordinal)

    def locate(self, ordinal: int, rows: np.ndarray) -> Tuple[int, int, int, int, np.ndarray]:
        ns, label, dg, batches, S, at = self.plan_at(ordinal)
        return ns, label, dg, batches, rows[at:at + S]

    def sized(self) -> 'ListedWindow':
        """Ask the listing for the window's exact record count and pool size (no records written)."""
        if self.num_recs is None:
            self.num_recs, self.pool_bytes = self.listing.size(self.ranges)
        return self

    def arena_sizes(self) -> Dict[str, int]:
        self.sized()
        return _arena_sizes(self.layout, self.num_recs * np.dtype(native.COMP_DTYPE).itemsize, self.pool_bytes)


def _row_union(ivs: List[Tuple[int, int]], a: int, e: int) -> List[Tuple[int, int]]:
    out: List[Tuple[int, int]] = []
    for x, y in sorted(ivs + [(a, e)]):
        if out and x <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], y))
        else:
            out.append((x, y))
    return out


def _new_rows(ivs: List[Tuple[int, int]], a: int, e: int) -> int:
    """Rows of [a, e) outside the disjoint intervals ``ivs``."""
    return (e - a) - sum(max(0, min(e, y) - max(a, x)) for x, y in ivs)


def plan_listed_windows(space: FlatPlanSpace, budget: float, plan_bytes: float = 1.0, row_bytes: float = 0.0,
                        rec_bytes: float = 0.0, listing=None) -> List[ListedWindow]:
    """plan_windows for a listed space (listed_plan_space): windows in ordinal order, each within the limits of one
    search, such that one arena sized for all of them fits ``budget`` under the same cost model, counting one
    composition record per row (a record holds at least one row; the exact count is not known before the window is
    listed).  Cuts fall on any row; a window holds at least one slice's rows (METIS_COMP_SLICE_ROWS), whatever the
    budget.  Deterministic: every rank cuts the same windows from the same budget."""
    target = budget
    for _ in range(8):
        windows = _cut_listed(space, target, plan_bytes, row_bytes, rec_bytes, listing)
        peak = (max(w.layout.num_plans for w in windows) * plan_bytes
                + max(int(w.layout.rows_total_bytes) for w in windows) * row_bytes
                + max(w.rec_bound for w in windows) * rec_bytes)
        if peak <= budget or target <= 0:
            break
        target = min(target * budget / peak, target - 1)
    return windows


METIS_COMP_SLICE_ROWS = 64


def _cut_listed(space: FlatPlanSpace, budget: float, plan_bytes: float, row_bytes: float, rec_bytes: float,
                listing) -> List[ListedWindow]:
    ndiv = len(space.batches)
    windows: List[ListedWindow] = []
    seg: List[Tuple[int, int, int]] = []                  # (parent block, first row, end row)
    covered: Dict[int, List[Tuple[int, int]]] = {}        # S -> disjoint row intervals of the window's rows
    state = [0, 0, 0, 0]                                  # plans, row bytes, rows (record bound), base ordinal

    def close():
        windows.append(_listed_window(space, seg, covered, state[3], state[2], listing))
        state[3] += state[0]
        state[:3] = [0, 0, 0]
        seg.clear()
        covered.clear()

    for b in range(len(space.blocks)):
        S, n = int(space.blocks['num_stage'][b]), int(space.blocks['num_rows'][b])
        r = 0
        while r < n:
            ivs = covered.get(S, [])

            def fits(e: int) -> bool:
                new = _new_rows(ivs, r, e)
                plans, rows = state[0] + (e - r) * ndiv, state[1] + new * S
                cost = plans * plan_bytes + rows * row_bytes + (state[2] + new) * rec_bytes
                return plans <= MAX_SEARCH_PLANS and rows <= MAX_SEARCH_ROW_BYTES and cost <= budget

            if fits(n):
                fit = n
            else:                                         # largest end row that fits (the cost grows with it)
                lo, hi = r, n
                while hi - lo > 1:
                    mid = (lo + hi) // 2
                    if fits(mid):
                        lo = mid
                    else:
                        hi = mid
                fit = lo
            if fit == r:
                if seg:                                   # nothing more fits: the next window starts here
                    close()
                    continue
                fit = min(n, r + METIS_COMP_SLICE_ROWS)   # an empty window takes one slice
            new = _new_rows(ivs, r, fit)
            state[0] += (fit - r) * ndiv
            state[1] += new * S
            state[2] += new
            seg.append((b, r, fit))
            covered[S] = _row_union(ivs, r, fit)
            r = fit
            if r < n:
                close()
    if seg:
        close()
    return windows


def _listed_window(space: FlatPlanSpace, seg, covered, base: int, rec_bound: int, listing) -> ListedWindow:
    ndiv = len(space.batches)
    ranges = np.zeros(sum(len(v) for v in covered.values()), dtype=native.RANGE_DTYPE)
    at: Dict[Tuple[int, int], int] = {}                   # (S, interval start) -> byte offset in the window's rows
    k = off = 0
    for S in sorted(covered):
        for a, e in covered[S]:
            ranges[k] = (S, 0, a, e)
            at[(S, a)] = off
            off += (e - a) * S
            k += 1
    blocks = np.zeros(len(seg), dtype=native.BLOCK_DTYPE)
    row_base = np.zeros(len(seg), dtype=np.int64)
    ordinal = 0
    for i, (b, r0, r1) in enumerate(seg):
        src = space.blocks[b]
        S = int(src['num_stage'])
        a = next(a for a, e in covered[S] if a <= r0 and r1 <= e)
        blocks[i] = src
        blocks[i]['first_ordinal'] = ordinal
        blocks[i]['rows_offset'] = at[(S, a)] + (r0 - a) * S
        blocks[i]['num_rows'] = r1 - r0
        row_base[i] = r0
        ordinal += (r1 - r0) * ndiv
    layout = FlatPlanSpace(ordinal, blocks, space.batches, np.zeros(0, dtype=np.uint8))
    layout.rows_total_bytes = off
    return ListedWindow(base, layout, row_base, ranges, rec_bound, listing)


def whole_space_ranges(space: FlatPlanSpace) -> np.ndarray:
    """native.RANGE_DTYPE: every row of every stage count the blocks of ``space`` use, in stage-count order (the layout
    of a one-window listed space)."""
    stages = sorted({int(S) for S in space.blocks['num_stage']})
    rows = {int(b['num_stage']): int(b['num_rows']) for b in space.blocks}
    return np.array([(S, 0, 0, rows[S]) for S in stages], dtype=native.RANGE_DTYPE)
