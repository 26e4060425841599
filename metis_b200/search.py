"""Device-side plan search: the GPU replacement of the loops in cost_het_cluster.py:21-50
and cost_homo_cluster.py:21-37 of the reference.

PyTorch is used only for device buffers, streams and (multi-GPU) torch.distributed; all
search arithmetic runs in libmetis_b200.so (hand-written sm_90a CUDA) behind the C ABI of
include/metis_b200.h.  There is no CPU path: without CUDA these functions raise.
"""
from __future__ import annotations

import copy
import ctypes as C
import math
import time
import weakref
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import flatten, native


def _require_cuda(device) -> torch.device:
    if not torch.cuda.is_available():
        raise native.MetisNativeError('CUDA device required: metis_b200 has no CPU fallback')
    return torch.device(device if device is not None else f'cuda:{torch.cuda.current_device()}')


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


def upload(a: np.ndarray, device) -> torch.Tensor:
    """A copy of the bytes of ``a`` on ``device`` (flat uint8)."""
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(device)


def _ptr(t: torch.Tensor, offset: int = 0) -> C.c_void_p:
    """The device address ``offset`` bytes into ``t``."""
    return C.c_void_p(t.data_ptr() + offset)


def bind_problem(problem: flatten.FlatProblem, device, space: Optional[flatten.FlatPlanSpace] = None,
                 rows: Optional[torch.Tensor] = None, workspace: bool = True):
    """``problem``'s tables (and ``space``'s blocks and batches, with ``rows``, its device-group rows on ``device``)
    uploaded to ``device``: (lib, problem struct, space struct or None, a workspace for the replay kernels (None
    without ``workspace``), the tensors the structs point into)."""
    lib = native.load_library()
    with torch.cuda.device(device):
        tens = {k: upload(v, device) for k, v in problem.arrays.items()}
        if space is not None:
            tens.update(blocks=upload(space.blocks, device), batches=upload(space.batches, device), rows=rows)
        p = problem.as_struct(lambda n: tens[n].data_ptr())
        sp = space.as_struct(lambda n: tens[n].data_ptr()) if space is not None else None
        ws = torch.empty(int(lib.metis_het_workspace_bytes(C.byref(p), 0, 1)), dtype=torch.uint8, device=device) \
            if workspace else None
    return lib, p, sp, ws, tens


def device_sort(buf: torch.Tensor, n: int, mode: int, stream: torch.cuda.Stream, want_perm: bool = False,
                workspace: Optional[torch.Tensor] = None) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
    """metis_sort_records on the first n rows of ``buf`` (device, in place, asynchronous on ``stream``): (the
    permutation as int32 [n] (a view of the uint32 indices) when asked, else None; the workspace, ``workspace`` when it
    is large enough, so that a caller can keep it for the next sort)."""
    lib = native.load_library()
    need = int(lib.metis_sort_workspace_bytes(C.c_int64(n)))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need + need // 8, dtype=torch.uint8, device=buf.device)
    perm = torch.empty(max(n, 1), dtype=torch.int32, device=buf.device) if want_perm else None
    rc = lib.metis_sort_records(C.c_void_p(buf.data_ptr()), C.c_int64(n), C.c_int32(mode),
                                C.c_void_p(perm.data_ptr() if perm is not None else 0),
                                C.c_void_p(workspace.data_ptr()), C.c_int64(workspace.numel()),
                                C.c_void_p(stream.cuda_stream))
    native.check(rc, 'metis_sort_records')
    return (perm[:n] if perm is not None else None), workspace


def sorted_positions(rows: np.ndarray, mode: int, device) -> np.ndarray:
    """Positions of the 16-byte ``rows`` (MetisRecord or MetisMiss) in metis_sort_records(``mode``) order (int64)."""
    with torch.cuda.device(device):
        perm, _ws = device_sort(upload(rows, device), len(rows), mode, torch.cuda.current_stream(device), True)
        return perm.cpu().numpy().view(np.uint32).astype(np.int64)


_PROBLEM_ARRAYS = ('key_index', 'layer_compute', 'layer_memory', 'exec_full', 'fb_sync', 'norm_lc', 'type_memory',
                   'type_bw_first', 'type_bw_min', 'ns_run_type', 'ns_run_end', 'ns_q10_end')
# 'rows' is last: spaces whose rows the GPU writes itself (flatten.build_plan_space(device_rows=True)) upload
# everything before it - the composition list instead of the rows - and fill it with metis_generate_rows
_ARENA_ORDER = _PROBLEM_ARRAYS + ('blocks', 'batches', 'comp_recs', 'comp_pool', 'rows')
_EMPTY = np.zeros(0, dtype=np.uint8)


class DeviceProblem:
    """A flattened problem + candidate space resident in HBM (one upload, many searches).

    All tables live in ONE pinned host arena and ONE device arena at the same offsets, so an upload is a single
    host -> device copy; ``reload`` puts another problem / space of compatible size into the same buffers."""

    def __init__(self, problem: flatten.FlatProblem, space: flatten.FlatPlanSpace, device=None,
                 pinned: bool = True, rows_capacity: int = 0, reserve: Sequence = ()):
        """``reserve``: the windows of a windowed search (flatten.PlanWindow / ListedWindow, ``arena_sizes()``) the
        arena is sized for up front, so that reloading any of them reuses the buffers."""
        self.device = _require_cuda(device)
        self.lib = native.load_library()
        self.pinned = pinned
        self._host = self._dev = None
        self._off: Dict[str, Tuple[int, int]] = {}           # name -> (offset, capacity)
        self._used: Dict[str, int] = {}
        self._reserve: Dict[str, int] = {}
        self._uploaded = None       # event after the last upload's copy: until then the copy may still read _host
        for w in reserve:
            for name, n in w.arena_sizes().items():
                self._reserve[name] = max(self._reserve.get(name, 0), n)
        self._allocate(self._arrays(problem, space), space, rows_capacity)
        self.reload(problem, space)
        self.upload()

    @staticmethod
    def _arrays(problem: flatten.FlatProblem, space: flatten.FlatPlanSpace) -> Dict[str, np.ndarray]:
        arrays = {k: problem.arrays[k] for k in _PROBLEM_ARRAYS}
        arrays.update(blocks=space.blocks.view(np.uint8).reshape(-1), batches=space.batches, rows=space.rows,
                      comp_recs=space.comp_recs.view(np.uint8).reshape(-1) if space.comp_recs is not None else _EMPTY,
                      comp_pool=space.comp_pool if space.comp_pool is not None else _EMPTY)
        return {k: np.ascontiguousarray(v).view(np.uint8).reshape(-1) for k, v in arrays.items()}

    @staticmethod
    def _need(flat: Dict[str, np.ndarray], space: flatten.FlatPlanSpace, name: str) -> int:
        if name == 'rows' and space.comp_recs is not None:
            return int(space.rows_total_bytes)               # written by the GPU, never staged on the host
        return int(flat[name].size)

    def _allocate(self, flat: Dict[str, np.ndarray], space: flatten.FlatPlanSpace, rows_capacity: int) -> None:
        off = host_bytes = 0
        self._off = {}
        for name in _ARENA_ORDER:
            need = max(self._need(flat, space, name), self._reserve.get(name, 0), 16)
            cap = _align(need + need // 4 if name in ('rows', 'blocks', 'comp_recs', 'comp_pool') else need)
            if name == 'rows':
                cap = max(cap, _align(rows_capacity))
                host_bytes = off + (16 if space.comp_recs is not None and not rows_capacity else cap)
            self._off[name] = (off, cap)
            off += cap
        host = torch.zeros(host_bytes, dtype=torch.uint8)
        self._host = host.pin_memory() if self.pinned else host
        with torch.cuda.device(self.device):
            self._dev = torch.zeros(off, dtype=torch.uint8, device=self.device)

    def fits(self, problem: flatten.FlatProblem, space: flatten.FlatPlanSpace) -> bool:
        flat = self._arrays(problem, space)
        return (all(self._need(flat, space, n) <= self._off[n][1] for n in _ARENA_ORDER)
                and self._off['rows'][0] + flat['rows'].size <= self._host.numel())

    def reload(self, problem: flatten.FlatProblem, space: flatten.FlatPlanSpace) -> None:
        """Stage another problem / space (host side only; call upload()).  Tables that already live in the staging
        arena (``build_plan_space(rows_out=staging('rows'))``) are not copied again."""
        flat = self._arrays(problem, space)
        self._wait_upload()
        if not self.fits(problem, space):
            keep = {n: flat[n].copy() for n in _ARENA_ORDER}     # a view into the old arena must survive the swap
            self._allocate(keep, space, 0)
            flat = keep
        host = self._host.numpy()
        for name in _ARENA_ORDER:
            src = flat[name]
            off, _cap = self._off[name]
            dst = host[off:off + src.size]
            if src.size and not np.shares_memory(src, dst):
                dst[:] = src
            self._used[name] = int(src.size)
        self.problem, self.space = problem, space
        base = self._dev.data_ptr()
        self.p_struct = problem.as_struct(lambda n: base + self._off[n][0])
        self.s_struct = space.as_struct(lambda n: base + self._off[n][0])
        self.device_rows = space.comp_recs is not None
        self.h2d_bytes = self._off['rows'][0] + self._used['rows']          # device_rows: nothing of 'rows'

    def staging(self, name: str) -> np.ndarray:
        """The pinned host region of one table (numpy view, full capacity): fill it in place, then upload()."""
        self._wait_upload()
        off, cap = self._off[name]
        return self._host.numpy()[off:off + cap]

    def _wait_upload(self) -> None:
        """Block until the last upload's copy has read the pinned staging arena: the copy is asynchronous, so a host
        write into the arena (reload, staging) before it ran would reach the device as the next problem's tables."""
        if self._uploaded is not None:
            self._uploaded.synchronize()
            self._uploaded = None

    def restage_space(self, space: flatten.FlatPlanSpace) -> None:
        """Put a freshly enumerated space into the staging arena (same problem)."""
        self.reload(self.problem, space)

    def upload(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Host -> HBM: ONE copy of the arena's used prefix (part of the end-to-end timed region)."""
        n = self.h2d_bytes
        with torch.cuda.device(self.device), torch.cuda.stream(stream or torch.cuda.current_stream(self.device)):
            self._dev[:n].copy_(self._host[:n], non_blocking=True)
            self._uploaded = torch.cuda.Event()
            self._uploaded.record()
            if self.device_rows:                              # SURVEY.md 8(f)-1: the GPU writes the rows itself
                base = self._dev.data_ptr()
                s = torch.cuda.current_stream(self.device)
                rc = self.lib.metis_generate_rows(C.c_void_p(base + self._off['comp_recs'][0]),
                                                  C.c_int64(len(self.space.comp_recs)),
                                                  C.c_void_p(base + self._off['comp_pool'][0]),
                                                  C.c_void_p(base + self._off['rows'][0]), C.c_void_p(s.cuda_stream))
                native.check(rc, 'metis_generate_rows')

    def rows_device(self) -> torch.Tensor:
        """The row blob in HBM (uint8 view; MetisPlanBlock.rows_offset addresses it)."""
        off = self._off['rows'][0]
        n = int(self.space.rows_total_bytes) if self.device_rows else self._used['rows']
        return self._dev[off:off + n]

    def workspace_bytes(self, num_plans: int) -> int:
        n = self.lib.metis_het_workspace_bytes(C.byref(self.p_struct), num_plans, self.s_struct.max_stage)
        if n < 0:
            native.check(int(n), 'metis_het_workspace_bytes')
        return int(n)


@dataclass
class HetSearchOutput:
    """Result of one shard's search.  ``records`` (host, numpy) are in estimate_costs order; ``detail`` rows are
    aligned with them: a numpy array when the searcher copies them to the host, else only ``detail_dev``."""
    summary: Dict[str, int]
    best: Optional[Tuple[float, int, int, int, int]]      # cost, ordinal, step, num_repartition, num_stage
    records: Optional[np.ndarray]                         # native.RECORD_DTYPE sorted by (ordinal, step)
    detail: Optional[np.ndarray]                          # uint8 [n, stride] aligned with records
    d2h_bytes: int = 0
    rank_order: Optional[np.ndarray] = None               # uint32: records[rank_order] = sorted(..., key=cost), stable
    detail_dev: Optional[torch.Tensor] = None             # uint8 [n, stride] on the device
    records_dev: Optional[torch.Tensor] = None            # int64 [2n]: the sorted records on the device
    headroom: Optional[np.ndarray] = None                 # float64 [n] aligned with records (want_headroom)
    headroom_dev: Optional[torch.Tensor] = None           # the same on the device
    headroom_s: float = 0.0                               # host time spent ordering and copying the headroom
    misses: Optional[np.ndarray] = None                   # MISS_HOST_DTYPE in reference order (want_misses)
    misses_s: float = 0.0                                 # host time spent ordering and copying the misses


# Host form of the out-of-memory partition attempts of a search (native.MISS_DTYPE with a global 64-bit ordinal and the
# key split): three 64-bit words without padding, so that a padded int64 tensor carries it through the multi-rank gathers
# and the conversion below is word arithmetic.
MISS_HOST_DTYPE = np.dtype([('deficit', '<f8'), ('ordinal', '<i8'), ('call', '<u2'), ('attempt', 'u1'), ('stage', 'u1'),
                            ('num_stage', '<u4')])


def misses_to_host(raw: np.ndarray, base: int = 0) -> np.ndarray:
    """native.MISS_DTYPE rows (ordinals relative to ``base``) -> MISS_HOST_DTYPE rows, same order."""
    words = np.ascontiguousarray(raw).view(np.uint64).reshape(-1, 2)
    hi = words[:, 1]                                         # ordinal | key << 32 | stage << 48 | num_stage << 56
    out = np.empty((len(raw), 3), dtype=np.uint64)
    out[:, 0] = words[:, 0]
    out[:, 1] = (hi & np.uint64(0xFFFFFFFF)) + np.uint64(base)
    key = (hi >> np.uint64(32)) & np.uint64(0xFFFF)
    out[:, 2] = ((key >> np.uint64(2)) | ((key & np.uint64(3)) << np.uint64(16)) |
                 (((hi >> np.uint64(48)) & np.uint64(0xFF)) << np.uint64(24)) | ((hi >> np.uint64(56)) << np.uint64(32)))
    return out.view(MISS_HOST_DTYPE).reshape(-1)


def host_rows_device(words: torch.Tensor) -> torch.Tensor:
    """misses_to_host on the device, base 0: int64 [2m] MetisMiss words -> int64 [m, 3] MISS_HOST_DTYPE words."""
    w = words.view(-1, 2)
    hi = w[:, 1]
    key = (hi >> 32) & 0xFFFF
    out = torch.empty((w.shape[0], 3), dtype=torch.int64, device=words.device)
    out[:, 0] = w[:, 0]
    out[:, 1] = hi & 0xFFFFFFFF
    out[:, 2] = (key >> 2) | ((key & 3) << 16) | (((hi >> 48) & 0xFF) << 24) | (((hi >> 56) & 0xFF) << 32)
    return out


def position_order(misses: np.ndarray) -> np.ndarray:
    """The reference's order of MISS_HOST_DTYPE rows: (ordinal, call, attempt)."""
    return misses[np.lexsort((misses['attempt'], misses['call'], misses['ordinal']))]


class HetSearcher:
    """Owns the output buffers for repeated searches over one DeviceProblem."""

    def __init__(self, dp: DeviceProblem, rank: int = 0, world: int = 1, tile: int = 128,
                 want_records: bool = True, want_detail: bool = False, capacity: Optional[int] = None,
                 want_ranking: bool = False, detail_to_host: bool = True, detail_stride: Optional[int] = None,
                 want_headroom: bool = False, want_misses: bool = False):
        """``want_headroom``: the search also writes each record's memory headroom; ``want_misses``: and every
        out-of-memory partition attempt (both side outputs of metis_het_search_outputs)."""
        self.dp = dp
        self.want_misses = want_misses
        self.misses = None                                   # int64 [2 * miss_capacity]: MetisMiss rows
        self.miss_capacity = 0
        self.want_headroom = want_headroom and want_records
        self.headroom = None
        self.want_ranking = want_ranking and want_records
        self._sort_ws = None
        self.shard = native.MetisShard(rank, world, tile, 0)
        self.want_records = want_records
        self.want_detail = want_detail and want_records
        self.detail_to_host = detail_to_host
        self.detail_stride = int(detail_stride or native.DETAIL_STRIDE)
        self.capacity = 0
        self.workspace = None
        self.summary_host = torch.zeros(C.sizeof(native.MetisSearchSummary), dtype=torch.uint8).pin_memory()
        self._host_buf: Dict[str, list] = {}                 # name -> [[pinned tensor, weakref to the array handed out]]
        self.records = self.detail = None
        self._fixed_capacity = capacity
        self.rebind()

    def rebind(self) -> None:
        """(Re)size the buffers for the DeviceProblem's current space (after DeviceProblem.reload)."""
        dp = self.dp
        tile, world = self.shard.tile, self.shard.world
        rounds = -(-dp.space.num_plans // (tile * world))
        self.shard_plans = rounds * tile
        need = dp.workspace_bytes(self.shard_plans)
        if self.workspace is None or self.workspace.numel() < need:
            with torch.cuda.device(dp.device):
                self.workspace = torch.empty(need + need // 8, dtype=torch.uint8, device=dp.device)
        if self.want_records and self.records is None:
            self._alloc(self._fixed_capacity if self._fixed_capacity is not None else min(self.shard_plans + 4096, 1 << 18))

    def reserve_workspace(self, num_plans: int) -> None:
        """Size the workspace for a space of ``num_plans`` plans now, so that rebind() for a smaller one keeps it."""
        dp = self.dp
        tile, world = self.shard.tile, self.shard.world
        need = dp.workspace_bytes(-(-num_plans // (tile * world)) * tile)
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = None
            with torch.cuda.device(dp.device):
                self.workspace = torch.empty(need + need // 8, dtype=torch.uint8, device=dp.device)

    def _alloc(self, capacity: int) -> None:
        dev = self.dp.device
        self.capacity = capacity
        with torch.cuda.device(dev):
            self.records = torch.empty(capacity * 2, dtype=torch.int64, device=dev)
            self.headroom = torch.empty(capacity, dtype=torch.float64, device=dev) if self.want_headroom else None
            self.detail = (torch.empty((capacity, self.detail_stride), dtype=torch.uint8, device=dev)
                           if self.want_detail else None)

    def _alloc_misses(self, capacity: int) -> None:
        self.miss_capacity = capacity
        with torch.cuda.device(self.dp.device):
            self.misses = torch.empty(capacity * 2, dtype=torch.int64, device=self.dp.device)

    def set_outputs(self, headroom: bool, misses: bool) -> None:
        """Which side outputs the next searches write: each record's memory headroom, every out-of-memory partition
        attempt.  The buffers of an output no longer written are freed."""
        self.want_headroom = headroom and self.want_records
        if not self.want_headroom:
            self.headroom = None
        self.want_misses = misses
        if not misses:
            self.misses, self.miss_capacity = None, 0

    def release(self) -> None:
        """Free the search buffers, keeping only what replaying picks needs (metis_het_detail's workspace): what a
        windowed result holds on to while it is alive."""
        self.records = self.workspace = self.headroom = self.misses = None
        self.capacity = self.miss_capacity = 0
        with torch.cuda.device(self.dp.device):
            self.workspace = torch.empty(self.dp.workspace_bytes(0), dtype=torch.uint8, device=self.dp.device)

    def launch(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Enqueue pack + search + finalize + summary copy on ``stream`` (asynchronous)."""
        dp = self.dp
        s = stream or torch.cuda.current_stream(dp.device)
        if self.want_misses and self.misses is None:         # the count is not known before the first search
            self._alloc_misses(min(self.shard_plans + 4096, 1 << 18))
        if self.want_headroom and self.records is not None and self.headroom is None:
            with torch.cuda.device(dp.device):
                self.headroom = torch.empty(self.capacity, dtype=torch.float64, device=dp.device)
        headroom = self.headroom if self.want_headroom else None
        misses = self.misses if self.want_misses else None
        rc = dp.lib.metis_het_search_outputs(
            C.byref(dp.p_struct), C.byref(dp.s_struct), C.byref(self.shard),
            C.c_void_p(self.records.data_ptr() if self.records is not None else 0), C.c_int64(self.capacity),
            C.c_void_p(self.detail.data_ptr() if self.detail is not None else 0), C.c_int32(self.detail_stride),
            C.c_void_p(headroom.data_ptr() if headroom is not None else 0),
            C.c_void_p(misses.data_ptr() if misses is not None else 0),
            C.c_int64(self.miss_capacity if misses is not None else 0), C.c_void_p(self.workspace.data_ptr()),
            C.c_int64(self.workspace.numel()), C.c_void_p(self.summary_host.data_ptr()), C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_het_search_outputs')

    def summary(self) -> native.MetisSearchSummary:
        return native.MetisSearchSummary.from_buffer_copy(self.summary_host.numpy().tobytes())

    def _to_host(self, name: str, dev_tensor: torch.Tensor, stream: torch.cuda.Stream) -> np.ndarray:
        """Device -> pinned host memory, handed out WITHOUT another copy.

        A pinned buffer is reused only when the array handed out from it last time is gone (its weak reference is
        dead: numpy views keep their root array alive), so a result a caller still holds is never overwritten; a
        caller that keeps every result makes each call allocate a new buffer (slow, correct)."""
        n = dev_tensor.numel() * dev_tensor.element_size()
        pool = self._host_buf.setdefault(name, [])
        slot = None
        for entry in pool:
            if entry[1] is None or entry[1]() is None:
                if entry[0].numel() >= n:
                    slot = entry
                    break
        if slot is None:
            pool[:] = [e for e in pool if not (e[1] is None or e[1]() is None)]     # too small and free: drop
            slot = [torch.empty(max(n + n // 8, 1 << 16), dtype=torch.uint8).pin_memory(), None]
            pool.append(slot)
        view = slot[0][:n]
        with torch.cuda.stream(stream):
            view.copy_(dev_tensor.reshape(-1).view(torch.uint8), non_blocking=True)
        stream.synchronize()
        arr = view.numpy()
        slot[1] = weakref.ref(arr)
        return arr

    def run(self, stream: Optional[torch.cuda.Stream] = None) -> HetSearchOutput:
        """launch + synchronise + bring results to the host; grows the record buffer if needed."""
        dp = self.dp
        s = stream or torch.cuda.current_stream(dp.device)
        with torch.cuda.device(dp.device):
            self.launch(s)
            s.synchronize()
            sm = self.summary()
            grow_misses = self.want_misses and sm.reserved[3] > self.miss_capacity
            if (self.want_records and sm.num_records > self.capacity) or grow_misses:
                # C is not known before the first search of a space: size the buffers and search again
                if self.want_records and sm.num_records > self.capacity:
                    self._alloc(int(sm.num_records) + max(1024, int(sm.num_records) // 64))
                if grow_misses:
                    self._alloc_misses(int(sm.reserved[3]) + max(1024, int(sm.reserved[3]) // 64))
                self.launch(s)
                s.synchronize()
                sm = self.summary()
            out_summary = dict(num_records=int(sm.num_records), num_partition_calls=int(sm.num_partition_calls),
                               num_balancer_runs=int(sm.num_balancer_runs), num_keyerror=int(sm.num_keyerror),
                               fatal_ordinal=int(sm.fatal_ordinal), fatal_code=int(sm.fatal_code),
                               fatal_aux=int(sm.fatal_aux), num_admitted=int(sm.reserved[0]),
                               num_chained=int(sm.reserved[1]),
                               instantiation=(int(sm.reserved[2]) & 0xFFFF, int(sm.reserved[2]) >> 16 & 0xFFFF,
                                              bool(int(sm.reserved[2]) >> 32 & 1)))   # (MAXS, MAXL, ONE) that ran
            best = None
            if sm.num_records > 0:
                b = sm.best
                best = (float(b.cost), int(b.ordinal), int(b.step), int(b.num_repartition), int(b.num_stage))
            records = detail = rank_order = detail_dev = records_dev = headroom = headroom_dev = misses = None
            headroom_s = misses_s = 0.0
            if self.want_misses:                              # reference order: the record sort's position mode
                t = time.perf_counter()
                m = int(sm.reserved[3])
                out_summary['num_oom_attempts'] = m
                self.sort_records(m, native.SORT_POSITION, s, buf=self.misses)
                with torch.cuda.stream(s):
                    rows = host_rows_device(self.misses[:2 * m])
                # a copy of plain words: the pinned buffer is reused by the next search, the result keeps the rows
                misses = self._to_host('misses', rows, s).view(np.uint64).copy().view(MISS_HOST_DTYPE).reshape(-1)
                misses_s = time.perf_counter() - t
            d2h = C.sizeof(native.MetisSearchSummary)
            if self.want_records:
                n = int(sm.num_records)
                # estimate_costs order = (ordinal, step): rank_records_kernel, in place
                order = self.sort_records(n, native.SORT_POSITION, s, want_perm=self.want_detail or self.want_headroom)
                records_dev = self.records[:2 * n]
                records = self._to_host('records', records_dev, s).view(native.RECORD_DTYPE)
                d2h += n * 16
                if self.want_detail:
                    detail_dev = self.detail[:n].index_select(0, order.long())
                    if self.detail_to_host:
                        detail = self._to_host('detail', detail_dev, s).reshape(n, self.detail_stride)
                        d2h += n * self.detail_stride
                if self.want_headroom:                       # the same permutation as the detail rows
                    t = time.perf_counter()
                    headroom_dev = self.headroom[:n].index_select(0, order.long())
                    headroom = self._to_host('headroom', headroom_dev, s).view(np.float64)
                    d2h += n * 8
                    headroom_s = time.perf_counter() - t
                if self.want_ranking:
                    # sorted(estimate_costs, key=cost): stable by cost on a copy of the ordered records
                    by_cost = self.records[:2 * n].clone()
                    perm = self.sort_records(n, native.SORT_BY_COST_STABLE, s, want_perm=True, buf=by_cost)
                    rank_order = self._to_host('rank', perm, s).view(np.uint32)
                    d2h += n * 4
        return HetSearchOutput(out_summary, best, records, detail, d2h, rank_order, detail_dev, records_dev, headroom,
                               headroom_dev, headroom_s, misses, misses_s)

    def sort_records(self, n: int, mode: int, stream: torch.cuda.Stream, want_perm: bool = False, buf=None):
        """device_sort of the first n records of ``buf`` (default: the record buffer), with the sort workspace kept
        for the next sort; returns the permutation when asked."""
        perm, self._sort_ws = device_sort(self.records if buf is None else buf, n, mode, stream, want_perm,
                                          self._sort_ws)
        return perm

    def detail_for(self, picks: np.ndarray, stream: Optional[torch.cuda.Stream] = None) -> np.ndarray:
        """Strategies and partition of chosen records (metis_het_detail replay)."""
        dp = self.dp
        s = stream or torch.cuda.current_stream(dp.device)
        n = len(picks)
        with torch.cuda.device(dp.device):
            raw = upload(picks, dp.device)
            out = torch.zeros((max(n, 1), native.DETAIL_STRIDE), dtype=torch.uint8, device=dp.device)
            rc = dp.lib.metis_het_detail(C.byref(dp.p_struct), C.byref(dp.s_struct), C.c_void_p(raw.data_ptr()),
                                         C.c_int64(n), C.c_void_p(out.data_ptr()), C.c_int32(native.DETAIL_STRIDE),
                                         C.c_void_p(self.workspace.data_ptr()), C.c_int64(self.workspace.numel()),
                                         C.c_void_p(s.cuda_stream))
            native.check(rc, 'metis_het_detail')
            s.synchronize()
            return out[:n].cpu().numpy()


def raise_fatal(summary: Dict[str, int], problem: flatten.FlatProblem) -> None:
    """Re-raise what the reference would have raised at the first failing plan (quirk Q8)."""
    code = summary['fatal_code']
    if summary['fatal_ordinal'] == 2 ** 64 - 1 or code == 0:
        return
    aux = summary['fatal_aux']
    tp, bs = 1 << ((aux >> 16) & 0xFF), aux & 0xFFFF
    if code in (1, 2):
        raise KeyError(f'tp{tp}_bs{bs}')
    if code == 3:
        raise IndexError('list index out of range')
    if code == 6:
        raise ZeroDivisionError('float division by zero')
    raise RuntimeError(f'plan {summary["fatal_ordinal"]}: {native.FATAL_NAMES.get(code, code)} '
                       f'(the reference does not complete this search either)')


class Candidates:
    """Vectorised view of the costed candidates: every column of the reference's 7-tuples
    (cost_het_cluster.py:44-46) as a numpy array, the tuples themselves built on demand.

    The records (host, estimate_costs order) are split into segments: the records [first, end) of one plan space,
    whose ordinals are global ordinals less the segment's ``base``.  One search is one SearchSegment at base 0, a
    windowed search one WindowSegment per window.  A segment binds its tables on the device and gives its records'
    detail rows (dp codes[S], tp codes[S] (log2) and layer_partition[S+1]); every view below splits its request by
    segment (``_split``)."""

    def __init__(self, records: np.ndarray, detail: Optional[np.ndarray], space: Optional[flatten.FlatPlanSpace],
                 node_sequences: Sequence[Tuple], detail_dev: Optional[torch.Tensor] = None,
                 rows_dev: Optional[torch.Tensor] = None, problem: Optional[flatten.FlatProblem] = None,
                 headroom: Optional[np.ndarray] = None, misses: Optional[np.ndarray] = None,
                 segments: Optional[Sequence] = None):
        """The candidates of one search (a SearchSegment of ``space`` with the search's ``detail`` / ``detail_dev``
        rows and ``rows_dev`` device-group rows, replayed on ``problem``), or, given ``segments``, records split into
        those (a windowed search: window_candidates)."""
        self.records = records
        self.misses = misses                  # MISS_HOST_DTYPE, global ordinals, reference order; else None
        self.headroom = headroom              # float64 per record (a search with headroom), else None
        self.space = space                    # the plan space of a one-search result; None for segments
        if segments is None:
            segments = [SearchSegment(space, len(records), problem, detail, detail_dev, rows_dev)]
        self.segments = list(segments)
        self.device = self.segments[0].device     # where the search ran (None: not known)
        self.problem = self.segments[0].problem   # the tables the candidates are replayed on
        self.node_sequences = [tuple(s) for s in node_sequences]
        self.cost = records['cost']
        self.bases = np.asarray([s.base for s in self.segments], dtype=np.int64)
        self.firsts = np.asarray([s.first for s in self.segments] + [self.segments[-1].end], dtype=np.int64)

    def __len__(self) -> int:
        return len(self.records)

    @property
    def windows(self) -> list:
        """The windows of a windowed result, in ordinal order."""
        return [s.window for s in self.segments]

    def _split(self, values: np.ndarray, starts: np.ndarray):
        """(segment, positions into ``values``) of every segment holding some of ``values``: positions of records
        (``starts`` = self.firsts) or global ordinals (``starts`` = self.bases)."""
        seg = np.searchsorted(starts, values, side='right') - 1
        for s in np.unique(seg).tolist():
            yield self.segments[s], np.nonzero(seg == s)[0]

    def index_of(self, ordinal: int, step: int) -> Optional[int]:
        """Position of the candidate (global ordinal, step), or None: bisection over the (ordinal, step)-sorted records
        of the segment that holds the ordinal."""
        s = int(np.searchsorted(self.bases, ordinal, side='right')) - 1
        rel = int(ordinal) - int(self.bases[s]) if s >= 0 else -1
        if not 0 <= rel <= 0xFFFFFFFF:
            return None
        return _bisect_records(self.records, self.segments[s].first, self.segments[s].end, rel, int(step))

    def detail_rows(self, idx) -> np.ndarray:
        """dp codes[S], tp codes[S] (log2) and layer_partition[S+1] of the candidates ``idx``, uint8 [n, stride]."""
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        got = [(at, seg.detail(idx[at] - seg.first, self.records[idx[at]])) for seg, at in self._split(idx, self.firsts)]
        out = np.zeros((len(idx), max((d.shape[1] for _, d in got), default=native.DETAIL_STRIDE)), dtype=np.uint8)
        for at, d in got:
            out[at, :d.shape[1]] = d
        return out

    def tuples(self, idx) -> List[Tuple]:
        """The reference's 7-tuples of the candidates ``idx`` (any integer sequence)."""
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        out: List[Optional[Tuple]] = [None] * len(idx)
        for seg, at in self._split(idx, self.firsts):
            rec = self.records[idx[at]]
            det = seg.detail(idx[at] - seg.first, rec)
            col = plan_geometry(seg.space, rec['ordinal'])
            codes = seg.group_codes(col['row_byte'], col['num_stage'])
            nrep, cost = rec['num_repartition'].astype(np.int64), rec['cost']
            for k, i in enumerate(at.tolist()):
                S = int(col['num_stage'][k])
                d = det[k]
                groups = (1 << codes[k, :S].astype(np.int64)).tolist()
                dp = (1 << d[:S].astype(np.int64)).tolist()
                tp = (1 << d[S:2 * S].astype(np.int64)).tolist()
                part = d[2 * S:3 * S + 1].astype(np.int64).tolist()
                out[i] = (self.node_sequences[int(col['ns_idx'][k])], groups, list(zip(dp, tp)), int(col['batches'][k]),
                          part, int(nrep[k]), float(cost[k]))
        return out

    def plan_columns(self, ordinals: np.ndarray) -> Dict[str, np.ndarray]:
        """ns_idx, num_stage, batches and the log2 device-group codes (``codes``, [n, METIS_MAX_STAGES]) of the plans of
        the global ``ordinals``."""
        ordinals = np.asarray(ordinals, dtype=np.int64).reshape(-1)
        n = len(ordinals)
        out: Dict[str, np.ndarray] = {}
        for seg, at in self._split(ordinals, self.bases):
            col = plan_geometry(seg.space, ordinals[at] - seg.base)
            col['codes'] = seg.group_codes(col['row_byte'], col['num_stage'])
            for k, v in col.items():
                if k not in out:
                    out[k] = np.zeros((n, native.METIS_MAX_STAGES) if k == 'codes' else n, dtype=v.dtype)
                if k == 'codes':
                    out[k][at, :v.shape[1]] = v
                else:
                    out[k][at] = v
        return out

    def trace(self, ordinals: np.ndarray) -> List[list]:
        """verbose.decode_plan of the plans of the global ``ordinals`` (metis_het_trace)."""
        ordinals = np.asarray(ordinals, dtype=np.int64).reshape(-1)
        out: List[Optional[list]] = [None] * len(ordinals)
        for seg, at in self._split(ordinals, self.bases):
            lib, p, sp, ws, dev, _keep = seg.bind()
            got = trace_decoded(lib, p, sp, ws, dev, ordinals[at] - seg.base, int(seg.space.blocks['num_stage'].max()))
            for k, t in zip(at.tolist(), got):
                out[k] = t
        return out

    def breakdown(self, idx, per_stage: bool = True) -> Breakdown:
        """Cost terms and memory headroom of the candidates ``idx`` (metis_het_breakdown)."""
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        width = max(int(self.records['num_stage'][idx].max()), 1) if len(idx) else 1
        raw = np.zeros(len(idx), dtype=native.BREAKDOWN_DTYPE)
        stages = np.full((len(idx), native.BD_FIELDS, width), np.nan) if per_stage else None
        for seg, at in self._split(idx, self.firsts):
            lib, p, sp, ws, dev, _keep = seg.bind()
            het_breakdown(lib, p, sp, ws, self.records[idx[at]], dev, at, raw, stages)
        return Breakdown.from_raw(raw, stages)

    def recost(self, bandwidths: np.ndarray) -> 'Recost':
        """Every candidate under the bandwidth scenarios ``bandwidths`` (float64 [K, 2, num_types]: bw_first, bw_min per
        type), _RECOST_CHUNK records per launch, each with its detail rows.  timings: ``recost_s`` up to the costs on
        the host, ``regret_s`` the regret kernels and their copy."""
        t0 = time.perf_counter()
        dev = _require_cuda(self.device)
        K = len(bandwidths)
        with torch.cuda.device(dev):
            bw = torch.from_numpy(np.ascontiguousarray(bandwidths, dtype=np.float64)).to(dev)
            costs_dev = torch.empty((K, len(self.records)), dtype=torch.float64, device=dev)
            s = torch.cuda.current_stream(dev)
            for (lib, p, sp, ws, _dev, _keep), lo, hi, rec, detail in self._replay_chunks(dev):
                c = torch.empty((K, hi - lo), dtype=torch.float64, device=dev)
                native.check(lib.metis_het_recost(
                    C.byref(p), C.byref(sp), _ptr(rec), C.c_int64(hi - lo), _ptr(detail), C.c_int32(detail.shape[1]),
                    _ptr(bw), C.c_int32(K), _ptr(c), _ptr(ws), C.c_int64(ws.numel()), C.c_void_p(s.cuda_stream)),
                    'metis_het_recost')
                costs_dev[:, lo:hi] = c
            costs = costs_dev.cpu().numpy()
        t1 = time.perf_counter()
        best, regret = recost_regret(costs_dev)
        t2 = time.perf_counter()
        return Recost(self, costs, best, regret, dev, {'recost_s': t1 - t0, 'regret_s': t2 - t1})

    def recost_profiles(self, problems: Sequence[flatten.FlatProblem]) -> 'Recost':
        """Every candidate under the scenario profiles ``problems`` (each flattened under the searched cluster, model
        flags and corrections), with its device groups, strategies and partition held fixed: cost, headroom and status
        per scenario (metis_het_profile_recost), segment by segment, _RECOST_CHUNK records per launch.  The scenarios'
        tables are uploaded once.  timings: ``recost_s`` up to the arrays on the host, ``regret_s`` the usable mask,
        the regret kernels and their copy."""
        t0 = time.perf_counter()
        dev = _require_cuda(self.device)
        K, n = len(problems), len(self.records)
        with torch.cuda.device(dev):
            bound = [bind_problem(pr, dev, workspace=False) for pr in problems]
            lib = bound[0][0]
            scen = (native.MetisProblem * K)(*[b[1] for b in bound])
            need = int(lib.metis_het_profile_recost_workspace_bytes(C.c_void_p(C.addressof(scen)), C.c_int32(K)))
            native.check(min(need, 0), 'metis_het_profile_recost_workspace_bytes')
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            costs_dev = torch.empty((K, n), dtype=torch.float64, device=dev)
            head_dev = torch.empty((K, n), dtype=torch.float64, device=dev)
            status_dev = torch.empty((K, n), dtype=torch.uint8, device=dev)
            s = torch.cuda.current_stream(dev)
            for (_lib, _p, sp, _ws, _dev, _keep), lo, hi, rec, detail in self._replay_chunks(dev):
                c, h = (torch.empty((K, hi - lo), dtype=torch.float64, device=dev) for _ in range(2))
                st = torch.empty((K, hi - lo), dtype=torch.uint8, device=dev)
                native.check(lib.metis_het_profile_recost(
                    C.byref(sp), C.c_void_p(C.addressof(scen)), C.c_int32(K), _ptr(rec), C.c_int64(hi - lo),
                    _ptr(detail), C.c_int32(detail.shape[1]), _ptr(c), _ptr(h), _ptr(st), _ptr(ws),
                    C.c_int64(ws.numel()), C.c_void_p(s.cuda_stream)), 'metis_het_profile_recost')
                costs_dev[:, lo:hi], head_dev[:, lo:hi], status_dev[:, lo:hi] = c, h, st
            costs, headroom, status = costs_dev.cpu().numpy(), head_dev.cpu().numpy(), status_dev.cpu().numpy()
        t1 = time.perf_counter()
        with torch.cuda.device(dev):
            # an unusable entry at +inf: fmax would skip a NaN, and a plan that does not fit somewhere would look
            # robust.  A NaN headroom compares false, so it is unusable.
            usable = (status_dev == 0) & (head_dev >= 0)
            best, regret = recost_regret(torch.where(usable, costs_dev, math.inf))
        t2 = time.perf_counter()
        return Recost(self, costs, best, regret, dev, {'recost_s': t1 - t0, 'regret_s': t2 - t1}, headroom, status)

    def profile_noise(self, sigma: np.ndarray, type_code: Sequence[int], seed: int, samples: int,
                      within: float) -> 'ProfileNoise':
        """The profile-noise what-if of every candidate over samples 0 .. ``samples`` - 1 of the searched profile
        (noisy_profile), drawn, evaluated and reduced on the device (metis_het_profile_noise_*).  ``sigma`` [3,
        METIS_MAX_TYPES] and ``type_code`` are per device type of the searched problem.  The samples go in chunks sized
        by _NOISE_BUDGET_BYTES; each chunk is drawn and packed once, then evaluated segment by segment, _RECOST_CHUNK
        records per launch (a window replays its detail rows once per chunk), then reduced.  Only the per-sample best
        and the per-candidate counts come back.  timings: ``noise_s`` the whole call, ``chunks`` how many."""
        t0 = time.perf_counter()
        dev = _require_cuda(self.device)
        n = len(self.records)
        spec = noise_spec(sigma, type_code, seed, within)
        with torch.cuda.device(dev):
            lib, p, _sp, _ws, _keep = bind_problem(self.problem, dev, workspace=False)
            one = int(lib.metis_het_profile_noise_workspace_bytes(C.byref(p), 1))
            native.check(min(one, 0), 'metis_het_profile_noise_workspace_bytes')
            per = int(lib.metis_het_profile_noise_workspace_bytes(C.byref(p), 2)) - one
            chunk = int(max(1, min(samples, (_NOISE_BUDGET_BYTES - one + per) // (per + 9 * max(n, 1)))))
            ws = torch.empty(int(lib.metis_het_profile_noise_workspace_bytes(C.byref(p), chunk)), dtype=torch.uint8,
                             device=dev)
            cost = torch.empty((chunk, max(n, 1)), dtype=torch.float64, device=dev)
            usable = torch.empty((chunk, max(n, 1)), dtype=torch.uint8, device=dev)
            best_pos = torch.empty(samples, dtype=torch.int64, device=dev)
            best_cost = torch.empty(samples, dtype=torch.float64, device=dev)
            wins, near, count = (torch.zeros(max(n, 1), dtype=torch.int32, device=dev) for _ in range(3))
            regret = torch.full((max(n, 1),), -math.inf, dtype=torch.float64, device=dev)
            total = torch.zeros(max(n, 1), dtype=torch.float64, device=dev)
            s = torch.cuda.current_stream(dev)
            for first in range(0, samples, chunk):
                spec.first, spec.count = first, min(chunk, samples - first)
                native.check(lib.metis_het_profile_noise_draw(
                    C.byref(p), C.byref(spec), _ptr(ws), C.c_int64(ws.numel()), C.c_void_p(s.cuda_stream)),
                    'metis_het_profile_noise_draw')
                for (_lib, _p, sp, _w, _d, _k), lo, hi, rec, detail in self._replay_chunks(dev):
                    native.check(lib.metis_het_profile_noise_eval(
                        C.byref(sp), C.byref(spec), _ptr(ws), _ptr(rec), C.c_int64(hi - lo), _ptr(detail),
                        C.c_int32(detail.shape[1]), _ptr(cost, 8 * lo), _ptr(usable, lo), C.c_int64(n),
                        C.c_void_p(s.cuda_stream)), 'metis_het_profile_noise_eval')
                native.check(lib.metis_het_profile_noise_reduce(
                    C.byref(spec), _ptr(cost), _ptr(usable), C.c_int64(n), _ptr(best_pos, 8 * first),
                    _ptr(best_cost, 8 * first), _ptr(wins), _ptr(near), _ptr(count), _ptr(regret), _ptr(total),
                    C.c_void_p(s.cuda_stream)), 'metis_het_profile_noise_reduce')
            out = [t.cpu().numpy() for t in (best_pos, best_cost, wins, near, count, regret, total)]
        best_pos, best_cost, wins, near, count, regret, total = out
        wins, near, count, regret, total = (a[:n] for a in (wins, near, count, regret, total))
        with np.errstate(invalid='ignore', divide='ignore'):
            mean = np.where(count > 0, total / np.maximum(count, 1), np.nan)
        t1 = time.perf_counter()
        return ProfileNoise(self, best_pos, best_cost, wins.astype(np.int64), near.astype(np.int64),
                            count.astype(np.int64), regret, mean,
                            {'noise_s': t1 - t0, 'chunks': -(-samples // chunk), 'chunk': chunk})

    def search_scenarios(self, scenarios, kept: Optional[int], within: float) -> 'ScenarioSearch':
        """A fresh search of this result's plan space under each of ``scenarios`` (NoiseScenarios or
        ProfileScenarios), and the candidate at position ``kept`` (the searched best; None when there is none) under
        each with its device groups, strategies and partition held fixed.  Per chunk of scenarios, on one stream: the
        scenarios' tables are staged, each is searched best-only (metis_het_search, no records) into its own pinned
        summary slot, the kept candidate is evaluated under all of them (het_profile_kernel), then one synchronise;
        each scenario's best is replayed under its own tables (metis_het_detail) before the next chunk is staged.
        Chunks are sized by _SCENARIO_BUDGET_BYTES; the results do not depend on it.  Owns its buffers: the cached
        search engine of api.cost_het_cluster is not touched.  timings: ``search_s`` the whole call, ``chunks``."""
        t0 = time.perf_counter()
        seg = one_search_segment(self)
        dev = _require_cuda(self.device)
        K = scenarios.count
        size = C.sizeof(native.MetisSearchSummary)
        with torch.cuda.device(dev):
            lib, p, sp, _ws, _dev, _keep = seg.bind()
            stride = 3 * int(sp.max_stage) + 1
            shard = native.MetisShard(0, 1, 128, 0)
            slots = -(-int(sp.num_plans) // 128) * 128
            chunk = scenarios.reserve(lib, p, dev)
            sws = torch.empty(scenarios.search_bytes(lib, p, slots, int(sp.max_stage)), dtype=torch.uint8, device=dev)
            summaries = torch.zeros(K * size, dtype=torch.uint8).pin_memory()
            picks_host = torch.zeros(K * 16, dtype=torch.uint8).pin_memory()
            picks = torch.zeros(K * 16, dtype=torch.uint8, device=dev)
            detail = torch.zeros((K, stride), dtype=torch.uint8, device=dev)
            kept_cost = torch.full((K,), math.nan, dtype=torch.float64, device=dev)
            kept_usable = torch.zeros(K, dtype=torch.uint8, device=dev)
            if kept is not None:
                rec = self.records_device()[16 * kept:16 * (kept + 1)]
                det = seg.detail_device(kept, kept + 1, self.records[kept:kept + 1], dev)
            s = torch.cuda.current_stream(dev)
            found = np.zeros(K, dtype=bool)
            for first in range(0, K, chunk):
                n = min(chunk, K - first)
                probs = scenarios.stage(lib, p, first, n, s)
                for k, pr in enumerate(probs):
                    if pr is None:
                        continue
                    native.check(lib.metis_het_search(
                        C.byref(pr), C.byref(sp), C.byref(shard), None, C.c_int64(0), None, C.c_int32(0), _ptr(sws),
                        C.c_int64(sws.numel()), C.c_void_p(summaries.data_ptr() + size * (first + k)),
                        C.c_void_p(s.cuda_stream)), 'metis_het_search')
                if kept is not None:
                    scenarios.eval_kept(lib, sp, first, n, rec, det, kept_cost, kept_usable, s)
                s.synchronize()
                for k in range(n):
                    sm = native.MetisSearchSummary.from_buffer_copy(
                        summaries.numpy()[size * (first + k):size * (first + k + 1)].tobytes())
                    if sm.num_records == 0 or (sm.fatal_ordinal != _NO_FATAL and sm.fatal_code != 0):
                        continue
                    found[first + k] = True
                    at = 16 * (first + k)
                    picks_host.numpy()[at:at + 16] = np.frombuffer(bytes(sm.best), dtype=np.uint8)
                    with torch.cuda.stream(s):
                        picks[at:at + 16].copy_(picks_host[at:at + 16], non_blocking=True)
                    native.check(lib.metis_het_detail(
                        C.byref(probs[k]), C.byref(sp), _ptr(picks, at), C.c_int64(1), _ptr(detail, stride * (first + k)),
                        C.c_int32(stride), _ptr(sws), C.c_int64(sws.numel()), C.c_void_p(s.cuda_stream)),
                        'metis_het_detail')
            out = [t.cpu().numpy() for t in (detail, kept_cost, kept_usable, scenarios.preset())]
        detail, kept_cost, kept_usable, preset = out
        raw = summaries.numpy().copy()
        sums = [native.MetisSearchSummary.from_buffer_copy(raw[size * j:size * (j + 1)].tobytes()) for j in range(K)]
        status = np.array([int(sm.fatal_code) if sm.fatal_ordinal != _NO_FATAL else 0 for sm in sums], dtype=np.int64)
        status = np.where(preset != 0, preset, status)
        found &= status == 0
        count = np.array([int(sm.num_records) for sm in sums], dtype=np.int64)
        best = np.zeros(K, dtype=native.RECORD_DTYPE)
        best.view(np.uint8).reshape(K, 16)[:] = picks_host.numpy().reshape(K, 16)
        winners = Candidates(best[found], detail[found], seg.space, self.node_sequences, rows_dev=seg._rows_dev)
        return ScenarioSearch(self, kept, status, np.where(status == 0, count, 0), best, found, winners, kept_cost,
                              kept_usable.astype(bool), within,
                              {'search_s': time.perf_counter() - t0, 'chunks': -(-K // chunk), 'chunk': chunk})

    def records_device(self) -> torch.Tensor:
        """The records (estimate_costs order) on the device, uploaded on first use: what the replays and the group
        passes read."""
        if getattr(self, '_records_dev', None) is None:
            self._records_dev = upload(self.records, _require_cuda(self.device))
        return self._records_dev

    def _replay_chunks(self, dev, with_detail: bool = True):
        """Every non-empty segment's records, _RECOST_CHUNK at a time: (the segment's bound structs (``bind()``), lo,
        hi, the device bytes of the records [lo, hi) (records_device), their device detail rows, or None without
        ``with_detail``).  An empty segment is skipped: a window is not reloaded for it."""
        recs, width = self.records_device(), self.records.itemsize
        for seg in self.segments:
            if seg.first == seg.end:
                continue
            bound = seg.bind()
            for lo in range(seg.first, seg.end, _RECOST_CHUNK):
                hi = min(seg.end, lo + _RECOST_CHUNK)
                detail = seg.detail_device(lo - seg.first, hi - seg.first, self.records[lo:hi], dev) \
                    if with_detail else None
                yield bound, lo, hi, recs[width * lo:width * hi], detail

    def query(self, flt: native.MetisPlanFilter, reads_tp: bool, headroom: Optional[torch.Tensor] = None,
              min_headroom: float = 0.0, groups: bool = False) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """The filter ``flt`` on every candidate (metis_query_mark), segment by segment, _RECOST_CHUNK records per
        launch: (mask, uint8 [N] on the device; group, int32 [N] (uint32 bits), when ``groups``).  The detail rows are
        read only when ``reads_tp`` (a window replays them then); ``headroom`` (device, aligned with the records) ANDs
        in headroom >= min_headroom.  Nothing comes to the host."""
        dev = _require_cuda(self.device)
        n = len(self.records)
        with torch.cuda.device(dev):
            mask = torch.zeros(max(n, 1), dtype=torch.uint8, device=dev)
            group = torch.empty(max(n, 1), dtype=torch.int32, device=dev) if groups else None
            s = torch.cuda.current_stream(dev)
            for (lib, p, sp, _ws, _dev, _keep), lo, hi, rec, detail in self._replay_chunks(dev, reads_tp):
                rc = lib.metis_query_mark(
                    C.byref(p), C.byref(sp), C.byref(flt), _ptr(rec), C.c_int64(hi - lo),
                    C.c_void_p(detail.data_ptr() if detail is not None else 0),
                    C.c_int32(detail.shape[1] if detail is not None else 0),
                    C.c_void_p(headroom.data_ptr() + 8 * lo if headroom is not None else 0), C.c_double(min_headroom),
                    _ptr(mask, lo), C.c_void_p(group.data_ptr() + 4 * lo if groups else 0), C.c_void_p(s.cuda_stream))
                native.check(rc, 'metis_query_mark')
        return mask, group


def mask_select(mask: torch.Tensor, n: int, order: Optional[torch.Tensor], k: int) -> Tuple[np.ndarray, int]:
    """metis_mask_select: (the first ``k`` entries i whose mask[order[i]] (mask[i] without ``order``) is set, as
    order[i] (i), int64 on the host; how many are set in all)."""
    lib = native.load_library()
    dev = mask.device
    k = max(0, min(int(k), n))
    with torch.cuda.device(dev):
        ws = torch.empty(int(lib.metis_headroom_workspace_bytes(C.c_int64(n))), dtype=torch.uint8, device=dev)
        out = torch.empty(max(k, 1), dtype=torch.int32, device=dev)
        count = torch.zeros(1, dtype=torch.int64).pin_memory()
        s = torch.cuda.current_stream(dev)
        rc = lib.metis_mask_select(C.c_void_p(mask.data_ptr()), C.c_void_p(order.data_ptr() if order is not None else 0),
                                   C.c_int64(n), C.c_int64(k), C.c_void_p(out.data_ptr()), C.c_void_p(count.data_ptr()),
                                   C.c_void_p(ws.data_ptr()), C.c_int64(ws.numel()), C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_mask_select')
        s.synchronize()
        total = int(count[0])
        return out[:min(k, total)].cpu().numpy().view(np.uint32).astype(np.int64), total


def group_best(records: torch.Tensor, group: torch.Tensor, n: int, num_groups: int
               ) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """metis_query_groups, then the groups with members compacted on the device (metis_mask_select): (group ids,
    counts, lowest costs, first positions of that cost), host arrays, by ascending group id."""
    lib = native.load_library()
    dev = records.device
    with torch.cuda.device(dev):
        count = torch.empty(num_groups, dtype=torch.int64, device=dev)
        cost = torch.empty(num_groups, dtype=torch.float64, device=dev)
        first = torch.empty(num_groups, dtype=torch.int64, device=dev)
        present = torch.empty(num_groups, dtype=torch.uint8, device=dev)
        s = torch.cuda.current_stream(dev)
        rc = lib.metis_query_groups(C.c_void_p(records.data_ptr()), C.c_void_p(group.data_ptr()), C.c_int64(n),
                                    C.c_int64(num_groups), C.c_void_p(count.data_ptr()), C.c_void_p(cost.data_ptr()),
                                    C.c_void_p(first.data_ptr()), C.c_void_p(present.data_ptr()), C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_query_groups')
        ids, _m = mask_select(present, num_groups, None, num_groups)
        at = torch.from_numpy(ids).to(dev)
        return (ids, count.index_select(0, at).cpu().numpy(), cost.index_select(0, at).cpu().numpy(),
                first.index_select(0, at).cpu().numpy())


# ---------------------------------------------------------------------------------------------
# plan queries: filters on the candidates and the best candidate per key (metis_query.cu)
# ---------------------------------------------------------------------------------------------
QUERY_KEYS = native.QUERY_KEYS
_NO_LIMIT = 255
_MAX_GROUPS = 1 << 24


def _is_int(v) -> bool:
    return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))


def _tp_code(field: str, t) -> int:
    if not _is_int(t) or t < 1 or t & (t - 1):
        raise ValueError(f'{field} must be a positive power of two, not {t!r}')
    return min(int(t).bit_length() - 1, _NO_LIMIT - 1)


def _clamp(v: Optional[int], default: int) -> int:
    return default if v is None else max(-1, min(int(v), 1 << 30))


def _names(seq) -> Tuple[str, ...]:
    return tuple(flatten._type_name(x) for x in seq)


@dataclass(frozen=True)
class PlanFilter:
    """Conditions on one of the reference's candidates, the 7-tuple (node_sequence, device_groups, strategies, batches,
    layer_partition, num_repartition, cost); a field left at None (False) sets no condition.  A filter selects among
    the candidates a search found: it is not a search that forbids strategies.  The strategy chain ran unconstrained,
    so a search constrained the same way could find plans that are not in the list.

    ``admits(t, placement)`` is the definition; the GPU (metis_query_mark) computes the same on every candidate."""
    min_stages: Optional[int] = None              # min_stages <= len(device_groups)
    max_stages: Optional[int] = None              # len(device_groups) <= max_stages
    node_sequences: Optional[Sequence[Sequence]] = None   # node_sequence is one of these (by device-type name)
    batches: Optional[Sequence[int]] = None       # batches is one of these
    max_tp: Optional[int] = None                  # every stage's tp <= max_tp
    max_tp_by_type: Optional[Dict[str, int]] = None   # every stage that holds a device of type d has tp <= [d]
    uniform_tp: bool = False                      # every stage has the same tp
    max_repartition: Optional[int] = None         # num_repartition <= max_repartition

    @property
    def reads_strategies(self) -> bool:
        """Whether the conditions read the strategies (then a query reads the detail rows)."""
        return self.max_tp is not None or bool(self.max_tp_by_type) or bool(self.uniform_tp)

    def admits(self, t: Tuple, placement=None) -> bool:
        """Does candidate ``t`` pass?  ``placement``: the reference's rank_device_map of t's node sequence (rank ->
        device type name, model/device_group.py:22-32), needed with ``max_tp_by_type``: stage s holds the ranks
        [sum(groups[:s]), sum(groups[:s+1]))."""
        ns, groups, strategies, batches, _part, nrep, _cost = t
        S = len(groups)
        if self.min_stages is not None and S < self.min_stages:
            return False
        if self.max_stages is not None and S > self.max_stages:
            return False
        if self.node_sequences is not None and _names(ns) not in {_names(q) for q in self.node_sequences}:
            return False
        if self.batches is not None and batches not in set(self.batches):
            return False
        if self.max_repartition is not None and nrep > self.max_repartition:
            return False
        tps = [tp for _dp, tp in strategies]
        if self.max_tp is not None and any(tp > self.max_tp for tp in tps):
            return False
        if self.uniform_tp and len(set(tps)) > 1:
            return False
        if self.max_tp_by_type:
            lo = 0
            for g, tp in zip(groups, tps):
                for r in range(lo, lo + g):
                    limit = self.max_tp_by_type.get(placement[r])
                    if limit is not None and tp > limit:
                        return False
                lo += g
        return True

    def check(self, type_names: Sequence[str]) -> None:
        """ValueError naming the field when a field is not valid for a cluster of the device types ``type_names``."""
        for field in ('min_stages', 'max_stages', 'max_repartition'):
            v = getattr(self, field)
            if v is not None and not _is_int(v):
                raise ValueError(f'{field} must be an int, not {v!r}')
        if self.min_stages is not None and self.max_stages is not None and self.min_stages > self.max_stages:
            raise ValueError(f'min_stages ({self.min_stages}) > max_stages ({self.max_stages})')
        if self.max_tp is not None:
            _tp_code('max_tp', self.max_tp)
        for name, t in (self.max_tp_by_type or {}).items():
            if name not in type_names:
                raise ValueError(f'max_tp_by_type: unknown device type {name!r} (the cluster has {list(type_names)})')
            _tp_code(f'max_tp_by_type[{name!r}]', t)
        for q in self.node_sequences if self.node_sequences is not None else ():
            if isinstance(q, str) or sorted(_names(q)) != sorted(type_names):
                raise ValueError(f'node_sequences: {q!r} is not a permutation of the cluster device types '
                                 f'{list(type_names)}')
        for b in self.batches if self.batches is not None else ():
            if not _is_int(b):
                raise ValueError(f'batches must hold ints, not {b!r}')

    def to_struct(self, type_names: Sequence[str], node_sequences: Sequence[Tuple], batches: np.ndarray
                  ) -> native.MetisPlanFilter:
        """The MetisPlanFilter of this filter for candidates of ``node_sequences`` and the divisors ``batches``."""
        self.check(type_names)
        f = native.MetisPlanFilter()
        # stage counts and num_repartition are small: clamping keeps every bound's meaning inside int32
        f.min_stages = _clamp(self.min_stages, 0)
        f.max_stages = _clamp(self.max_stages, 1 << 30)
        f.max_repartition = _clamp(self.max_repartition, 1 << 30)
        f.max_tp_code = _tp_code('max_tp', self.max_tp) if self.max_tp is not None else _NO_LIMIT
        f.uniform_tp = int(bool(self.uniform_tp))
        for k in range(native.METIS_MAX_TYPES):
            f.type_tp_code[k] = _NO_LIMIT
        for name, t in (self.max_tp_by_type or {}).items():
            f.type_tp_code[list(type_names).index(name)] = _tp_code('max_tp_by_type', t)
        f.flags = (native.QUERY_NEEDS_TP if self.reads_strategies else 0) | \
            (native.QUERY_BY_TYPE if self.max_tp_by_type else 0)
        want = {_names(q) for q in self.node_sequences} if self.node_sequences is not None else None
        for i, q in enumerate(node_sequences):
            if want is None or _names(q) in want:
                f.ns_mask[i >> 5] |= 1 << (i & 31)
        want_b = {int(b) for b in self.batches} if self.batches is not None else None
        if len(batches) > 256:
            raise NotImplementedError(f'{len(batches)} divisors of gbs: a filter addresses 256')
        for i, b in enumerate(batches.tolist()):
            if want_b is None or int(b) in want_b:
                f.div_mask[i >> 5] |= 1 << (i & 31)
        return f


def query_key(t: Tuple, keys: Sequence[str]) -> Tuple:
    """The values of ``keys`` (of QUERY_KEYS) of candidate ``t``; 'max_tp' is the largest tp of any stage."""
    val = {'node_sequence': lambda: t[0], 'num_stage': lambda: len(t[1]), 'batches': lambda: t[3],
           'max_tp': lambda: max(tp for _dp, tp in t[2]), 'num_repartition': lambda: t[5]}
    return tuple(val[k]() for k in keys)


def check_keys(keys) -> Tuple[str, ...]:
    if isinstance(keys, str):
        keys = (keys,)
    keys = tuple(keys)
    if not keys:
        raise ValueError('keys: at least one key')
    for k in keys:
        if k not in QUERY_KEYS:
            raise ValueError(f'keys: unknown key {k!r} (choose from {QUERY_KEYS})')
    if len(set(keys)) != len(keys):
        raise ValueError(f'keys: {keys} repeats a key')
    return keys


def rank_device_map(problem: flatten.FlatProblem, ns_idx: int) -> List[str]:
    """The device type name of every rank under node sequence ``ns_idx`` (the reference's rank_device_map,
    model/device_group.py:22-32), from the problem's ns_run_type / ns_run_end."""
    a = problem.arrays
    out: List[str] = []
    for typ, end in zip(a['ns_run_type'][ns_idx].tolist(), a['ns_run_end'][ns_idx].tolist()):
        out += [problem.type_names[typ]] * (end - len(out))
    return out


class Groups:
    """The best candidate of every key value (HetSearchResult.best_by): for each value of ``keys`` that some admitted
    candidate has, in ascending key order (node sequences by their type names), ``values[g]`` (the key values),
    ``count[g]`` (admitted candidates with them), ``position[g]`` (estimate_costs position of the first of them in
    sorted(result, key=cost), i.e. lowest cost, then lowest position) and ``cost[g]``."""

    def __init__(self, candidates, keys: Tuple[str, ...], values: List[Tuple], count: np.ndarray, position: np.ndarray,
                 cost: np.ndarray):
        self.candidates = candidates
        self.keys = keys
        self.values = values
        self.count = count
        self.position = position
        self.cost = cost

    def __len__(self) -> int:
        return len(self.values)

    def tuples(self) -> List[Tuple]:
        """The reference's 7-tuple of each group's best candidate."""
        return self.candidates.tuples(self.position)


_BULK = 4096           # rows a one-search result gathers on the device per request; more are fetched whole, once


def group_codes(rows, row_byte: np.ndarray, stages: np.ndarray) -> np.ndarray:
    """log2(device count) of every stage of the device-group rows at ``row_byte`` in the row blob ``rows`` (numpy, or a
    device tensor: gathered there), uint8 [n, max stages] (columns past a row's stage count are junk)."""
    at = row_byte[:, None] + np.arange(int(stages.max()), dtype=np.int64)[None, :]
    if isinstance(rows, np.ndarray):
        return rows[np.minimum(at, len(rows) - 1)]
    return rows[torch.from_numpy(np.minimum(at, rows.numel() - 1)).to(rows.device)].cpu().numpy()


class SearchSegment:
    """The ``end`` records of one search (base 0) with the detail rows and device-group rows the search kept: host
    arrays, or device tensors (``detail_dev``, ``rows_dev``) gathered per request (a ranked slice costs one small
    gather + copy) or fetched whole the first time a request needs more than _BULK rows.  Its tables are bound from
    this object's own copies, so a later search cannot change what is replayed."""

    base = first = 0

    def __init__(self, space: flatten.FlatPlanSpace, end: int, problem: Optional[flatten.FlatProblem] = None,
                 detail: Optional[np.ndarray] = None, detail_dev: Optional[torch.Tensor] = None,
                 rows_dev: Optional[torch.Tensor] = None):
        self.space = space
        self.end = end
        self.problem = problem
        self.device = rows_dev.device if rows_dev is not None else None
        self._detail = detail
        self._detail_dev = detail_dev
        # device-group rows: the blob the GPU wrote (``rows_dev``, SURVEY.md 8(f)-1) or the host enumerator's
        self._rows_dev = rows_dev
        self._rows = None if rows_dev is not None else space.host_rows()

    def bind(self):
        """(lib, problem struct, space struct, workspace, device, the tensors the structs point into)."""
        if self.problem is None:
            raise ValueError('these candidates were built without their problem tables: no replay')
        dev = self.device if self.device is not None else _require_cuda(None)
        rows = self._rows_dev if self._rows_dev is not None else torch.from_numpy(self._rows).to(dev)
        lib, p, sp, ws, tens = bind_problem(self.problem, dev, self.space, rows)
        return lib, p, sp, ws, dev, tens

    def detail(self, pos: np.ndarray, rec: np.ndarray) -> np.ndarray:
        """Detail rows of the records at ``pos`` (segment positions; ``rec``: those records) on the host."""
        if self._detail is None:
            if self._detail_dev is None:
                raise ValueError('the search was run without detail rows')
            if len(pos) > _BULK:
                self._detail, self._detail_dev = self._detail_dev.cpu().numpy(), None
            else:
                sel = torch.from_numpy(np.ascontiguousarray(pos, dtype=np.int64)).to(self._detail_dev.device)
                return self._detail_dev.index_select(0, sel).cpu().numpy()
        return self._detail[pos]

    def detail_device(self, lo: int, hi: int, rec: np.ndarray, device) -> torch.Tensor:
        """Detail rows of the records [lo, hi) of the segment on ``device``."""
        if self._detail_dev is not None:
            return self._detail_dev[lo:hi]
        return torch.from_numpy(self.detail(np.arange(lo, hi), rec)).to(device)

    def group_codes(self, row_byte: np.ndarray, stages: np.ndarray) -> np.ndarray:
        if self._rows is None and len(row_byte) > _BULK:
            self._rows, self._rows_dev = self._rows_dev.cpu().numpy(), None
        return group_codes(self._rows if self._rows is not None else self._rows_dev, row_byte, stages)


class WindowSegment:
    """The records [first, end) of one window of a windowed search: only the 16 B records are kept.  Device groups,
    strategies and partitions are rebuilt per request in the search's DeviceProblem / HetSearcher (the arena, sized
    for the largest window's rows, and metis_het_detail's small workspace stay allocated while the result is alive):
    the window is reloaded whenever the arena holds something else, its rows regenerated on the device (row kernel)
    and its picks replayed by metis_het_detail.  The blob is never fetched: only the rows asked for are gathered."""

    def __init__(self, window, first: int, end: int, problem: flatten.FlatProblem, searcher: 'HetSearcher'):
        self.window = window
        self.space = window.space
        self.base, self.first, self.end = int(window.base), int(first), int(end)
        self.problem = problem
        self.searcher = searcher
        self.device = searcher.dp.device

    def bind(self):
        dp = self.searcher.dp
        if dp.space is not self.space or dp.problem is not self.problem:
            dp.reload(self.problem, self.space)               # metis_het_detail needs no more workspace than it has
            dp.upload()
        return dp.lib, dp.p_struct, dp.s_struct, self.searcher.workspace, dp.device, None

    def detail(self, pos: np.ndarray, rec: np.ndarray) -> np.ndarray:
        self.bind()
        return self.searcher.detail_for(rec)

    def detail_device(self, lo: int, hi: int, rec: np.ndarray, device) -> torch.Tensor:
        return torch.from_numpy(self.detail(None, rec)).to(device)

    def group_codes(self, row_byte: np.ndarray, stages: np.ndarray) -> np.ndarray:
        self.bind()
        return group_codes(self.searcher.dp.rows_device(), row_byte, stages)


def plan_geometry(space: flatten.FlatPlanSpace, ordinals: np.ndarray) -> Dict[str, np.ndarray]:
    """row (dg_idx), batches, ns_idx, num_stage and the byte offset of the device-group row of the plans
    ``ordinals`` of ``space``."""
    blocks = space.blocks
    ordinal = np.asarray(ordinals).astype(np.int64)
    blk = (np.searchsorted(blocks['first_ordinal'], ordinal, side='right') - 1) if len(ordinal) \
        else np.zeros(0, dtype=np.int64)
    rel = ordinal - blocks['first_ordinal'][blk]
    ndiv = len(space.batches)
    row, stages = rel // ndiv, blocks['num_stage'][blk].astype(np.int64)
    return dict(row=row, batches=space.batches[rel % ndiv].astype(np.int64),
                ns_idx=blocks['ns_idx'][blk].astype(np.int64), num_stage=stages,
                row_byte=blocks['rows_offset'][blk].astype(np.int64) + row * stages)


def trace_decoded(lib, p_struct, s_struct, workspace: torch.Tensor, device, ordinals: np.ndarray,
                  max_stage: int) -> List[list]:
    """metis_het_trace of ``ordinals`` on the bound problem / space, each plan decoded (verbose.decode_plan).  A plan
    whose events overflow its buffer is traced again with four times the room."""
    from . import verbose
    ordinals = np.ascontiguousarray(ordinals, dtype=np.uint32)
    out: List[Optional[list]] = [None] * len(ordinals)
    todo = np.arange(len(ordinals))
    words = max(256, 64 * (4 * max_stage + 24))
    while len(todo):
        n = len(todo)
        with torch.cuda.device(device):
            d_ord = upload(ordinals[todo], device)
            buf = torch.zeros((max(n, 1), words), dtype=torch.int64, device=device)
            s = torch.cuda.current_stream(device)
            rc = lib.metis_het_trace(C.byref(p_struct), C.byref(s_struct), C.c_void_p(d_ord.data_ptr()), C.c_int64(n),
                                     C.c_void_p(buf.data_ptr()), C.c_int32(words), C.c_void_p(workspace.data_ptr()),
                                     C.c_int64(workspace.numel()), C.c_void_p(s.cuda_stream))
            native.check(rc, 'metis_het_trace')
            host = buf[:n].cpu().numpy().view(np.uint64)
        again = []
        for k, i in enumerate(todo.tolist()):
            if int(host[k, 0]) & 0xFF == verbose.TAG_OVERFLOW:
                again.append(i)
            else:
                out[i] = verbose.decode_plan(host[k])
        todo = np.asarray(again, dtype=np.int64)
        words *= 4
    return out


TERM_NAMES = ('execution', 'fb_sync', 'parameter_update', 'dp', 'pp', 'batch_generate')
# the per-stage fields of metis_het_breakdown, in the order of METIS_BD_*
STAGE_FIELDS = ('performance', 'stage_time', 'memory_capacity', 'memory_demand', 'memory_state', 'dp_cost',
                'update_cost', 'pp_cost')


@dataclass
class Breakdown:
    """Cost terms and memory headroom of chosen candidates (metis_het_breakdown), one row per candidate in the order
    asked for.  ``terms[:, k]`` is TERM_NAMES[k] (model/cost_estimator.py:235-242): summed left to right they give the
    candidate's cost.  The per-stage arrays ([n, largest num_stage], NaN past a candidate's stages) hold the accepted
    partition attempt's values (model/load_balancer.py:57-63); the cost fields (stage_time, dp_cost, update_cost,
    pp_cost) cover the ``costed_stages`` stages get_cost walks and are NaN after them (quirk Q1).  They are None when
    the breakdown was asked for without per-stage values."""
    terms: np.ndarray                     # float64 [n, 6]
    min_headroom: np.ndarray              # float64 [n]: min over the stages of memory_state
    min_headroom_stage: np.ndarray        # int [n]: its stage, lowest on ties
    num_stage: np.ndarray                 # int [n]: len(device_groups)
    costed_stages: np.ndarray             # int [n]: min(InterStagePlan.num_stage, len(device_groups))
    performance: Optional[np.ndarray] = None
    stage_time: Optional[np.ndarray] = None
    memory_capacity: Optional[np.ndarray] = None
    memory_demand: Optional[np.ndarray] = None
    memory_state: Optional[np.ndarray] = None
    dp_cost: Optional[np.ndarray] = None
    update_cost: Optional[np.ndarray] = None
    pp_cost: Optional[np.ndarray] = None

    def __len__(self) -> int:
        return len(self.terms)

    @classmethod
    def from_raw(cls, raw: np.ndarray, stages: Optional[np.ndarray]) -> 'Breakdown':
        """MetisBreakdown rows (+ [n, METIS_BD_FIELDS, width] per-stage values) -> Breakdown."""
        per = {} if stages is None else {f: np.ascontiguousarray(stages[:, k, :]) for k, f in enumerate(STAGE_FIELDS)}
        return cls(np.array(raw['terms']), np.array(raw['min_headroom']), raw['min_stage'].astype(np.int64),
                   raw['num_stage'].astype(np.int64), raw['costed_stages'].astype(np.int64), **per)


_BREAKDOWN_CHUNK = 1 << 16                 # picks per launch: bounds the per-stage buffers of one call


def het_breakdown(lib, p_struct, s_struct, workspace: torch.Tensor, records: np.ndarray, device, at: np.ndarray,
                  raw: np.ndarray, stages: Optional[np.ndarray]) -> None:
    """metis_het_breakdown of ``records`` (any order) on the problem / space bound in ``p_struct`` / ``s_struct``:
    the picks are sorted by (ordinal, step), so that each plan is replayed once, and the row of records[k] is written
    to raw[at[k]] (MetisBreakdown) and, unless ``stages`` is None, stages[at[k]] (per-stage values
    [METIS_BD_FIELDS, width])."""
    n = len(records)
    order = np.lexsort((records['step'], records['ordinal']))
    picks = np.ascontiguousarray(records[order])
    dest = at[order]
    per_stage = stages is not None
    width = stages.shape[2] if per_stage else 1
    with torch.cuda.device(device):
        s = torch.cuda.current_stream(device)
        for lo in range(0, n, _BREAKDOWN_CHUNK):
            hi = min(n, lo + _BREAKDOWN_CHUNK)
            d_picks = upload(picks[lo:hi], device)
            d_out = torch.empty((hi - lo) * raw.itemsize, dtype=torch.uint8, device=device)
            d_st = torch.empty((hi - lo) * native.BD_FIELDS * width, dtype=torch.float64, device=device) \
                if per_stage else None
            rc = lib.metis_het_breakdown(C.byref(p_struct), C.byref(s_struct), C.c_void_p(d_picks.data_ptr()),
                                         C.c_int64(hi - lo), C.c_void_p(d_out.data_ptr()),
                                         C.c_void_p(d_st.data_ptr() if per_stage else 0), C.c_int32(width),
                                         C.c_void_p(workspace.data_ptr()), C.c_int64(workspace.numel()),
                                         C.c_void_p(s.cuda_stream))
            native.check(rc, 'metis_het_breakdown')
            raw[dest[lo:hi]] = d_out.cpu().numpy().view(native.BREAKDOWN_DTYPE)
            if per_stage:
                stages[dest[lo:hi]] = d_st.cpu().numpy().reshape(hi - lo, native.BD_FIELDS, width)


_RECOST_CHUNK = 1 << 20                   # records per replay launch: bounds a window's replayed detail rows


def recost_regret(costs: torch.Tensor) -> Tuple[np.ndarray, np.ndarray]:
    """metis_recost_regret of the device costs [K, n]: (best [K], regret [n]) on the host."""
    K, n = int(costs.shape[0]), int(costs.shape[1])
    lib = native.load_library()
    dev = costs.device
    with torch.cuda.device(dev):
        best = torch.empty(K, dtype=torch.float64, device=dev)
        regret = torch.empty(max(n, 1), dtype=torch.float64, device=dev)
        ws = torch.empty(int(lib.metis_recost_regret_workspace_bytes(C.c_int32(K), C.c_int64(n))), dtype=torch.uint8,
                         device=dev)
        s = torch.cuda.current_stream(dev)
        rc = lib.metis_recost_regret(C.c_void_p(costs.data_ptr()), C.c_int32(K), C.c_int64(n), C.c_void_p(best.data_ptr()),
                                     C.c_void_p(regret.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_int64(ws.numel()),
                                     C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_recost_regret')
        return best.cpu().numpy(), regret[:n].cpu().numpy()


def stable_cost_order(records: np.ndarray, cost: np.ndarray, device) -> np.ndarray:
    """Positions of ``records`` (in estimate_costs order) by ascending ``cost``, ties in that order: the existing
    metis_sort_records(METIS_SORT_BY_COST_STABLE) on a copy of the records whose cost field holds ``cost``."""
    if len(records) == 0:
        return np.zeros(0, dtype=np.int64)
    rows = np.array(records)
    rows['cost'] = cost
    return sorted_positions(rows, native.SORT_BY_COST_STABLE, device)


class Recost:
    """The candidates of one search re-costed under K scenarios: bandwidths (HetSearchResult.recost) or profiles
    (HetSearchResult.recost_profiles).

    ``costs[j, i]`` is candidate i's HeteroCostEstimator.get_cost under scenario j, candidates in estimate_costs order;
    for a bandwidth scenario, bit for bit what a fresh search under that scenario's cluster returns for the same
    candidate.  ``regret[i]`` is max_j (costs[j, i] - best cost of scenario j), absolute and in fp64 (costs may be
    negative on rough profiles).

    A profile what-if also has ``headroom`` and ``status`` [K, N] and the ``usable`` mask (status == 0 and headroom >=
    0).  Its rankings list only the candidates usable under the scenario, and its regret takes an unusable entry as
    +inf: best_costs[j] is the best usable cost (+inf when none is usable, and such a scenario adds nothing to the
    regret), and robust(k) lists only the candidates usable in every scenario."""

    def __init__(self, candidates, costs: np.ndarray, best_costs: np.ndarray, regret: np.ndarray, device,
                 timings: Dict[str, float], headroom: Optional[np.ndarray] = None,
                 status: Optional[np.ndarray] = None):
        self.candidates = candidates
        self.costs = costs                    # float64 [K, N]
        self.best_costs = best_costs          # float64 [K]: min over the candidates of each scenario (+inf when N == 0)
        self.regret = regret                  # float64 [N]
        self.headroom = headroom              # float64 [K, N] (profile what-if), else None
        self.status = status                  # uint8 [K, N]: cost code | memory code << 4 (profile what-if), else None
        self.usable = None if status is None else (status == 0) & (headroom >= 0)
        self.timings = timings
        self._device = device
        self._orders: Dict[int, np.ndarray] = {}
        self._robust: Optional[np.ndarray] = None

    def __len__(self) -> int:
        return self.costs.shape[0]

    def _scenario(self, j) -> int:
        j = int(j)
        K = self.costs.shape[0]
        if not -K <= j < K:
            raise IndexError(f'scenario {j} out of range: {K} scenarios')
        return j % K

    def order(self, j) -> np.ndarray:
        """Positions of the candidates in scenario j's ranking: by its cost, ties in estimate_costs order (of a profile
        what-if, only those usable under scenario j)."""
        j = self._scenario(j)
        if j not in self._orders:
            if self.usable is None:
                self._orders[j] = stable_cost_order(self.candidates.records, self.costs[j], self._device)
            else:
                ok = self.usable[j]
                pos = stable_cost_order(self.candidates.records, np.where(ok, self.costs[j], np.inf), self._device)
                self._orders[j] = pos[:int(ok.sum())]
        return self._orders[j]

    def _tuples(self, pos: np.ndarray, cost: np.ndarray) -> List[Tuple]:
        return [t[:6] + (float(c),) for t, c in zip(self.candidates.tuples(pos), cost[pos])]

    def ranked(self, j, k: Optional[int] = None) -> List[Tuple]:
        """The first ``k`` (default: all) of ``sorted(candidates, key=cost)`` under scenario j: the reference's 7-tuples
        with slot 6 holding scenario j's cost."""
        j = self._scenario(j)
        pos = self.order(j)
        if k is not None:
            pos = pos[:k]
        return self._tuples(pos, self.costs[j])

    def best(self, j) -> Optional[Tuple]:
        """The first entry of ranked(j), or None when the search returned no candidate."""
        top = self.ranked(j, 1)
        return top[0] if top else None

    def robust(self, k: int) -> Tuple[np.ndarray, np.ndarray]:
        """The ``k`` candidates of least regret: (positions in estimate_costs order, their regrets), by ascending regret,
        ties in estimate_costs order (of a profile what-if, only those usable in every scenario)."""
        if int(k) < 0:
            raise ValueError(f'k must be >= 0, not {k}')
        if self._robust is None:
            self._robust = stable_cost_order(self.candidates.records, self.regret, self._device)
            if self.usable is not None:
                self._robust = self._robust[self.usable.all(axis=0)[self._robust]]
        pos = self._robust[:int(k)]
        return pos, self.regret[pos]


# ---------------------------------------------------------------------------------------------
# profile-noise what-if: seeded samples of the searched profile (noisy_profile), evaluated and reduced on the device
# ---------------------------------------------------------------------------------------------
NOISE_FIELDS = ('layer-computes', 'memory', 'fb_sync')       # field codes 1, 2, 3 of the Philox counter
MAX_NOISE_SAMPLES = 65535
_NOISE_BUDGET_BYTES = 1 << 30             # device memory of one chunk of samples: workspace, costs and usable bits
_M32 = 0xFFFFFFFF


def philox4x32_10(counter: Sequence[int], key: Sequence[int]) -> Tuple[int, int, int, int]:
    """Philox4x32-10 (Salmon et al., SC'11, the Random123 constants) of four 32-bit counter words under two key words."""
    c0, c1, c2, c3 = (int(v) & _M32 for v in counter)
    k0, k1 = (int(v) & _M32 for v in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & _M32, p1 & _M32, ((p0 >> 32) ^ c3 ^ k1) & _M32, p0 & _M32
    return c0, c1, c2, c3


def noise_factor(s: float, seed: int, j: int, index: int, bs: int, field: int, type_code: int, tpl: int) -> float:
    """The factor 1 + s * (2u - 1) of one value of sample j (metis_noise.cuh's noise_factor)."""
    r0, r1, _, _ = philox4x32_10((j, index, bs, field << 16 | type_code << 8 | tpl), (seed & _M32, seed >> 32))
    u = ((r0 << 32 | r1) >> 11) * 2.0 ** -53
    return 1.0 + s * (2.0 * u - 1.0)


def _real(v) -> bool:
    return isinstance(v, (int, float)) and not isinstance(v, bool)


def _sigma_value(v, where: str) -> float:
    if not _real(v) or not math.isfinite(v) or not 0.0 <= v < 1.0:
        raise ValueError(f'sigma {where}: must be a finite number in [0, 1), not {v!r}')
    return float(v)


def noise_sigmas(sigma) -> Dict[str, Tuple[float, Dict[str, float]]]:
    """``sigma`` (a float for every field and device type, or {field: float or {device type: float}}, fields of
    NOISE_FIELDS, device types named as in utils.DeviceType) as {field: (sigma of a type not named, {type: sigma})}.
    ValueError for an unknown field or device type, or a sigma that is not finite or outside [0, 1)."""
    from .utils import DeviceType
    if not isinstance(sigma, dict):
        s = _sigma_value(sigma, 'for every field')
        return {f: (s, {}) for f in NOISE_FIELDS}
    out = {f: (0.0, {}) for f in NOISE_FIELDS}
    for field, v in sigma.items():
        if field not in NOISE_FIELDS:
            raise ValueError(f'sigma: unknown field {field!r} (one of {", ".join(NOISE_FIELDS)})')
        if isinstance(v, dict):
            per = {}
            for name, s in v.items():
                if name not in DeviceType.__members__:
                    raise ValueError(f'sigma {field!r}: unknown device type {name!r}')
                per[name] = _sigma_value(s, f'{field!r} {name}')
            out[field] = (0.0, per)
        else:
            out[field] = (_sigma_value(v, repr(field)), {})
    return out


def _sigma_of(sig, field: str, type_name: str) -> float:
    default, per = sig[field]
    return per.get(type_name, default)


def check_seed(seed) -> int:
    if not isinstance(seed, int) or isinstance(seed, bool) or not 0 <= seed < 2 ** 64:
        raise ValueError(f'seed must be an int in [0, 2^64), not {seed!r}')
    return seed


def device_type_code(name: str) -> int:
    """The 1-based position of device type ``name`` in utils.DeviceType (A100 = 1 ... B200 = 6)."""
    from .utils import DeviceType
    names = list(DeviceType.__members__)
    if name not in names:
        raise ValueError(f'unknown device type {name!r}')
    return names.index(name) + 1


def noisy_profile(profile: Dict, sigma, seed: int, j: int) -> Dict:
    """Sample ``j`` of ``profile`` (a dict like ProfileDataLoader.load_profile_data_all()[0]) under ``sigma`` and
    ``seed``: a deep copy whose every ``time.layer-computes`` entry (field 1), ``memory`` entry (field 2) and
    ``time.fb_sync`` (field 3) of every DeviceType.<T> / tp<t>_bs<b> entry is multiplied by its own factor
    f = 1.0 + s * (2.0 * u - 1.0), s the field's sigma for T (noise_sigmas), u = ((r0 << 32 | r1) >> 11) * 2**-53 and
    (r0, r1, r2, r3) = Philox4x32-10 of the counter (j, index in the list (0 for fb_sync), b,
    field << 16 | type << 8 | log2(t)) under the key (seed & 0xffffffff, seed >> 32), type the 1-based position of T in
    utils.DeviceType.  Every operation is one IEEE double operation.  A field whose sigma is 0 is left as it is (ints
    stay ints); the 'model' section is never touched.  This is the definition of the samples of
    HetSearchResult.profile_noise."""
    sig = noise_sigmas(sigma)
    seed = check_seed(seed)
    if not isinstance(j, int) or isinstance(j, bool) or not 0 <= j <= _M32:
        raise ValueError(f'sample index must be an int in [0, 2^32), not {j!r}')
    out = copy.deepcopy(profile)
    for entry_name, entries in out.items():
        if not entry_name.startswith('DeviceType.'):
            continue
        name = entry_name[len('DeviceType.'):]
        s = [_sigma_of(sig, f, name) for f in NOISE_FIELDS]
        if not any(s):
            continue
        code = device_type_code(name)
        for key, entry in entries.items():
            t, b = int(key[2:].split('_bs')[0]), int(key.split('_bs')[1])
            tpl = t.bit_length() - 1
            tm = entry['time']
            if s[0]:
                tm['layer-computes'] = [v * noise_factor(s[0], seed, j, i, b, 1, code, tpl)
                                        for i, v in enumerate(tm['layer-computes'])]
            if s[1]:
                entry['memory'] = [v * noise_factor(s[1], seed, j, i, b, 2, code, tpl)
                                   for i, v in enumerate(entry['memory'])]
            if s[2] and _real(tm.get('fb_sync')):
                tm['fb_sync'] = tm['fb_sync'] * noise_factor(s[2], seed, j, 0, b, 3, code, tpl)
    return out


class ProfileNoise:
    """The profile-noise what-if of one search (HetSearchResult.profile_noise): every candidate, with its device groups,
    strategies and layer partition held fixed, under K seeded samples of the searched profile (noisy_profile).  With
    c[j, i], usable[j, i] what recost_profiles gives candidate i under sample j:

      best_pos[j], best_cost[j]  the usable candidate of lowest cost, ties to the lowest position (-1, NaN: none)
      wins[i]                    samples whose best_pos is i
      usable[i]                  samples in which candidate i is usable
      near[i]                    samples in which it is usable and c[j, i] <= best_cost[j] * (1.0 + within)
      regret[i]                  max_j (c[j, i] - best_cost[j]); +inf if it is unusable in any sample
      mean[i]                    its costs over the samples where it is usable, added in sample order, / usable[i]
                                 (NaN when usable[i] is 0)

    Candidates are in estimate_costs order.  Nothing here is a search under a sample: a search would re-run the
    strategy chain and the balancer and pick other partitions."""

    _DESCENDING = ('wins', 'near')
    _ASCENDING = ('regret', 'mean')

    def __init__(self, candidates, best_pos, best_cost, wins, near, usable, regret, mean, timings):
        self.candidates = candidates
        self.best_pos = best_pos              # int64 [K]
        self.best_cost = best_cost            # float64 [K]
        self.wins = wins                      # int64 [N]
        self.near = near                      # int64 [N]
        self.usable = usable                  # int64 [N]
        self.regret = regret                  # float64 [N]
        self.mean = mean                      # float64 [N]
        self.timings = timings

    def __len__(self) -> int:
        return len(self.best_pos)

    def order(self, by: str) -> np.ndarray:
        """Positions of the candidates by statistic ``by``: wins or near descending, regret or mean ascending (NaN
        last), ties by the searched cost, then the position."""
        if by in self._DESCENDING:
            key = -getattr(self, by)
        elif by in self._ASCENDING:
            key = getattr(self, by)
        else:
            raise ValueError(f'by must be one of {self._DESCENDING + self._ASCENDING}, not {by!r}')
        n = len(self.wins)
        return np.lexsort((np.arange(n), self.candidates.records['cost'][:n], key))

    def ranked(self, by: str, k: Optional[int] = None) -> List[Tuple]:
        """The first ``k`` (default: all) candidates by ``by`` (order) as the reference's 7-tuples, slot 6 the searched
        cost.  A ranking of the searched candidates, not a search under the samples."""
        pos = self.order(by)
        if k is not None:
            if int(k) < 0:
                raise ValueError(f'k must be >= 0, not {k}')
            pos = pos[:int(k)]
        return self.candidates.tuples(pos)


# ---------------------------------------------------------------------------------------------
# search what-if: a fresh search under each scenario profile (Candidates.search_scenarios)
# ---------------------------------------------------------------------------------------------
_SCENARIO_BUDGET_BYTES = 1 << 30         # device memory of one chunk of scenarios: their tables and staging


def noise_spec(sigma, type_code: Sequence[int], seed: int, within: float) -> native.MetisNoiseSpec:
    """The MetisNoiseSpec of a noise what-if: ``sigma`` [3, METIS_MAX_TYPES] and ``type_code`` per device type of the
    searched problem, the seed and near_factor = 1.0 + ``within`` (first and count are set per chunk)."""
    spec = native.MetisNoiseSpec()
    for f in range(3):
        for t in range(native.METIS_MAX_TYPES):
            spec.sigma[f][t] = float(sigma[f][t])
    for t, code in enumerate(type_code):
        spec.type_code[t] = int(code)
    spec.seed = int(seed)
    spec.near_factor = 1.0 + float(within)
    return spec


def one_search_segment(candidates) -> 'SearchSegment':
    """The one segment of a result searched at once; NotImplementedError naming the window count otherwise."""
    segs = candidates.segments
    if len(segs) != 1 or not isinstance(segs[0], SearchSegment):
        raise NotImplementedError(f'a search what-if of a result searched in {len(segs)} windows: only results '
                                  f'searched at once are supported')
    return segs[0]


class NoiseScenarios:
    """Samples first .. first + count - 1 of noisy_profile, drawn on the device with their norm_lc
    (metis_het_search_noise_*); the kept candidate is evaluated by metis_het_profile_noise_eval."""

    def __init__(self, spec: native.MetisNoiseSpec, count: int, norm_row: Optional[np.ndarray], norm_code: int,
                 norm_sigma: float):
        self.spec, self.count = spec, count
        self.norm = native.MetisNormSource(None, 0, norm_code, norm_sigma)
        self._norm_row = norm_row
        self._row = self._zero = self._ws = None

    def reserve(self, lib, p, device) -> int:
        """Allocates the device buffers of the call: the norm row, the zero-total flags and the draw workspace of one
        chunk, sized under _SCENARIO_BUDGET_BYTES.  Returns the samples of a chunk."""
        one = int(lib.metis_het_search_noise_workspace_bytes(C.byref(p), 1))
        native.check(min(one, 0), 'metis_het_search_noise_workspace_bytes')
        per = int(lib.metis_het_search_noise_workspace_bytes(C.byref(p), 2)) - one
        n = int(max(1, min(self.count, (_SCENARIO_BUDGET_BYTES - one + per) // per)))
        if self._norm_row is not None:
            self._row = upload(np.ascontiguousarray(self._norm_row, dtype=np.float64), device)
        self._zero = torch.zeros(self.count, dtype=torch.uint8, device=device)
        self._ws = torch.empty(int(lib.metis_het_search_noise_workspace_bytes(C.byref(p), n)), dtype=torch.uint8,
                               device=device)
        return n

    def search_bytes(self, lib, p, slots: int, max_stage: int) -> int:
        need = int(lib.metis_het_workspace_bytes(C.byref(p), slots, max_stage))     # a sample's layout is the base's
        native.check(min(need, 0), 'metis_het_workspace_bytes')
        return need

    def stage(self, lib, p, first: int, n: int, stream) -> List[native.MetisProblem]:
        if self._row is None:                       # sigma 0 for the norm entry: the row is not read
            self.norm.row, self.norm.len = p.norm_lc, p.norm_len
        else:
            self.norm.row, self.norm.len = self._row.data_ptr(), self._row.numel() // 8
        self.spec.first, self.spec.count = first, n
        native.check(lib.metis_het_search_noise_draw(C.byref(p), C.byref(self.spec), C.byref(self.norm), _ptr(self._ws),
                                                     C.c_int64(self._ws.numel()), _ptr(self._zero, first),
                                                     C.c_void_p(stream.cuda_stream)), 'metis_het_search_noise_draw')
        out = []
        for k in range(n):
            pr = native.MetisProblem()
            native.check(lib.metis_het_search_noise_problem(C.byref(p), C.byref(self.spec), C.c_int32(k),
                                                            _ptr(self._ws), C.byref(pr)), 'metis_het_search_noise_problem')
            out.append(pr)
        return out

    def eval_kept(self, lib, sp, first: int, n: int, rec, det, cost, usable, stream) -> None:
        native.check(lib.metis_het_profile_noise_eval(
            C.byref(sp), C.byref(self.spec), _ptr(self._ws), _ptr(rec), C.c_int64(1), _ptr(det),
            C.c_int32(det.shape[1]), _ptr(cost, 8 * first), _ptr(usable, first), C.c_int64(1),
            C.c_void_p(stream.cuda_stream)), 'metis_het_profile_noise_eval')

    def preset(self) -> torch.Tensor:
        """METIS_FATAL_ZERODIV where a sample's noisy norm total is 0, else 0."""
        return self._zero.to(torch.int64) * native.FATAL_ZERODIV


class ProfileScenarios:
    """Caller-given profiles, each flattened with its own norm_lc (``problems``); ``zerodiv[j]``: profile j's norm
    total is 0, so it is flattened with the searched norm_lc (as recost_profiles does) and not searched.  The kept
    candidate is evaluated by metis_het_profile_recost."""

    def __init__(self, problems: Sequence[flatten.FlatProblem], zerodiv: Sequence[bool]):
        self.problems, self.count, self.device = list(problems), len(problems), None
        self.zerodiv = np.asarray(zerodiv, dtype=bool)
        self._bound = []

    def reserve(self, lib, p, device) -> int:
        """The scenarios of one chunk under _SCENARIO_BUDGET_BYTES (their tables are bound per chunk by stage)."""
        self.device = device
        per = max(int(lib.metis_het_workspace_bytes(C.byref(pr.as_struct(lambda n: 0)), 0, 1)) +
                  sum(a.nbytes for a in pr.arrays.values()) for pr in self.problems)
        return int(max(1, min(self.count, _SCENARIO_BUDGET_BYTES // max(2 * per, 1))))

    def search_bytes(self, lib, p, slots: int, max_stage: int) -> int:
        need = [int(lib.metis_het_workspace_bytes(C.byref(pr.as_struct(lambda n: 0)), slots, max_stage))
                for pr in self.problems]
        native.check(min(min(need), 0), 'metis_het_workspace_bytes')
        return max(need)

    def stage(self, lib, p, first: int, n: int, stream) -> List[native.MetisProblem]:
        with torch.cuda.stream(stream):
            self._bound = [bind_problem(pr, self.device, workspace=False) for pr in self.problems[first:first + n]]
        return [b[1] if not self.zerodiv[first + k] else None for k, b in enumerate(self._bound)]

    def eval_kept(self, lib, sp, first: int, n: int, rec, det, cost, usable, stream) -> None:
        scen = (native.MetisProblem * n)(*[b[1] for b in self._bound])
        need = int(lib.metis_het_profile_recost_workspace_bytes(C.c_void_p(C.addressof(scen)), C.c_int32(n)))
        native.check(min(need, 0), 'metis_het_profile_recost_workspace_bytes')
        with torch.cuda.stream(stream):
            ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            head = torch.empty(n, dtype=torch.float64, device=self.device)
            status = torch.empty(n, dtype=torch.uint8, device=self.device)
            native.check(lib.metis_het_profile_recost(
                C.byref(sp), C.c_void_p(C.addressof(scen)), C.c_int32(n), _ptr(rec), C.c_int64(1), _ptr(det),
                C.c_int32(det.shape[1]), _ptr(cost, 8 * first), _ptr(head), _ptr(status), _ptr(ws),
                C.c_int64(ws.numel()), C.c_void_p(stream.cuda_stream)), 'metis_het_profile_recost')
            usable[first:first + n] = ((status == 0) & (head >= 0)).to(torch.uint8)

    def preset(self) -> torch.Tensor:
        return torch.from_numpy(self.zerodiv.astype(np.int64) * native.FATAL_ZERODIV)


class ScenarioSearch:
    """A fresh search under each of K scenario profiles P_j, next to the searched winner held fixed
    (HetSearchResult.search_noise / search_profiles).  S_j is what api.cost_het_cluster returns under P_j (the searched
    args, cluster, node sequences and corrections, the cost estimator and the layer balancer built from P_j, so its
    norm_lc too); R the searched result.  Arrays of length K:

      status           0, or the METIS_FATAL_* code with which cost_het_cluster under P_j raises (raise_fatal's
                       mapping; a norm_lc total of 0 is METIS_FATAL_ZERODIV)
      num_candidates   len(S_j), 0 when status != 0
      best_cost        S_j.best()'s cost, bit for bit (NaN when S_j has no best)
      kept_cost        R.best(), its device groups, strategies and partition fixed, under P_j: recost_profiles([P_j])'s
      kept_usable      cost and usable flag (status 0 and headroom >= 0); NaN / False when R is empty
      loss             kept_cost - best_cost when the kept plan is usable (not clamped: the balancer is not
                       cost-optimal, so it can be negative), +inf when it is not, NaN when S_j has no best
      near             kept usable and kept_cost <= best_cost * (1.0 + within)
      same             winner(j)[:6] == R.best()[:6];  same_plan: the same ordinal (node sequence, device groups, batches)

    ``winner(j)`` is S_j.best(), a 7-tuple, or None; ``winners()`` the distinct winners."""

    def __init__(self, candidates, kept: Optional[int], status, num_candidates, best, found, winners, kept_cost,
                 kept_usable, within: float, timings):
        K = len(status)
        self.status = status                            # int64 [K]
        self.num_candidates = num_candidates            # int64 [K]
        self._best = best                               # MetisRecord per scenario (valid where found)
        self._found = found                             # bool [K]: S_j has a best
        self._at = np.cumsum(found) - 1                 # scenario -> row of ``winners``
        self._winners = winners
        self.best_cost = np.where(found, best['cost'], np.nan)
        self.kept_cost = kept_cost                      # float64 [K]
        self.kept_usable = kept_usable                  # bool [K]
        self.kept = None if kept is None else candidates.tuples([kept])[0]
        with np.errstate(invalid='ignore'):
            self.loss = np.where(~found, np.nan, np.where(kept_usable, kept_cost - self.best_cost, np.inf))
            t = 1.0 + within
            self.near = kept_usable & found & (kept_cost <= self.best_cost * t)
        tuples = self._winners.tuples(np.arange(len(self._winners))) if len(self._winners) else []
        self._tuples = [tuples[self._at[j]] if found[j] else None for j in range(K)]
        kept_ordinal = -1 if kept is None else int(candidates.records['ordinal'][kept])
        self.same = np.array([w is not None and self.kept is not None and w[:6] == self.kept[:6]
                              for w in self._tuples], dtype=bool)
        self.same_plan = found & (best['ordinal'].astype(np.int64) == kept_ordinal)
        self.timings = timings

    def __len__(self) -> int:
        return len(self.status)

    def winner(self, j) -> Optional[Tuple]:
        """S_j.best(): the reference's 7-tuple, or None when S_j has no candidate or its search raises."""
        return self._tuples[int(j)]

    def winners(self) -> List[Tuple[Tuple, int, int]]:
        """The distinct winners, (7-tuple of the first sample that picked it, count, that first sample), keyed by
        ordinal, strategies, partition and num_repartition, by count descending, then first sample."""
        seen: Dict[Tuple, List[int]] = {}
        for j, t in enumerate(self._tuples):
            if t is None:
                continue
            key = (int(self._best['ordinal'][j]), tuple(t[2]), tuple(t[4]), t[5])
            if key in seen:
                seen[key][1] += 1
            else:
                seen[key] = [j, 1]
        return [(self._tuples[j], c, j) for j, c in sorted(seen.values(), key=lambda v: (-v[1], v[0]))]


def materialize(records: np.ndarray, detail: np.ndarray, space: flatten.FlatPlanSpace,
                node_sequences: Sequence[Tuple]) -> List[Tuple]:
    """Records -> the reference's 7-tuples (cost_het_cluster.py:44-46), all of them, eagerly."""
    cand = Candidates(records, detail, space, node_sequences)
    return cand.tuples(np.arange(len(records)))


def _bisect_records(rec: np.ndarray, lo: int, hi: int, ordinal: int, step: int) -> Optional[int]:
    """Index of (ordinal, step) in rec[lo:hi], sorted by (ordinal, step); None when absent."""
    want = (ordinal, step)
    end = hi
    while lo < hi:
        mid = (lo + hi) >> 1
        r = rec[mid]
        if (int(r['ordinal']), int(r['step'])) < want:
            lo = mid + 1
        else:
            hi = mid
    if lo < end and (int(rec[lo]['ordinal']), int(rec[lo]['step'])) == want:
        return lo
    return None


# ---------------------------------------------------------------------------------------------
# windowed search: a space larger than one search holds, walked in ordinal windows (flatten.plan_windows)
# ---------------------------------------------------------------------------------------------
_NO_FATAL = 2 ** 64 - 1
_SUMMED_KEYS = ('num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror', 'num_admitted',
                'num_chained')


@dataclass
class WindowedOutput:
    """The merged outputs of the windows searched: ``records`` (host) are every window's records in window order, each
    window's in (ordinal, step) order - together estimate_costs order; a record of window w has the global ordinal
    ``bases[w] + ordinal``.  ``firsts[w]`` is the index of window w's first record (``firsts[-1]`` = all records)."""
    summary: Dict[str, int]
    best: Optional[Tuple[float, int, int, int, int]]      # cost, GLOBAL ordinal, step, num_repartition, num_stage
    records: np.ndarray
    bases: np.ndarray                                     # int64 per window searched
    firsts: np.ndarray                                    # int64, one more than windows searched
    headroom: Optional[np.ndarray] = None                 # float64 aligned with records, when the windows had it
    headroom_s: float = 0.0
    misses: Optional[np.ndarray] = None                   # MISS_HOST_DTYPE, global ordinals, reference order
    misses_s: float = 0.0


class WindowMerge:
    """Host merge of per-window outputs: counters summed, the best as the lexicographic min of (cost, global ordinal,
    step), the fatal ordinal made global.  ``add`` returns True at the first window that reports a fatal plan: the
    reference dies at that plan (quirk Q8), so later windows are not searched."""

    def __init__(self, num_windows: int, with_headroom: bool = False, with_misses: bool = False):
        """``with_headroom``: the windows carry headroom, so an empty result gets an empty headroom array;
        ``with_misses``: the windows carry their out-of-memory attempts."""
        self.with_headroom = with_headroom
        self.with_misses = with_misses
        self._misses: List[np.ndarray] = []
        self.misses_s = 0.0
        self.summary: Dict[str, object] = {k: 0 for k in _SUMMED_KEYS}
        self.summary.update(fatal_ordinal=_NO_FATAL, fatal_code=0, fatal_aux=0, num_windows=num_windows,
                            windows_searched=0, instantiation=[])
        self.best = None
        self._records: List[np.ndarray] = []
        self._headroom: List[np.ndarray] = []
        self.headroom_s = 0.0
        self.bases: List[int] = []
        self.firsts: List[int] = [0]

    def add(self, base: int, summary: Dict[str, int], best, records: Optional[np.ndarray],
            headroom: Optional[np.ndarray] = None, misses: Optional[np.ndarray] = None) -> bool:
        """``headroom``: the window's per-record headroom, aligned with ``records`` (give it for every window or none);
        ``misses``: the window's out-of-memory attempts with window-relative ordinals (native.MISS_DTYPE or
        MISS_HOST_DTYPE), in (ordinal, call, attempt) order."""
        for k in _SUMMED_KEYS:
            self.summary[k] += int(summary.get(k, 0))
        if misses is not None:
            self.summary['num_oom_attempts'] = self.summary.get('num_oom_attempts', 0) + int(
                summary.get('num_oom_attempts', len(misses)))
            if len(misses):
                if misses.dtype == MISS_HOST_DTYPE:
                    misses = misses.copy()
                    misses['ordinal'] += int(base)
                else:
                    misses = misses_to_host(misses, base)
                self._misses.append(misses)
        self.summary['windows_searched'] += 1
        if 'instantiation' in summary:
            self.summary['instantiation'].append(summary['instantiation'])
        if best is not None:
            cand = (best[0], base + int(best[1]), int(best[2]), int(best[3]), int(best[4]))
            if self.best is None or cand[:3] < self.best[:3]:
                self.best = cand
        n = 0 if records is None else len(records)
        if n:
            self._records.append(records)
            if headroom is not None:
                self._headroom.append(headroom)
        self.bases.append(int(base))
        self.firsts.append(self.firsts[-1] + n)
        if int(summary.get('fatal_ordinal', _NO_FATAL)) != _NO_FATAL:
            self.summary.update(fatal_ordinal=base + int(summary['fatal_ordinal']), fatal_code=int(summary['fatal_code']),
                                fatal_aux=int(summary['fatal_aux']))
            return True
        return False

    def result(self) -> WindowedOutput:
        rec = np.concatenate(self._records) if self._records else np.zeros(0, dtype=native.RECORD_DTYPE)
        head = None
        if self._headroom or (self.with_headroom and not self._records):
            head = np.concatenate(self._headroom) if self._headroom else np.zeros(0)
            assert len(head) == len(rec), 'headroom given for some windows only'
        miss = None
        if self.with_misses or self._misses:
            miss = np.concatenate(self._misses) if self._misses else np.zeros(0, dtype=MISS_HOST_DTYPE)
            self.summary.setdefault('num_oom_attempts', len(miss))
        return WindowedOutput(dict(self.summary), self.best, rec, np.asarray(self.bases, dtype=np.int64),
                              np.asarray(self.firsts, dtype=np.int64), head, self.headroom_s, miss, self.misses_s)


def window_cost_model(problem: flatten.FlatProblem, lib=None) -> Tuple[float, float, float, float]:
    """(bytes per plan, per byte of rows, per composition record, fixed bytes) of one window's search on the device, from
    metis_het_workspace_bytes and the buffers the driver allocates around it: the workspace (with HetSearcher's 1/8
    headroom), a 16 B record slot per plan, and the arena's 1/4 headroom on the rows and composition records."""
    lib = lib or native.load_library()
    p = problem.as_struct(lambda n: problem.arrays[n].ctypes.data)
    n = 1 << 24
    w1, w2 = (int(lib.metis_het_workspace_bytes(C.byref(p), k, native.METIS_MAX_STAGES)) for k in (n, 2 * n))
    if min(w1, w2) < 0:
        native.check(min(w1, w2), 'metis_het_workspace_bytes')
    per_plan = (w2 - w1) / n * 9 / 8
    fixed = (w1 - n * (w2 - w1) / n) * 9 / 8 + sum(a.nbytes for a in problem.arrays.values())
    return per_plan + 16.0, 1.25, 20.0, fixed


def window_budget(device, fixed: float) -> float:
    """Device bytes a window may use: what is free on ``device`` (including memory this process has cached but does not
    use), less a tenth for the sorts and transfers around a search, less the fixed part of the cost model."""
    free, _total = torch.cuda.mem_get_info(device)
    free += torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)
    return free * 0.9 - fixed


def agree_budget(budget: float, device) -> float:
    """With torch.distributed initialised: the smallest ``budget`` of all ranks (one all_reduce), so that every rank
    makes the same one-search / windows choice and cuts the same windows; else ``budget``."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return budget
    t = torch.tensor([int(budget)], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    return float(t.item())


def search_windows(problem: flatten.FlatProblem, windows: Sequence[flatten.PlanWindow], device=None, rank: int = 0,
                   world: int = 1, tile: int = 128, headroom: bool = False, misses: bool = False
                   ) -> Tuple[WindowedOutput, DeviceProblem, 'HetSearcher']:
    """Search the windows in ordinal order in ONE DeviceProblem arena (sized for every window up front) with ONE
    HetSearcher (the shard's tiles of every window, workspace sized for the window with the most plans), records only,
    and merge on the host (WindowMerge).  Afterwards the searcher keeps only what rebuilding candidates needs
    (metis_het_detail's workspace): the work lists and the record buffer are released."""
    dp = DeviceProblem(problem, windows[0].space, device, reserve=windows)
    searcher = HetSearcher(dp, rank, world, tile, want_records=True, want_detail=False, want_headroom=headroom,
                           want_misses=misses)
    searcher.reserve_workspace(max(w.space.num_plans for w in windows))
    merge = WindowMerge(len(windows), with_headroom=headroom, with_misses=misses)
    for w in windows:
        if dp.space is not w.space:                           # the first window was uploaded by the constructor
            dp.reload(problem, w.space)
            dp.upload()
            searcher.rebind()
        out = searcher.run()
        merge.headroom_s += out.headroom_s
        merge.misses_s += out.misses_s
        if merge.add(w.base, out.summary, out.best, np.array(out.records) if out.records is not None else None,
                     np.array(out.headroom) if out.headroom is not None else None, out.misses):
            break
    searcher.release()
    return merge.result(), dp, searcher


def window_candidates(merged: WindowedOutput, windows: Sequence, problem: flatten.FlatProblem,
                      node_sequences: Sequence[Tuple], searcher: HetSearcher) -> Candidates:
    """The candidates of a windowed search (search_windows' searcher, its merged or gathered output): one WindowSegment
    per window searched."""
    segments = [WindowSegment(w, merged.firsts[k], merged.firsts[k + 1], problem, searcher)
                for k, w in enumerate(windows[:len(merged.bases)])]
    return Candidates(merged.records, None, None, node_sequences, headroom=merged.headroom, misses=merged.misses,
                      segments=segments)


def merge_rank_windows(all_counts: np.ndarray, records: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """The records of every rank -> estimate_costs order.  ``records``: every rank's records, rank after rank, each
    rank's window by window; ``all_counts[r, w]``: records of rank r in window w.  Returns (positions into ``records``
    in estimate_costs order: each window's union by (ordinal, step), windows in order; first record per window +
    total), so that whatever travels with the records follows them by the same positions."""
    world, nwin = all_counts.shape
    starts = np.concatenate([[0], np.cumsum(all_counts.reshape(-1))]).astype(np.int64)    # rank-major
    parts, firsts = [], [0]
    for w in range(nwin):
        at = np.concatenate([np.arange(starts[r * nwin + w], starts[r * nwin + w + 1]) for r in range(world)])
        union = records[at]
        parts.append(at[np.lexsort((union['step'], union['ordinal']))])
        firsts.append(firsts[-1] + len(at))
    return (np.concatenate(parts) if parts else np.zeros(0, dtype=np.int64)), np.asarray(firsts, dtype=np.int64)


def gather_window_records(merged: WindowedOutput, device) -> WindowedOutput:
    """Multi-GPU: every rank receives every rank's records (with their headroom, and the misses, when the windows had
    them), window by window in estimate_costs order.  The per-window record counts in one all_gather on ``device``,
    then gather_padded of the records and of the headroom, merged by merge_rank_windows.  Every rank must have searched
    the same windows (no fatal plan: api.cost_het_cluster raises before gathering)."""
    miss = gather_misses(merged.misses, device) if merged.misses is not None else None   # global ordinals already
    counts = torch.tensor(np.diff(merged.firsts), dtype=torch.int64, device=device)
    all_counts = _gather_rows(counts).numpy().astype(np.int64)     # [world, windows]
    totals = all_counts.sum(axis=1).tolist()
    mine = torch.from_numpy(np.ascontiguousarray(merged.records).view(np.int64).reshape(-1, 2)).to(device)
    records = gather_padded(mine, totals).cpu().numpy().reshape(-1).view(native.RECORD_DTYPE)
    order, firsts = merge_rank_windows(all_counts, records)
    headroom = None
    if merged.headroom is not None:
        mine = torch.from_numpy(np.ascontiguousarray(merged.headroom, dtype=np.float64)).to(device)
        headroom = gather_padded(mine, totals).cpu().numpy()[order]
    return WindowedOutput(merged.summary, merged.best, records[order], merged.bases, firsts, headroom,
                          merged.headroom_s, miss, merged.misses_s)


def _rank_on_device(searcher: 'HetSearcher', buf: torch.Tensor, n: int) -> np.ndarray:
    """Permutation (uint32) of ``sorted(records, key=cost)`` (stable) of the n device records in ``buf``, which the
    sort reorders."""
    dev = searcher.dp.device
    with torch.cuda.device(dev):
        s = torch.cuda.current_stream(dev)
        perm = searcher.sort_records(n, native.SORT_BY_COST_STABLE, s, want_perm=True, buf=buf)
        s.synchronize()
        return perm.cpu().numpy().view(np.uint32)


def make_window_ranker(searcher: 'HetSearcher', records: np.ndarray, summary: Dict):
    """() -> permutation of ``sorted(records, key=cost)`` (stable) for the concatenated records of a windowed search:
    metis_sort_records(METIS_SORT_BY_COST_STABLE) on the device when the records and the sort workspace fit in free
    device memory, else numpy's stable sort on the host.  ``summary['ranking']`` says which one ran."""
    n = len(records)
    if n > 0xFFFFFFFF:
        raise NotImplementedError(f'ranking {n} candidates: the rank permutation holds 2^32 indices')
    dev = searcher.dp.device

    def rank() -> np.ndarray:
        need = n * 16 + n * 4 + int(searcher.dp.lib.metis_sort_workspace_bytes(C.c_int64(n)))
        if need <= window_budget(dev, 0.0):
            out = _rank_on_device(searcher, torch.from_numpy(records.view(np.int64).reshape(-1)).to(dev), n)
            summary['ranking'] = 'device'
            return out
        summary['ranking'] = 'host'
        return np.argsort(records['cost'], kind='stable').astype(np.uint32)
    return rank


# ---------------------------------------------------------------------------------------------
# multi-GPU: shard by plan ordinal, one collective at the end (SURVEY.md section 8e)
# ---------------------------------------------------------------------------------------------
def _gather_rows(vec: torch.Tensor) -> torch.Tensor:
    """all_gather of one small vector per rank -> [world, len] on the host (ONE collective, one synchronisation)."""
    import torch.distributed as dist
    world = dist.get_world_size()
    out = torch.empty(world * vec.numel(), dtype=vec.dtype, device=vec.device)
    dist.all_gather_into_tensor(out, vec)
    return out.view(world, vec.numel()).cpu()


def _rank_counts(n: int, device) -> List[int]:
    """``n`` of every rank (one all_gather)."""
    return _gather_rows(torch.tensor([n], dtype=torch.int64, device=device)).reshape(-1).tolist()


def gather_padded(rows: torch.Tensor, counts: Sequence[int]) -> torch.Tensor:
    """Every rank's ``rows`` [counts[r], ...] (same trailing shape and dtype on every rank), concatenated in rank order
    on ``rows.device``: ONE all_gather_into_tensor of the rows padded to the largest count."""
    import torch.distributed as dist
    world = dist.get_world_size()
    cap = max(max(counts), 1)
    pad = torch.empty((cap,) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
    pad[:rows.shape[0]] = rows
    got = torch.empty((world * cap,) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
    dist.all_gather_into_tensor(got.view(-1), pad.view(-1))
    return torch.cat([got[cap * r:cap * r + counts[r]] for r in range(world)])


_NO_ORDINAL = 2 ** 40
_COUNTER_KEYS = ['num_records', 'num_partition_calls', 'num_balancer_runs', 'num_keyerror']


def _best_row(local_best: Optional[Tuple[float, int, int, int, int]]) -> List[int]:
    """(cost bits, ordinal, step, meta) as int64; a rank without records sends an ordinal nobody has."""
    if local_best is None:
        return [0, _NO_ORDINAL, 0, 0]
    cost, ordinal, step, nrep, nstage = local_best
    return [int(np.array([cost], dtype=np.float64).view(np.int64)[0]), int(ordinal), int(step), int(nrep) * 256 + int(nstage)]


def _pick_best(rows: List[List[int]]) -> Optional[Tuple]:
    """Exact lexicographic min of (cost, ordinal, step) over the ranks' bests."""
    cand = []
    for bits, o, st, m in rows:
        if o < _NO_ORDINAL:
            cand.append((float(np.array([bits], dtype=np.int64).view(np.float64)[0]), int(o), int(st), int(m)))
    if not cand:
        return None
    c, o, st, m = min(cand, key=lambda r: (r[0], r[1], r[2]))
    return (c, o, st, m // 256, m % 256)


def _merge_counters(summary: Dict[str, int], rows: List[List[int]]) -> Dict[str, int]:
    """rows[r] = counters (4), error flag, fatal ordinal, fatal code, fatal aux of rank r."""
    out = dict(summary)
    for i, k in enumerate(_COUNTER_KEYS):
        out[k] = int(sum(r[i] for r in rows))
    out['records_per_rank'] = [int(r[0]) for r in rows]
    out['any_rank_failed'] = int(sum(r[4] for r in rows))
    fatal = [(r[5], r[6], r[7]) for r in rows if r[5] < _NO_ORDINAL]
    if fatal:
        fo, code, aux = min(fatal)                            # the lowest ordinal, with ITS code and aux
        out.update(global_fatal_ordinal=int(fo), global_fatal_code=int(code), global_fatal_aux=int(aux))
    else:
        out.update(global_fatal_ordinal=2 ** 62, global_fatal_code=0, global_fatal_aux=0)
    return out


def _counter_row(summary: Dict[str, int], local_error: int) -> List[int]:
    fo = min(summary.get('fatal_ordinal', 2 ** 64 - 1), _NO_ORDINAL)
    return [int(summary.get(k, 0)) for k in _COUNTER_KEYS] + \
        [int(local_error != 0), int(fo), int(summary.get('fatal_code', 0)) & 0xFF, int(summary.get('fatal_aux', 0))]


def global_best(local_best: Optional[Tuple[float, int, int, int, int]], device) -> Optional[Tuple]:
    """all_gather of one (cost, ordinal, step, meta) record per rank, then the exact lexicographic min."""
    rows = _gather_rows(torch.tensor(_best_row(local_best), dtype=torch.int64, device=device)).tolist()
    return _pick_best(rows)


def global_counters(summary: Dict[str, int], device, local_error: int = 0) -> Dict[str, int]:
    """Sum of the counters over the ranks, the records of every rank, the lowest fatal ordinal with ITS code and aux,
    and an error flag (``any_rank_failed``) so that a rank whose search raised makes every rank raise instead of
    leaving the others in a collective."""
    rows = _gather_rows(torch.tensor(_counter_row(summary, local_error), dtype=torch.int64, device=device)).tolist()
    return _merge_counters(summary, rows)


def global_exchange(summary: Dict[str, int], local_best, device, local_error: int = 0):
    """global_counters and global_best in ONE collective (the API path)."""
    vec = torch.tensor(_counter_row(summary, local_error) + _best_row(local_best), dtype=torch.int64, device=device)
    rows = _gather_rows(vec).tolist()
    return _merge_counters(summary, [r[:8] for r in rows]), _pick_best([r[8:] for r in rows])


def make_ranker(searcher: 'HetSearcher', records_dev: torch.Tensor):
    """() -> permutation of ``sorted(records, key=cost)`` (stable): the device sort on a private copy of the ordered
    records, run when a caller first asks for the ranking."""
    snap = records_dev.clone()
    return lambda: _rank_on_device(searcher, snap, snap.numel() // 2)


def check_threshold(min_headroom) -> float:
    """A headroom threshold must be a finite real number (MB)."""
    try:
        x = float(min_headroom)
    except (TypeError, ValueError):
        raise ValueError(f'min_headroom must be a finite number, not {min_headroom!r}') from None
    if isinstance(min_headroom, (bool, np.bool_)) or not math.isfinite(x):
        raise ValueError(f'min_headroom must be a finite number, not {min_headroom!r}')
    return x


class HeadroomIndex:
    """The records, their headroom and the ranked order of one result on the device, for metis_headroom_select and
    metis_headroom_front (uploaded once, on the first query)."""

    def __init__(self, records: np.ndarray, headroom: np.ndarray, rank_order: np.ndarray, device=None):
        self.device = _require_cuda(device)
        self.lib = native.load_library()
        self.n = len(records)
        if not (len(headroom) == len(rank_order) == self.n):
            raise ValueError('records, headroom and rank order differ in length')
        with torch.cuda.device(self.device):
            self.records = upload(records, self.device)
            self.headroom = upload(np.asarray(headroom, dtype=np.float64), self.device)
            self.rank = upload(np.asarray(rank_order, dtype=np.uint32), self.device)
            need = int(self.lib.metis_headroom_workspace_bytes(C.c_int64(self.n)))
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
            self.out = torch.empty(max(self.n, 1), dtype=torch.int32, device=self.device)
        self.count = torch.zeros(1, dtype=torch.int64).pin_memory()

    def launch_select(self, min_headroom: float, k: int, stream) -> None:
        rc = self.lib.metis_headroom_select(C.c_void_p(self.headroom.data_ptr()), C.c_void_p(self.rank.data_ptr()),
                                            C.c_int64(self.n), C.c_double(min_headroom), C.c_int64(k),
                                            C.c_void_p(self.out.data_ptr()), C.c_void_p(self.count.data_ptr()),
                                            C.c_void_p(self.workspace.data_ptr()), C.c_int64(self.workspace.numel()),
                                            C.c_void_p(stream.cuda_stream))
        native.check(rc, 'metis_headroom_select')

    def launch_front(self, stream) -> None:
        rc = self.lib.metis_headroom_front(C.c_void_p(self.records.data_ptr()), C.c_void_p(self.headroom.data_ptr()),
                                           C.c_void_p(self.rank.data_ptr()), C.c_int64(self.n),
                                           C.c_void_p(self.out.data_ptr()), C.c_void_p(self.count.data_ptr()),
                                           C.c_void_p(self.workspace.data_ptr()), C.c_int64(self.workspace.numel()),
                                           C.c_void_p(stream.cuda_stream))
        native.check(rc, 'metis_headroom_front')

    def select(self, min_headroom: float, k: Optional[int] = None) -> Tuple[np.ndarray, int]:
        """(positions of the first ``k`` (default: all) ranked entries with headroom >= min_headroom, how many
        qualify in all)."""
        x = check_threshold(min_headroom)
        if k is not None and int(k) < 0:
            raise ValueError(f'k must be >= 0 with min_headroom, not {k}')
        k = self.n if k is None else min(int(k), self.n)
        with torch.cuda.device(self.device):
            s = torch.cuda.current_stream(self.device)
            self.launch_select(x, k, s)
            s.synchronize()
            total = int(self.count[0])
            return self.out[:min(k, total)].cpu().numpy().view(np.uint32).astype(np.int64), total

    def front(self) -> np.ndarray:
        """Positions of the cost / headroom Pareto front, by ascending cost."""
        with torch.cuda.device(self.device):
            s = torch.cuda.current_stream(self.device)
            self.launch_front(s)
            s.synchronize()
            return self.out[:int(self.count[0])].cpu().numpy().view(np.uint32).astype(np.int64)


def gather_records(out: HetSearchOutput, searcher: HetSearcher, want_rank: bool = True,
                   counts: Optional[List[int]] = None) -> HetSearchOutput:
    """Every rank receives every rank's records (+ detail rows, headroom and misses when the search had them): padded
    tensor all_gathers over NCCL (gather_padded, no pickling), then the merged list is put into estimate_costs order and
    ranked by the device sort, the detail rows and the headroom permuted with it; the misses are merged into the
    reference's order (gather_misses).  ``counts``: the records of every rank, when the caller has them."""
    dev = searcher.dp.device
    if counts is None:
        counts = _rank_counts(len(out.records), dev)
    with torch.cuda.device(dev):
        rec_all = gather_padded(out.records_dev.view(-1, 2), counts).view(-1)
        det_all = gather_padded(out.detail_dev, counts) if out.detail_dev is not None else None
        head_all = gather_padded(out.headroom_dev, counts) if out.headroom_dev is not None else None
        n = sum(counts)
        s = torch.cuda.current_stream(dev)
        perm = searcher.sort_records(n, native.SORT_POSITION, s, want_perm=True, buf=rec_all)
        records = searcher._to_host('records_all', rec_all, s).view(native.RECORD_DTYPE)
        detail_dev = det_all.index_select(0, perm.long()) if det_all is not None else None
        rank_order = None
        if want_rank:
            rank = searcher.sort_records(n, native.SORT_BY_COST_STABLE, s, want_perm=True, buf=rec_all.clone())
            rank_order = searcher._to_host('rank_all', rank, s).view(np.uint32)
        detail = None
        if detail_dev is not None and searcher.detail_to_host:
            detail = searcher._to_host('detail_all', detail_dev, s).reshape(n, searcher.detail_stride)
        headroom = headroom_dev = None
        if head_all is not None:
            headroom_dev = head_all.index_select(0, perm.long())
            headroom = searcher._to_host('headroom_all', headroom_dev, s).view(np.float64)
    misses = gather_misses(out.misses, dev) if out.misses is not None else None
    return HetSearchOutput(out.summary, out.best, records, detail, out.d2h_bytes, rank_order, detail_dev, rec_all,
                           headroom, headroom_dev, out.headroom_s, misses, out.misses_s)


# ---------------------------------------------------------------------------------------------
# out-of-memory partition attempts of a search (misses)
# ---------------------------------------------------------------------------------------------
class Misses:
    """The out-of-memory partition attempts of a search, columnar, in the reference's order (ordinal, call, attempt):
    every pass of LayerLoadBalancer.partition_layer's loop whose memory test failed (model/load_balancer.py:57-63,
    127-143).  ``ordinal`` is the inter-stage plan's global ordinal, ``call`` the 0-based partition_layer call of that
    plan (one per valid strategy it tried), ``attempt`` 1..3, ``deficit`` = -min(memory_state) in MB (> 0) and
    ``stage`` the lowest stage with that smallest state."""

    def __init__(self, table: np.ndarray):
        self.table = table                                    # MISS_HOST_DTYPE
        self.ordinal = table['ordinal'].astype(np.int64)
        self.call = table['call'].astype(np.int64)
        self.attempt = table['attempt'].astype(np.int64)
        self.stage = table['stage'].astype(np.int64)
        self.num_stage = table['num_stage'].astype(np.int64)
        self.deficit = np.ascontiguousarray(table['deficit'])

    def __len__(self) -> int:
        return len(self.table)


def closest_order(deficit: np.ndarray, device=None) -> np.ndarray:
    """Positions of the misses by ascending deficit, ties in reference order: metis_sort_records(METIS_SORT_RANKED) on
    MetisMiss rows whose ordinal field holds the position (the rows are already in reference order)."""
    n = len(deficit)
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    if n > 0xFFFFFFFF:
        raise NotImplementedError(f'ordering {n} misses: positions are 32-bit')
    rows = np.zeros(n, dtype=native.MISS_DTYPE)
    rows['deficit'] = deficit
    rows['ordinal'] = np.arange(n, dtype=np.uint32)
    return sorted_positions(rows, native.SORT_RANKED, _require_cuda(device))


def _find_attempt(items: list, call: int, attempt: int):
    """The TraceCall of partition_layer call ``call`` and its TraceAttempt ``attempt`` in a decoded plan."""
    from .verbose import TraceCall
    calls = [it for it in items if isinstance(it, TraceCall)]
    c = calls[call]
    for a in c.attempts:
        if a.attempt == attempt:
            return c, a
    raise AssertionError(f'attempt {attempt} of call {call} not in the replay')


def replay_misses(candidates, misses: Misses, idx: np.ndarray):
    """(plan columns, [(TraceCall, TraceAttempt)]) of the misses ``idx``: each distinct plan is replayed once by
    metis_het_trace, and the failed attempt is looked up in its decoded events."""
    idx = np.asarray(idx, dtype=np.int64).reshape(-1)
    ords = misses.ordinal[idx]
    uniq, inv = np.unique(ords, return_inverse=True)
    traced = candidates.trace(uniq) if len(uniq) else []
    found = [_find_attempt(traced[inv[k]], int(misses.call[i]), int(misses.attempt[i])) for k, i in enumerate(idx)]
    return candidates.plan_columns(ords), found


def miss_tuples(candidates, misses: Misses, idx) -> List[Tuple]:
    """(node_sequence, device_groups, strategies, batches, layer_partition, attempt, deficit, stage) of misses ``idx``."""
    idx = np.asarray(idx, dtype=np.int64).reshape(-1)
    if not len(idx):
        return []
    col, found = replay_misses(candidates, misses, idx)
    out = []
    for k, i in enumerate(idx.tolist()):
        S = int(col['num_stage'][k])
        groups = (1 << col['codes'][k, :S].astype(np.int64)).tolist()
        call, att = found[k]
        strategies = [(g >> t, 1 << t) for g, t in zip(groups, call.tpc)]
        out.append((candidates.node_sequences[int(col['ns_idx'][k])], groups, strategies, int(col['batches'][k]),
                    list(att.partition), int(misses.attempt[i]), float(misses.deficit[i]), int(misses.stage[i])))
    return out


@dataclass
class MissDetail:
    """Per-stage values of chosen misses, one row per miss in the order asked for; NaN past a miss's stages."""
    performance: np.ndarray       # [n, width]: stage performance fed to the attempt's balancer run
    memory_capacity: np.ndarray   # stage_memory_capacity
    memory_demand: np.ndarray     # stage_memory_demand of the attempt
    memory_state: np.ndarray      # memory_state (capacity - demand) of the attempt
    num_stage: np.ndarray

    def __len__(self) -> int:
        return len(self.num_stage)


def memory_capacity(problem: flatten.FlatProblem, ns_idx: int, groups: Sequence[int]) -> List[float]:
    """StagePerformance.get_device_group_memory_capacity of every stage (model/device_group.py:87-101), like
    PlanEvaluator::memory_capacity: the stage's devices of each type run, summed in run order."""
    a = problem.arrays
    mem, typ, end = a['type_memory'], a['ns_run_type'][ns_idx], a['ns_run_end'][ns_idx]
    out, lo_rank = [], 0
    for g in groups:
        hi_rank = lo_rank + g
        if len(mem) == 1:
            out.append(float(mem[0]) * float(g))
        else:
            terms, lo = [], 0
            for k in range(len(end)):
                hi = int(end[k])
                x, y = max(lo_rank, lo), min(hi_rank, hi)
                if y > x:
                    terms.append(float(mem[typ[k]]) * float(y - x))
                lo = hi
            out.append(sum(terms))
        lo_rank = hi_rank
    return out


def miss_detail(candidates, misses: Misses, idx) -> MissDetail:
    idx = np.asarray(idx, dtype=np.int64).reshape(-1)
    width = max(int(misses.num_stage[idx].max()), 1) if len(idx) else 1
    f = {k: np.full((len(idx), width), np.nan) for k in ('performance', 'memory_capacity', 'memory_demand',
                                                          'memory_state')}
    if len(idx):
        col, found = replay_misses(candidates, misses, idx)
        for k in range(len(idx)):
            S = int(col['num_stage'][k])
            groups = (1 << col['codes'][k, :S].astype(np.int64)).tolist()
            _call, att = found[k]
            f['performance'][k, :S] = att.performance
            f['memory_capacity'][k, :S] = memory_capacity(candidates.problem, int(col['ns_idx'][k]), groups)
            f['memory_demand'][k, :S] = att.demand
            f['memory_state'][k, :S] = att.state
    return MissDetail(num_stage=misses.num_stage[idx].copy(), **f)


def gather_misses(misses: np.ndarray, device) -> np.ndarray:
    """Multi-rank: every rank receives every rank's misses (MISS_HOST_DTYPE, global ordinals), as int64 words through
    gather_padded, merged into the reference's order."""
    words = MISS_HOST_DTYPE.itemsize // 8
    mine = torch.from_numpy(np.ascontiguousarray(misses).view(np.int64).reshape(-1, words)).to(device)
    got = gather_padded(mine, _rank_counts(len(misses), device))
    return position_order(got.cpu().numpy().reshape(-1).view(MISS_HOST_DTYPE))


# ---------------------------------------------------------------------------------------------
# homogeneous path
# ---------------------------------------------------------------------------------------------
def homo_costs(problem: flatten.FlatProblem, type_id: int, plans: np.ndarray, device=None
               ) -> Tuple[np.ndarray, np.ndarray]:
    """HomoCostEstimator.get_cost for every row (dp, pp, tp, mbs, gbs) of ``plans`` on the GPU."""
    dev = _require_cuda(device)
    with torch.cuda.device(dev):
        lib, p, _sp, ws, _keep = bind_problem(problem, dev)
        n = len(plans)
        d_plans = torch.from_numpy(np.ascontiguousarray(plans, dtype=np.int32).reshape(-1)).to(dev)
        cost = torch.zeros(max(n, 1), dtype=torch.float64, device=dev)
        status = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        s = torch.cuda.current_stream(dev)
        rc = lib.metis_homo_cost(C.byref(p), C.c_int32(type_id), C.c_void_p(d_plans.data_ptr()), C.c_int64(n),
                                 C.c_void_p(cost.data_ptr()), C.c_void_p(status.data_ptr()),
                                 C.c_void_p(ws.data_ptr()), C.c_int64(ws.numel()), C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_homo_cost')
        s.synchronize()
        return cost[:n].cpu().numpy(), status[:n].cpu().numpy()


def homo_breakdown(problem: flatten.FlatProblem, type_id: int, plans: np.ndarray, device=None
                   ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """metis_homo_breakdown for every row (dp, pp, tp, mbs, gbs) of ``plans``: (terms [n, 6], per-stage memory
    [n, largest pp] NaN-padded, status: 0 ok, 1 KeyError, 2 oom)."""
    dev = _require_cuda(device)
    plans = np.ascontiguousarray(plans, dtype=np.int32).reshape(-1, 5)
    n = len(plans)
    width = max(int(plans[:, 1].max()) if n else 1, 1)
    with torch.cuda.device(dev):
        lib, p, _sp, ws, _keep = bind_problem(problem, dev)
        d_plans = torch.from_numpy(plans.reshape(-1)).to(dev)
        terms = torch.empty((max(n, 1), 6), dtype=torch.float64, device=dev)
        mem = torch.empty((max(n, 1), width), dtype=torch.float64, device=dev)
        status = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        s = torch.cuda.current_stream(dev)
        rc = lib.metis_homo_breakdown(C.byref(p), C.c_int32(type_id), C.c_void_p(d_plans.data_ptr()), C.c_int64(n),
                                      C.c_void_p(terms.data_ptr()), C.c_void_p(mem.data_ptr()), C.c_int32(width),
                                      C.c_void_p(status.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_int64(ws.numel()),
                                      C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_homo_breakdown')
        s.synchronize()
        return terms[:n].cpu().numpy(), mem[:n].cpu().numpy(), status[:n].cpu().numpy()


def layer_balance(capa_rows: Sequence[Sequence[float]], lc: Sequence[float], num_layers: int, device=None
                  ) -> List[List[int]]:
    """LayerComputeBalancer.run for many capacity vectors on the GPU (unit-level entry point)."""
    dev = _require_cuda(device)
    lib = native.load_library()
    n = len(capa_rows)
    stride = max(len(c) for c in capa_rows)
    capa = np.zeros((n, stride))
    ns = np.zeros(n, dtype=np.int32)
    for i, c in enumerate(capa_rows):
        capa[i, :len(c)] = c
        ns[i] = len(c)
    with torch.cuda.device(dev):
        d_capa = torch.from_numpy(capa).to(dev)
        d_ns = torch.from_numpy(ns).to(dev)
        d_lc = torch.tensor(list(lc), dtype=torch.float64, device=dev)
        out = torch.zeros((n, stride + 1), dtype=torch.int16, device=dev)
        ws = torch.empty(len(lc) * 8 + 512, dtype=torch.uint8, device=dev)
        s = torch.cuda.current_stream(dev)
        rc = lib.metis_layer_balance(C.c_void_p(d_capa.data_ptr()), C.c_void_p(d_ns.data_ptr()), C.c_int64(n),
                                     C.c_int32(stride), C.c_void_p(d_lc.data_ptr()), C.c_int32(len(lc)),
                                     C.c_int32(num_layers), C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()),
                                     C.c_int64(ws.numel()), C.c_void_p(s.cuda_stream))
        native.check(rc, 'metis_layer_balance')
        s.synchronize()
        res = out.cpu().numpy().view(np.uint16)
    return [res[i, :ns[i] + 1].tolist() for i in range(n)]
