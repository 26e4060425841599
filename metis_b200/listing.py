"""Device-side listing of a plan space's compositions (metis_list_*, include/metis_b200.h; SURVEY.md 8(f)-1).

The host enumerator (metis_enum_compositions) keeps every composition record of a space on the host.  Here the GPU
lists them, one thread per composition; the host receives the rows of each stage count (for the block list and the
window planner, flatten.plan_listed_windows) and, window by window, the window's own records and pool.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from . import flatten, native


class DeviceListing:
    """The compositions of stage counts 1..``cap`` of ``num_devices`` GPUs, listed on ``device``.  The workspace (the
    counting table and one row offset per composition) stays on the device while windows are emitted from it."""

    def __init__(self, num_devices: int, cap: int, variance, max_permute_len: int, device, max_ranges: int = 1):
        self.device = torch.device(device)
        self.lib = native.load_library()
        self.listing = native.MetisListing(1, cap, num_devices, max_permute_len, float(variance), max(1, max_ranges), 0)
        comps = np.zeros(cap, dtype=np.int64)
        n = int(self.lib.metis_list_workspace_bytes(C.byref(self.listing), comps.ctypes.data))
        if n < 0:
            native.check(n, 'metis_list_workspace_bytes')
        self.comps_per_stage = comps
        with torch.cuda.device(self.device):
            self.workspace = torch.empty(n, dtype=torch.uint8, device=self.device)
            rows = torch.zeros(cap, dtype=torch.int64).pin_memory()
            most = torch.zeros(1, dtype=torch.int32).pin_memory()
            s = torch.cuda.current_stream(self.device)
            rc = self.lib.metis_list_stages(C.byref(self.listing), C.c_void_p(self.workspace.data_ptr()), C.c_int64(n),
                                            C.c_void_p(rows.data_ptr()), C.c_void_p(most.data_ptr()),
                                            C.c_void_p(s.cuda_stream))
            native.check(rc, 'metis_list_stages')
            s.synchronize()
        self.rows_per_stage = rows.numpy().copy()
        self.max_groups = int(most.item())
        self._sizes = torch.zeros(3, dtype=torch.int64).pin_memory()
        self._recs = self._pool = None
        self._current: Optional[Tuple[object, flatten.FlatPlanSpace]] = None

    def _window(self, ranges: np.ndarray, write: bool) -> Tuple[int, int]:
        ranges = np.ascontiguousarray(ranges, dtype=native.RANGE_DTYPE)
        if len(ranges) > self.listing.max_ranges:
            raise ValueError(f'{len(ranges)} row ranges: the listing was sized for {self.listing.max_ranges}')
        with torch.cuda.device(self.device):
            s = torch.cuda.current_stream(self.device)
            recs = self._recs if write else None
            pool = self._pool if write else None
            rc = self.lib.metis_list_window(
                C.byref(self.listing), C.c_void_p(self.workspace.data_ptr()), C.c_int64(self.workspace.numel()),
                C.c_void_p(ranges.ctypes.data), C.c_int32(len(ranges)),
                C.c_void_p(recs.data_ptr() if recs is not None else 0),
                C.c_int64(recs.numel() // 24 if recs is not None else 0),
                C.c_void_p(pool.data_ptr() if pool is not None else 0), C.c_int64(pool.numel() if pool is not None else 0),
                C.c_void_p(self._sizes.data_ptr()), C.c_void_p(s.cuda_stream))
            native.check(rc, 'metis_list_window')
            s.synchronize()
        nrec, pool_bytes, status = (int(v) for v in self._sizes.tolist())
        if status & 3:
            raise native.MetisNativeError(f'metis_list_window: status {status} (a range outside its table, or a '
                                          f'composition of more than {native.METIS_MAX_PERMUTE_GROUPS} merged groups)')
        return nrec, pool_bytes

    def size(self, ranges: np.ndarray) -> Tuple[int, int]:
        """(records, pool bytes) of the window whose rows are ``ranges`` (native.RANGE_DTYPE)."""
        return self._window(ranges, False)

    def emit(self, ranges: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """The records (native.COMP_DTYPE) and pool of the window whose rows are ``ranges``, on the host."""
        nrec, pool_bytes = self.size(ranges)
        with torch.cuda.device(self.device):
            if self._recs is None or self._recs.numel() < nrec * 24:
                self._recs = torch.empty(max(nrec * 24 + nrec * 3, 24 * 64), dtype=torch.uint8, device=self.device)
            if self._pool is None or self._pool.numel() < pool_bytes:
                self._pool = torch.empty(max(pool_bytes + pool_bytes // 8, 4096), dtype=torch.uint8, device=self.device)
        got = self._window(ranges, True)
        if got != (nrec, pool_bytes):
            raise native.MetisNativeError('metis_list_window: inconsistent sizes')
        recs = self._recs[:nrec * 24].cpu().numpy().view(native.COMP_DTYPE)
        pool = np.zeros(max(pool_bytes, 16), dtype=np.uint8)
        pool[:pool_bytes] = self._pool[:pool_bytes].cpu().numpy()
        return recs, pool

    def window_space(self, window: flatten.ListedWindow) -> flatten.FlatPlanSpace:
        """``window``'s space with its records and pool (written on first use; the listing keeps one window's)."""
        if self._current is not None and self._current[0] is window:
            return self._current[1]
        recs, pool = self.emit(window.ranges)
        window.num_recs, window.pool_bytes = len(recs), int(pool.size)
        lay = window.layout
        sp = flatten.FlatPlanSpace(lay.num_plans, lay.blocks, lay.batches, lay.rows, rows_total_bytes=lay.rows_total_bytes,
                                   comp_recs=recs, comp_pool=pool)
        self._current = (window, sp)
        return sp
