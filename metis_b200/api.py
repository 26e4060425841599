"""Host-side mirror of the reference's interface for the plan-search path.

Same class / function names, argument meaning and error behaviour as the reference, so that
``cost_het_cluster.py`` / ``cost_homo_cluster.py`` read like the originals; the objects are thin
holders of inputs - every evaluation happens on the GPU (metis_b200.search).

  reference symbol                                   here
  -------------------------------------------------  -------------------------------------------
  model/activation_parameter.py GPTActivationAndParam  GPTActivationAndParam
  model/cost_estimator.py HeteroCostEstimator           HeteroCostEstimator   (holder)
  model/cost_estimator.py HomoCostEstimator             HomoCostEstimator     (holder)
  model/load_balancer.py LayerLoadBalancer              LayerLoadBalancer     (holder + norm_layer_duration)
  search_space/plan.py UniformPlan / InterStagePlan     same dataclasses
  search_space/plan.py UniformPlanGenerator             UniformPlanGenerator  (host iterator)
  search_space/plan.py InterStagePlanGenerator          InterStagePlanGenerator (iterator over the plan space)
  cost_het_cluster.py cost_het_cluster()                cost_het_cluster()    -> GPU
  cost_homo_cluster.py cost_homo_cluster()              cost_homo_cluster()   -> GPU
"""
from __future__ import annotations

import argparse
import math
import time
from dataclasses import dataclass
from itertools import permutations
from collections.abc import Sequence
from typing import Dict, Iterator, List, Optional, Tuple

import numpy as np

from . import flatten, native
from .utils import DeviceType, ModelConfig


@dataclass
class UniformPlan:
    dp: int
    pp: int
    tp: int
    mbs: int
    gbs: int


@dataclass
class InterStagePlan:
    ns_idx: int
    node_sequence: List[DeviceType]
    dg_idx: int
    device_groups: List[int]
    num_stage: int
    batches: int
    gbs: int


class GPTActivationAndParam:
    """model/activation_parameter.py:5-51 (only the three per-layer sizes reach the kernels)."""

    def __init__(self, model_config: ModelConfig, model_params):
        self.hidden_size = model_config.hidden_size
        self.sequence_length = model_config.sequence_length
        self.num_layers = model_config.num_layers
        self.vocab_size = model_config.vocab_size
        self.attention_head_size = model_config.attention_head_size
        self.input_params = float(model_params[0])
        self.output_params = float(model_params[-1])
        self.transformer_params = float(model_params[1])

    def get_num_layers(self):
        return self.num_layers


class _Estimator:
    def __init__(self, profile_data: Dict, model_config: ModelConfig, model_volume, gpu_cluster):
        self.profile_data = profile_data
        self.model_config = model_config
        self.model_volume = model_volume
        self.gpu_cluster = gpu_cluster


class HeteroCostEstimator(_Estimator):
    """Inputs of model/cost_estimator.py:141-244; evaluated by het_search_kernel."""


class HomoCostEstimator(_Estimator):
    """Inputs of model/cost_estimator.py:83-138; evaluated by homo_cost_kernel."""


class LayerLoadBalancer:
    """Inputs of model/load_balancer.py:14-144; ``norm_layer_duration`` is computed at construction
    like the reference (:20-27) and raises the same KeyError when tp1_bs1 is not profiled."""

    def __init__(self, gpu_cluster, profile_data: Dict, model_config, gbs: int):
        self.gpu_cluster = gpu_cluster
        self.profile_data = profile_data
        self.model_config = model_config
        self.gbs = gbs
        self.norm_layer_duration = flatten.norm_layer_duration(profile_data)


class UniformPlanGenerator:
    """search_space/plan.py:40-97; like the reference it re-yields ONE mutated object."""

    def __init__(self, num_devices: int, max_tp: int, max_gbs: int):
        self.num_devices = num_devices
        self.max_tp = max_tp
        self.max_gbs = max_gbs
        self.curr = UniformPlan(dp=num_devices, pp=1, tp=1, gbs=num_devices, mbs=0)

    def __iter__(self):
        return self

    def _advance_parallelism(self) -> bool:
        p = self.curr
        while True:
            if p.tp == self.max_tp and p.pp == self.num_devices:
                return False
            if p.tp == self.max_tp:
                p.pp += 1
                p.dp = self.num_devices // p.pp
                p.tp = self.num_devices // p.dp // p.pp
            else:
                p.tp += 1
                p.dp = self.num_devices // p.tp // p.pp
            if p.dp * p.pp * p.tp == self.num_devices:
                return True

    def __next__(self) -> UniformPlan:
        p = self.curr
        p.mbs += 1
        while p.gbs % p.mbs > 0 and p.mbs <= p.gbs:
            p.mbs += 1
        if p.mbs * p.dp > p.gbs:
            p.mbs = 1
            p.gbs += 1
            while self.max_gbs % p.gbs > 0 and p.gbs <= self.max_gbs:
                p.gbs += 1
        if p.gbs > self.max_gbs:
            p.mbs = 1
            if not self._advance_parallelism():
                raise StopIteration
            p.gbs = p.dp
        return p


class InterStagePlanGenerator:
    """search_space/plan.py:100-175 as an iterator over the enumerated plan space (quirk Q1 included).
    Each item is a fresh InterStagePlan (the reference mutates one object)."""

    def __init__(self, device_types: set, num_devices: int, gbs: int, num_layers: int, variance: float = 0.5,
                 max_permute_len: int = 4):
        self.node_sequences = list(permutations(device_types))
        self.gbs = gbs
        self.space = flatten.build_plan_space(len(self.node_sequences), num_devices, gbs, num_layers, variance,
                                              max_permute_len)

    def __iter__(self) -> Iterator[InterStagePlan]:
        for ordinal in range(self.space.num_plans):
            ns, label, row, batches, codes = self.space.locate(ordinal)
            yield InterStagePlan(ns_idx=ns, node_sequence=self.node_sequences[ns], dg_idx=row,
                                 device_groups=[1 << int(c) for c in codes], num_stage=label, batches=batches,
                                 gbs=self.gbs)


class HetSearchResult(Sequence):
    """What cost_het_cluster() returns: the reference's list of 7-tuples
    ``(node_sequence, device_groups, strategies, batches, layer_partition, num_repartition, cost)`` in
    ``estimate_costs`` order (cost_het_cluster.py:44-46), as a read-only sequence whose tuples are built when they
    are asked for (the columns live in numpy arrays; strategies / partitions stay on the GPU until needed).
    ``len()``, indexing, slicing, iteration, ``sorted(result, key=...)`` and comparison with a list behave like the
    reference's list.  ``ranked()`` is ``sorted(result, key=lambda kv: kv[6])`` (cost_het_cluster.py:76, a stable
    sort) taken from the device sort's permutation instead of sorting Python objects."""

    def __init__(self, candidates, rank_order: Optional[np.ndarray], summary: Dict[str, int],
                 timings: Optional[Dict[str, float]] = None, ranker=None, best_key: Optional[Tuple[int, int]] = None):
        self.candidates = candidates
        # fp64 memory headroom of every candidate in estimate_costs order: the smallest memory_state (capacity - demand,
        # MB) over the stages of its accepted partition attempt; None unless searched with headroom=True
        self.headroom = getattr(candidates, 'headroom', None)
        self._headroom_index = None
        self._misses = getattr(candidates, 'misses', None)   # MISS_HOST_DTYPE rows, or None without misses=True
        self._misses_view = None
        self._closest = None                  # positions of the misses by ascending deficit (device sort)
        self.rank_order = rank_order          # permutation of sorted(..., key=cost); computed on first use (``ranker``)
        self.summary = summary
        self.timings = timings or {}
        self._ranker = ranker                 # () -> uint32 permutation, the stable device sort by cost
        self._best_key = best_key             # (ordinal, step) of the argmin found by the search kernels
        self._searched = None                 # cluster_signature of the cluster searched (cost_het_cluster sets it)
        # (cluster, model_config, gbs, max_tp, max_bs, node_sequences, corrected) the search flattened its profile
        # under (cost_het_cluster sets it): a profile what-if flattens its scenarios the same way
        self._flat_inputs = None
        self._norm_source = None              # norm_source() of the searched profile (cost_het_cluster sets it)

    def __len__(self) -> int:
        return len(self.candidates)

    def __getitem__(self, i):
        n = len(self)
        if isinstance(i, slice):
            return self.candidates.tuples(np.arange(n)[i])
        i = int(i)
        if i < 0:
            i += n
        if not 0 <= i < n:
            raise IndexError('list index out of range')
        return self.candidates.tuples([i])[0]

    def __iter__(self) -> Iterator[Tuple]:
        n = len(self)
        for lo in range(0, n, 8192):
            yield from self.candidates.tuples(np.arange(lo, min(n, lo + 8192)))

    def __eq__(self, other) -> bool:
        if not isinstance(other, (list, tuple, Sequence)) or len(other) != len(self):
            return False
        return all(a == b for a, b in zip(self, other))

    __hash__ = None

    @property
    def costs(self) -> np.ndarray:
        """fp64 cost of every candidate, estimate_costs order (no tuples built)."""
        return self.candidates.cost

    def ranked(self, k: Optional[int] = None, min_headroom: Optional[float] = None, where=None) -> List[Tuple]:
        """The first ``k`` (default: all) entries of ``sorted(result, key=lambda kv: kv[6])``.  With ``min_headroom``
        (MB, finite; needs ``headroom=True``): the first ``k`` of those whose headroom is at least that, in ranked
        order (metis_headroom_select on the GPU); ``k`` must then be >= 0 (a count, not a slice bound).

        ``where`` (a search.PlanFilter): only the candidates it admits, ``[t for t in sorted(result, key=cost) if
        where.admits(t)]``, then the ``min_headroom`` condition, then the first ``k`` (metis_query_mark and
        metis_mask_select on the GPU).  The filter selects among the candidates this search found; it does not
        constrain the search."""
        if where is not None:
            from . import search
            if min_headroom is not None and k is not None and int(k) < 0:
                raise ValueError(f'k must be >= 0 with min_headroom, not {k}')
            mask, _group = self._mark(where, min_headroom)
            n = len(self)
            sliced = k is None or int(k) < 0
            pos, _total = search.mask_select(mask, n, self._rank_device(), n if sliced else int(k))
            return self.candidates.tuples(pos[:k] if sliced and k is not None else pos)
        if min_headroom is not None:
            from . import search
            x = search.check_threshold(min_headroom)
            if k is not None and int(k) < 0:
                raise ValueError(f'k must be >= 0 with min_headroom, not {k}')
            pos, _total = self._index().select(x, k)
            return self.candidates.tuples(pos)
        self._rank()
        order = self.rank_order
        if k is not None:
            order = order[:k]
        return self.candidates.tuples(order)

    def count(self, where=None, min_headroom: Optional[float] = None) -> int:
        """How many candidates ``where`` (a search.PlanFilter, default: all) admits with headroom >= ``min_headroom``
        (needs ``headroom=True``), counted on the GPU."""
        if where is None and min_headroom is None:
            return len(self)
        from . import search
        mask, _group = self._mark(where, min_headroom)
        return search.mask_select(mask, len(self), None, 0)[1]

    def best_by(self, keys, where=None, min_headroom: Optional[float] = None):
        """The best admitted candidate per key value: ``keys`` is a subset of ('node_sequence', 'num_stage', 'batches',
        'max_tp', 'num_repartition') ('max_tp': the largest tp of any stage).  For every value of the keys that some
        candidate admitted by ``where`` (with headroom >= ``min_headroom``) has, a search.Groups row holds the values,
        the count and the first such candidate of sorted(result, key=cost) - lowest cost, then lowest estimate_costs
        position - as its position and cost (``.tuples()`` builds them), in ascending key order.  Computed on the GPU
        over a dense table of groups, at most 2^24 (metis_query_groups)."""
        from . import search
        keys = search.check_keys(keys)
        cand = self.candidates
        n = len(cand.records)
        ranges = {'node_sequence': len(cand.node_sequences),
                  'num_stage': max(int(cand.records['num_stage'].max()), 1) if n else 1,
                  'batches': len(self._batches()), 'max_tp': int(cand.problem.scalars['num_tp']),
                  'num_repartition': 3}
        num_groups = int(np.prod([ranges[k] for k in keys], dtype=np.float64))
        if num_groups > 1 << 24:
            raise ValueError(f'best_by{keys}: {num_groups} groups, more than 2^24')
        mask, group = self._mark(where, min_headroom, keys, [ranges[k] for k in keys])
        admitted = search.mask_select(mask, n, None, 0)[1]
        ids, count, _cost, first = search.group_best(cand.records_device(), group, n, num_groups)
        if int(count.sum()) != admitted:
            raise native.MetisNativeError(f'best_by{keys}: {admitted - int(count.sum())} admitted candidates outside '
                                          f'the key ranges {ranges}')
        batches = self._batches()
        digits = []
        rest = ids.copy()
        for k in reversed(keys):
            digits.append(rest % ranges[k])
            rest //= ranges[k]
        digits = digits[::-1]
        decode = {'node_sequence': lambda d: cand.node_sequences[d], 'num_stage': lambda d: d + 1,
                  'batches': lambda d: int(batches[len(batches) - 1 - d]), 'max_tp': lambda d: 1 << d,
                  'num_repartition': lambda d: d + 1}
        values = [tuple(decode[k](int(digits[j][g])) for j, k in enumerate(keys)) for g in range(len(ids))]
        order = sorted(range(len(values)), key=lambda g: tuple(search._names(v) if k == 'node_sequence' else v
                                                               for k, v in zip(keys, values[g])))
        pos = first[order].astype(np.int64)
        return search.Groups(cand, keys, [values[g] for g in order], count[order].astype(np.int64), pos,
                             np.array(self.costs[pos]))

    def _batches(self) -> np.ndarray:
        """The divisors of gbs every plan space of the result enumerates (MetisPlanSpace.batches)."""
        spaces = [s.space for s in self.candidates.segments]
        b = spaces[0].batches
        if any(not np.array_equal(s.batches, b) for s in spaces[1:]):
            raise NotImplementedError('the windows of this result enumerate different batches')
        return b

    def _mark(self, where, min_headroom, keys=(), key_ranges=()):
        """metis_query_mark of ``where`` (and the headroom threshold) on every candidate: (mask, group) on the device."""
        from . import search
        where = search.PlanFilter() if where is None else where
        if not isinstance(where, search.PlanFilter):
            raise TypeError(f'where must be a search.PlanFilter, not {type(where).__name__}')
        cand = self.candidates
        flt = where.to_struct(cand.problem.type_names, cand.node_sequences, self._batches())
        flt.num_keys = len(keys)
        for j, k in enumerate(keys):
            flt.key_field[j] = search.QUERY_KEYS.index(k)
            flt.key_range[j] = key_ranges[j]
        headroom, x = None, 0.0
        if min_headroom is not None:
            x = search.check_threshold(min_headroom)
            headroom = self._index().headroom
        return cand.query(flt, where.reads_strategies or 'max_tp' in keys, headroom, x, groups=bool(keys))

    def _rank_device(self):
        """The rank permutation on the device (uploaded once)."""
        if getattr(self, '_rank_dev', None) is None:
            from . import search
            self._rank_dev = search.upload(np.ascontiguousarray(self._rank(), dtype=np.uint32),
                                           search._require_cuda(self.candidates.device))
        return self._rank_dev

    def _rank(self) -> np.ndarray:
        if self.rank_order is None:
            self.rank_order = self._ranker() if self._ranker is not None \
                else np.argsort(self.candidates.cost, kind='stable')
            self._ranker = None
        return self.rank_order

    def _index(self):
        if self.headroom is None:
            raise ValueError('this result has no headroom: call cost_het_cluster(..., headroom=True)')
        if self._headroom_index is None:
            from . import search
            self._headroom_index = search.HeadroomIndex(self.candidates.records, self.headroom, self._rank(),
                                                        getattr(self.candidates, 'device', None))
        return self._headroom_index

    @property
    def misses(self):
        """Every out-of-memory partition attempt of the search (needs ``misses=True``): a search.Misses of numpy columns
        ``ordinal`` (global, int64), ``call``, ``attempt``, ``stage`` and ``deficit`` (MB, > 0), in the order the
        reference prints them: (ordinal, call, attempt)."""
        if self._misses is None:
            raise ValueError('this result has no misses: call cost_het_cluster(..., misses=True)')
        if self._misses_view is None:
            from . import search
            self._misses_view = search.Misses(self._misses)
        return self._misses_view

    def _closest_order(self) -> np.ndarray:
        if self._closest is None:
            from . import search
            self._closest = search.closest_order(self.misses.deficit, getattr(self.candidates, 'device', None))
        return self._closest

    def closest_misses(self, k: int) -> List[Tuple]:
        """The ``k`` out-of-memory attempts with the smallest deficit (needs ``misses=True``), closest first, ties in
        the reference's order (the device record sort): tuples (node_sequence, device_groups, strategies, batches,
        layer_partition, attempt, deficit, stage).  The strategies and partition of each attempt come from replaying
        its plan (metis_het_trace)."""
        from . import search
        misses = self.misses
        if int(k) < 0:
            raise ValueError(f'k must be >= 0, not {k}')
        return search.miss_tuples(self.candidates, misses, self._closest_order()[:int(k)])

    def miss_detail(self, idx):
        """Per-stage performance (fed to the attempt's balancer run), memory capacity, demand and state of the misses
        ``idx`` (an int, a slice or an index array of positions into ``misses``), NaN past a miss's stages
        (search.MissDetail).  Replayed like closest_misses."""
        from . import search
        misses = self.misses
        if isinstance(idx, slice):
            idx = np.arange(len(misses))[idx]
        return search.miss_detail(self.candidates, misses, idx)

    def pareto(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The cost / headroom Pareto front (needs ``headroom=True``): (positions in estimate_costs order, their costs,
        their headrooms), by ascending cost, headroom strictly increasing.  A candidate is on the front iff no other
        one has cost <= and headroom >= with one of the two strict; of equal (cost, headroom) pairs only the first in
        estimate_costs order is kept.  Computed by metis_headroom_front on the GPU."""
        pos = self._index().front()
        return pos, self.costs[pos], self.headroom[pos]

    def breakdown(self, idx, per_stage: bool = True):
        """Cost terms and memory headroom of the candidates at ``idx`` (an int, a slice or an index array of positions
        in estimate_costs order; ranked positions: ``result.breakdown(result.rank_order[:k])`` after ``ranked()``),
        replayed on the GPU (metis_het_breakdown).  Returns a search.Breakdown with one row per position asked for;
        ``per_stage=False`` leaves out the per-stage arrays."""
        n = len(self)
        if isinstance(idx, slice):
            pos = np.arange(n)[idx]
        else:
            pos = np.asarray(idx, dtype=np.int64).reshape(-1)
            pos = np.where(pos < 0, pos + n, pos)
            if len(pos) and (pos.min() < 0 or pos.max() >= n):
                raise IndexError('list index out of range')
        return self.candidates.breakdown(pos, per_stage)

    def recost(self, clusters: Sequence) -> 'search.Recost':
        """Network what-if: every candidate re-costed under each GPUCluster of ``clusters`` on the GPU
        (metis_het_recost), with no new search.  Bandwidth enters only the cost model (model/cost_estimator.py:205-232),
        so a search under a cluster that differs from the searched one only in bandwidth returns the same candidates
        with these costs, bit for bit.  Each cluster must therefore have the searched hostfile entries (ip and GPU
        count, in order) and the same instance_type and memory on every node; every bandwidth the model reads
        (intra_bandwidth, and inter_bandwidth when the search used 'Q2') must be finite and > 0.  The corrections of
        the search apply to every scenario.  Returns a search.Recost: ``costs`` [K, N], ``ranked(j, k)``, ``best(j)``,
        ``regret`` and ``robust(k)``.  With torch.distributed every rank holds all candidates: no collective is
        issued."""
        from . import search
        if self._searched is None:
            raise ValueError('this result does not know the cluster it was searched on: no recost')
        clusters = list(clusters)
        if not clusters:
            raise ValueError('recost needs at least one cluster')
        corrected = tuple(self.summary.get('corrected', ()))
        type_names = self.candidates.problem.type_names
        bw = np.empty((len(clusters), 2, len(type_names)), dtype=np.float64)
        for j, cluster in enumerate(clusters):
            check_scenario(self._searched, cluster, type_names, corrected, j)
            bw[j, 0], bw[j, 1] = flatten.cluster_bandwidths(cluster, type_names, corrected)
        return self.candidates.recost(bw)

    def recost_profiles(self, profiles: Sequence[Dict]) -> 'search.Recost':
        """Profile what-if: every candidate, with its device groups, strategies and layer partition held fixed, under
        each profile of ``profiles`` (dicts shaped like ProfileDataLoader.load_profile_data_all()[0]) on the GPU
        (metis_het_profile_recost).  For scenario j: ``costs[j]`` is HeteroCostEstimator.get_cost
        (model/cost_estimator.py:199-244) under profile j, ``headroom[j]`` the smallest memory capacity -
        LayerLoadBalancer._get_stage_memory_demand (model/load_balancer.py:29-55) over all stages under profile j, and
        ``status[j]`` cost code | memory code << 4 (METIS_FATAL_*; a raising get_cost is METIS_FATAL_KEY_EXEC); a
        candidate is ``usable`` under j when status == 0 and headroom >= 0.  This is not what a search under profile j
        returns: a search would re-run the strategy chain and the balancer and pick other partitions.  Under the
        searched profile, costs and headroom equal the search's bit for bit.  The corrections of the search apply to
        every scenario.  A profile without a 'model' section holding parameters, optimizer_time and batch_generator,
        or without an entry for a device type of the cluster, is refused with a ValueError; wrong values are not:
        they become statuses, as they would be errors in the reference.  Returns a search.Recost whose ``ranked(j, k)``
        and ``best(j)`` list the candidates usable under j by scenario cost, and whose ``regret`` and ``robust(k)``
        take unusable entries as +inf.  With torch.distributed every rank holds all candidates: no collective is
        issued."""
        if self._flat_inputs is None:
            raise ValueError('this result does not know the inputs it was searched on: no recost_profiles')
        profiles = list(profiles)
        if not profiles:
            raise ValueError('recost_profiles needs at least one profile')
        cluster, model_config, gbs, max_tp, max_bs, seqs, corrected = self._flat_inputs
        problem = self.candidates.problem
        for j, prof in enumerate(profiles):
            check_profile(prof, problem.type_names, j)
        norm = problem.arrays['norm_lc']                      # read by the balancer only, which does not run here
        scen = [flatten.build_problem(prof, cluster, model_config, gbs, max_tp, max_bs, seqs, norm, corrected=corrected)
                for prof in profiles]
        return self.candidates.recost_profiles(scen)

    def profile_noise(self, samples: int, sigma, seed: int = 0, within: float = 0.01) -> 'search.ProfileNoise':
        """Profile-noise what-if: how often each candidate wins, stays within ``within`` (relative) of the best and
        fits, over ``samples`` seeded samples of the searched profile drawn on the GPU.  Sample j is
        ``search.noisy_profile(profile, sigma, seed, j)``: every layer-computes and memory entry and every fb_sync
        multiplied by its own factor 1 + s * (2u - 1), u uniform in [0, 1) from a counter-based generator, s the
        field's sigma for the device type (a float, or {field: float or {device type: float}} over 'layer-computes',
        'memory' and 'fb_sync'; each in [0, 1)).  Each sample is evaluated as recost_profiles evaluates a profile, with
        every candidate's device groups, strategies and layer partition held fixed; only the per-sample best and the
        per-candidate counts leave the device.  Every array of the returned search.ProfileNoise equals the numpy
        reductions of recost_profiles over the samples' dicts, bit for bit; under all-zero sigma every sample is the
        searched profile.  This is not a search under each sample.  ValueError for samples outside 1 .. 65535, a
        sigma, seed or within out of range, or an unknown field or device type.  With torch.distributed every rank
        computes locally: no collective is issued."""
        table, codes, seed, _sig = self._noise_args(samples, sigma, seed, within)
        return self.candidates.profile_noise(table, codes, seed, samples, float(within))

    def _noise_args(self, samples: int, sigma, seed: int, within: float):
        """The checked arguments of a noise what-if: (sigma table [3, METIS_MAX_TYPES] and device type codes per device
        type of the searched problem, the seed, noise_sigmas(sigma))."""
        from . import search
        if not isinstance(samples, int) or isinstance(samples, bool) or not 1 <= samples <= search.MAX_NOISE_SAMPLES:
            raise ValueError(f'samples must be an int in [1, {search.MAX_NOISE_SAMPLES}], not {samples!r}')
        if not search._real(within) or not math.isfinite(within) or within < 0:
            raise ValueError(f'within must be a finite number >= 0, not {within!r}')
        sig = search.noise_sigmas(sigma)
        seed = search.check_seed(seed)
        problem = self.candidates.problem
        table = np.zeros((3, native.METIS_MAX_TYPES))
        codes = [search.device_type_code(name) for name in problem.type_names]
        for f, field in enumerate(search.NOISE_FIELDS):
            for t, name in enumerate(problem.type_names):
                table[f, t] = search._sigma_of(sig, field, name)
        return table, codes, seed, sig

    def search_noise(self, samples: int, sigma, seed: int = 0, within: float = 0.01) -> 'search.ScenarioSearch':
        """Search what-if under profile noise: a fresh search under each of ``samples`` seeded samples of the searched
        profile, ``search.noisy_profile(profile, sigma, seed, j)`` as profile_noise draws them, with the balancer's
        layer weights (norm_lc) of the sample too, next to the searched best held fixed.  Sample j's search is
        bit for bit what cost_het_cluster returns under that sample's dict with the searched args, cluster, node
        sequences and corrections and a HeteroCostEstimator and LayerLoadBalancer built from the dict.  Returns a
        search.ScenarioSearch: each sample's status, candidate count, winner and best cost, the searched best's cost
        and fit under it, the loss of keeping the searched best and whether it stays ``within`` of the winner.  Under
        all-zero sigma every sample's search is this result's.  The same ValueErrors as profile_noise;
        NotImplementedError for a result searched in more than one window.  With torch.distributed every rank
        computes locally: no collective is issued."""
        from . import search
        table, codes, seed, sig = self._noise_args(samples, sigma, seed, within)
        if self._norm_source is None:
            raise ValueError('this result does not know the profile entry its layer weights come from: no search_noise')
        name, row = self._norm_source
        problem = self.candidates.problem
        s, code = 0.0, 1
        if name.startswith('DeviceType.'):
            tname = name[len('DeviceType.'):]
            if any(search._sigma_of(sig, f, tname) for f in search.NOISE_FIELDS):
                code = search.device_type_code(tname)            # noisy_profile refuses an unknown type the same way
            s = search._sigma_of(sig, 'layer-computes', tname)
        if s and len(row) != problem.scalars['norm_len']:
            raise ValueError(f"the searched layer weights have {problem.scalars['norm_len']} entries, the profile's "
                             f'first entry {name} has {len(row)}: not the profile the balancer was built from')
        spec = search.noise_spec(table, codes, seed, within)
        scen = search.NoiseScenarios(spec, samples, row if s else None, code, float(s))
        return self.candidates.search_scenarios(scen, self._best_position(), float(within))

    def search_profiles(self, profiles: Sequence[Dict], within: float = 0.01) -> 'search.ScenarioSearch':
        """Search what-if under given profiles: a fresh search under each profile of ``profiles``, flattened under
        the searched args, cluster, node sequences and corrections with its own layer weights (norm_lc, from its
        first-listed entry), next to the searched best held fixed, evaluated as recost_profiles evaluates it.  Returns
        a search.ScenarioSearch as search_noise does; a profile whose layer-weight total is 0 has the status
        METIS_FATAL_ZERODIV.  The same ValueErrors as recost_profiles; NotImplementedError for a result searched in
        more than one window.  With torch.distributed every rank computes locally: no collective is issued."""
        from . import search
        if self._flat_inputs is None:
            raise ValueError('this result does not know the inputs it was searched on: no search_profiles')
        profiles = list(profiles)
        if not profiles:
            raise ValueError('search_profiles needs at least one profile')
        if not search._real(within) or not math.isfinite(within) or within < 0:
            raise ValueError(f'within must be a finite number >= 0, not {within!r}')
        cluster, model_config, gbs, max_tp, max_bs, seqs, corrected = self._flat_inputs
        problem = self.candidates.problem
        for j, prof in enumerate(profiles):
            check_profile(prof, problem.type_names, j)
        scen, zerodiv = [], []
        for prof in profiles:
            try:
                norm, zero = flatten.norm_layer_duration(prof), False
            except ZeroDivisionError:                     # LayerLoadBalancer(prof) raises: nothing is searched
                norm, zero = problem.arrays['norm_lc'], True
            zerodiv.append(zero)
            scen.append(flatten.build_problem(prof, cluster, model_config, gbs, max_tp, max_bs, seqs, norm,
                                              corrected=corrected))
        return self.candidates.search_scenarios(search.ProfileScenarios(scen, zerodiv), self._best_position(),
                                                float(within))

    def _best_position(self) -> Optional[int]:
        """The position of best() in estimate_costs order, or None for an empty result."""
        if self.rank_order is None and self._best_key is not None and len(self):
            at = self.candidates.index_of(*self._best_key)    # records sorted by (ordinal, step): no temporaries
            if at is not None:
                return at
        order = self._rank()
        return int(order[0]) if len(order) else None

    def best(self) -> Optional[Tuple]:
        """argmin (cost, position): the first entry of the ranked list.  The search kernels reduce it on the device
        (het_finalize_kernel: lowest cost, then lowest ordinal, then lowest step), so no sort is needed for it."""
        at = self._best_position()
        return self.candidates.tuples([at])[0] if at is not None else None


def cluster_signature(gpu_cluster, type_names: Sequence[str]) -> Tuple[list, list]:
    """What a network what-if must keep from the searched cluster: (ip, GPU count, instance_type, memory) of every
    hostfile entry in order, and the memory each device type of ``type_names`` is given (the first clusterfile entry of
    the type, gpu_cluster.py:47-50)."""
    nodes = []
    for h in gpu_cluster.host_entries.values():
        info = gpu_cluster.nodes_info.get(h['ip'], {})
        nodes.append((h['ip'], h['num_device'], info.get('instance_type'), info.get('memory')))
    return nodes, [gpu_cluster.get_device_memory_for_device_type(t) for t in type_names]


_NODE_FIELDS = ('ip', 'GPU count', 'instance_type', 'memory')
_MODEL_FIELDS = ('parameters', 'optimizer_time', 'batch_generator')


def check_profile(profile, type_names: Sequence[str], j: int) -> None:
    """ValueError, naming scenario j and the missing item, unless ``profile`` has a 'model' section with parameters,
    optimizer_time and batch_generator and an entry for every device type of ``type_names``."""
    if not isinstance(profile, dict):
        raise ValueError(f'profile {j}: a dict like ProfileDataLoader.load_profile_data_all()[0], not '
                         f'{type(profile).__name__}')
    model = profile.get('model')
    if not isinstance(model, dict):
        raise ValueError(f"profile {j}: no 'model' section")
    for field in _MODEL_FIELDS:
        if field not in model:
            raise ValueError(f"profile {j}: the 'model' section has no {field!r}")
    for name in type_names:
        if not isinstance(profile.get(f'DeviceType.{name}'), dict):
            raise ValueError(f'profile {j}: no DeviceType.{name} entry for device type {name} of the cluster')


def check_scenario(searched: Tuple[list, list], cluster, type_names: Sequence[str], corrected: Sequence[str],
                   j: int) -> None:
    """ValueError, naming the node and the field, unless ``cluster`` (scenario j) differs from the searched cluster
    only in bandwidth and has a finite bandwidth > 0 wherever the cost model reads one."""
    nodes, type_memory = searched
    got, got_memory = cluster_signature(cluster, type_names)
    if len(got) != len(nodes):
        raise ValueError(f'cluster {j}: {len(got)} hostfile entries, the searched cluster has {len(nodes)}')
    for k, (want, have) in enumerate(zip(nodes, got)):
        for field, a, b in zip(_NODE_FIELDS, want, have):
            if a != b:
                raise ValueError(f'cluster {j}, node {k} ({have[0]}): {field} is {b!r}, the searched cluster has {a!r}')
    for name, a, b in zip(type_names, type_memory, got_memory):
        if a != b:
            raise ValueError(f'cluster {j}, device type {name}: memory (its first clusterfile entry) is {b!r}, the '
                             f'searched cluster has {a!r}')
    fields = ('intra_bandwidth', 'inter_bandwidth') if 'Q2' in corrected else ('intra_bandwidth',)
    for k, h in enumerate(cluster.host_entries.values()):
        info = cluster.nodes_info[h['ip']]
        for field in fields:
            v = info.get(field)
            ok = isinstance(v, (int, float)) and not isinstance(v, bool) and math.isfinite(v) and v > 0
            if not ok:
                raise ValueError(f'cluster {j}, node {k} ({h["ip"]}): {field} must be a finite number > 0, not {v!r}')


def het_problem(args, gpu_cluster, profile_data, model_config, layer_load_balancer=None,
                node_sequences: Optional[Sequence[Sequence]] = None, corrected: Sequence[str] = (),
                rows_out: Optional[np.ndarray] = None, device_rows: bool = False, unbounded: bool = False,
                rows_per_stage: Optional[np.ndarray] = None):
    """Flatten the inputs of cost_het_cluster() (order of ``set(device_types)`` = quirk Q4).  ``device_rows``: the
    host lists only the compositions, the GPU writes the device-group rows (SURVEY.md 8(f)-1).  ``unbounded`` (with
    ``device_rows``): a space beyond the limits of one search is returned too, for a windowed search.
    ``rows_per_stage`` (a device listing's, metis_b200.listing): the space is only its block list
    (flatten.listed_plan_space); its windows get their records from the listing."""
    if node_sequences is None:
        node_sequences = list(permutations(set(gpu_cluster.get_device_types())))
    norm = layer_load_balancer.norm_layer_duration if layer_load_balancer is not None else None
    problem = flatten.build_problem(profile_data, gpu_cluster, model_config, args.gbs,
                                    args.max_profiled_tp_degree, args.max_profiled_batch_size, node_sequences,
                                    norm, corrected=corrected)
    space = None
    if rows_per_stage is not None:
        space = flatten.listed_plan_space(len(node_sequences), gpu_cluster.get_total_num_devices(), args.gbs,
                                          args.num_layers, rows_per_stage, corrected=corrected)
    elif device_rows and unbounded:
        space = flatten.build_device_plan_space(len(node_sequences), gpu_cluster.get_total_num_devices(), args.gbs,
                                                args.num_layers, args.min_group_scale_variance, args.max_permute_len,
                                                corrected=corrected)
        # None: a composition has more merged groups than the row kernel handles, so the rows come from the host
        device_rows = False
    if space is None:
        space = flatten.build_plan_space(len(node_sequences), gpu_cluster.get_total_num_devices(), args.gbs,
                                         args.num_layers, args.min_group_scale_variance, args.max_permute_len,
                                         corrected=corrected, rows_out=rows_out, device_rows=device_rows)
    return problem, space, [tuple(s) for s in node_sequences]


# One engine per (device, rank, world): pinned staging arena, device arena, workspace, record / detail buffers.
# cost_het_cluster() is called once per process by the reference's CLI, but a planner service calls it repeatedly;
# the buffers grow to the largest problem seen and are reused (a pinned allocation costs more than a search).
_ENGINES: Dict[Tuple, Tuple] = {}


def _engine(problem, space, device, rank: int, world: int, stride: int):
    from . import search
    dev = search._require_cuda(device)
    key = (dev.index if dev.index is not None else -1, rank, world)
    eng = _ENGINES.get(key)
    if eng is None:
        dp = search.DeviceProblem(problem, space, dev)
        searcher = search.HetSearcher(dp, rank, world, want_records=True, want_detail=True, want_ranking=False,
                                      detail_to_host=False, detail_stride=stride)
        _ENGINES[key] = (dp, searcher)
        return dp, searcher
    dp, searcher = eng
    dp.reload(problem, space)
    if searcher.detail_stride != stride:
        searcher.detail_stride = stride
        searcher.records = searcher.detail = None
    searcher.rebind()
    return dp, searcher


def release_engines() -> None:
    """Drop the cached device / pinned buffers of cost_het_cluster()."""
    _ENGINES.clear()


def cost_het_cluster(args: argparse.Namespace, gpu_cluster, profile_data: Dict, model_config: ModelConfig,
                     cost_estimator: HeteroCostEstimator, layer_load_balancer: LayerLoadBalancer,
                     node_sequences: Optional[Sequence[Sequence]] = None, device=None,
                     corrected: Sequence[str] = (), headroom: bool = False, misses: bool = False) -> HetSearchResult:
    """cost_het_cluster.py:21-50 on the GPU.  Returns the same sequence of
    (node_sequence, device_groups, strategies, batches, layer_partition, num_repartition, cost) in the
    same order (see HetSearchResult).  With torch.distributed initialised the plans are sharded over the ranks and
    every rank returns the full list.

    ``corrected`` (opt-in, default = strict parity with the reference): a subset of ('Q1', 'Q2', 'Q5', 'Q6') - 'Q1'
    drops the mislabelled one-stage block of every node sequence after the first (plan.py:144-148), 'Q2' uses the
    clusterfile's inter_bandwidth between nodes (gpu_cluster.py:56-58 returns the intra value), 'Q5' gives every
    layer to the stage holding most of its seven sub-layers so that none is dropped (load_balancer.py:293-296), 'Q6'
    takes a stage's memory demand from the profile of its own device type (load_balancer.py:41-52 uses the first
    type of the node sequence and, for mixed stages, sums a whole-cluster split).  Results of a corrected search are
    NOT the reference's; ``result.summary['corrected']`` records what was applied.

    ``headroom=True``: the search kernels also write every candidate's memory headroom (``result.headroom``), which
    ``result.ranked(k, min_headroom=...)`` and ``result.pareto()`` need; ``timings['headroom_s']`` is the host time spent
    ordering and copying it.

    ``misses=True``: the search kernels also write every out-of-memory partition attempt (``result.misses``), which
    ``result.closest_misses(k)`` and ``result.miss_detail(idx)`` need; ``summary['num_oom_attempts']`` counts them and
    ``timings['misses_s']`` is the host time spent ordering and copying them."""
    unknown = set(corrected) - {'Q1', 'Q2', 'Q5', 'Q6'}
    if unknown:
        raise ValueError(f'unknown corrections {sorted(unknown)}: choose from Q1, Q2, Q5, Q6')
    import torch
    from . import search
    t0 = time.perf_counter()
    dist = torch.distributed if (torch.distributed.is_available() and torch.distributed.is_initialized()) else None
    rank, world = (dist.get_rank(), dist.get_world_size()) if dist else (0, 1)
    dev = search._require_cuda(device)
    if node_sequences is None:
        node_sequences = list(permutations(set(gpu_cluster.get_device_types())))
    listing = _device_listing(args, gpu_cluster, len(node_sequences), dev)
    # the host or, for a large space, the GPU lists the compositions; the rows themselves are written by the GPU
    problem, space, seqs = het_problem(args, gpu_cluster, profile_data, model_config, layer_load_balancer,
                                       node_sequences, corrected=tuple(corrected), device_rows=True, unbounded=True,
                                       rows_per_stage=listing.rows_per_stage if listing is not None else None)
    if listing is None:
        windows = _het_windows(problem, space, dev, rank, world)
    else:
        windows = _listed_windows(problem, space, listing, dev, rank, world)
        if len(windows) == 1:                                 # one search: the window is the whole space
            space, windows = windows[0].space, None
    t1 = time.perf_counter()
    if windows is None:
        run, gather, candidates = _one_search(problem, space, seqs, dev, rank, world, headroom, misses)
    else:
        run, gather, candidates = _window_search(problem, windows, seqs, dev, rank, world, headroom, misses)
    failure = out = None
    try:
        out = run()
    except Exception as exc:                                  # noqa: BLE001 - re-raised below on every rank
        if not dist:
            raise
        failure = exc
    if dist:
        # a rank whose search raised must not leave the others waiting in a collective
        summary, best = search.global_exchange(out.summary if out is not None else {}, out.best if out is not None else None,
                                               dev, int(failure is not None))
        if summary['any_rank_failed']:
            raise failure if failure is not None else native.MetisNativeError('the search failed on another rank')
        if summary['global_fatal_ordinal'] < 2 ** 62:
            summary.update(fatal_ordinal=summary['global_fatal_ordinal'], fatal_code=summary['global_fatal_code'],
                           fatal_aux=summary['global_fatal_aux'])
        else:
            summary['fatal_ordinal'] = 2 ** 64 - 1
            out = gather(out, summary['records_per_rank'])
            if misses:
                summary['num_oom_attempts'] = len(out.misses)
    else:
        summary, best = out.summary, out.best
    # the reference dies at the first failing plan: nothing is returned (quirk Q8)
    search.raise_fatal(summary, problem)
    t2 = time.perf_counter()
    summary = dict(summary, num_plans=space.num_plans, corrected=tuple(sorted(corrected)),
                   num_windows=len(windows) if windows is not None else 1,
                   listing='host' if listing is None else 'device')
    cand, ranker = candidates(out, summary)
    # sorted(result, key=cost) is the CALLER's step in the reference (cost_het_cluster.py:76): its permutation is
    # computed by the device sort when ranked() is first asked for; best() needs no sort at all
    result = HetSearchResult(cand, None, summary, ranker=ranker, best_key=(best[1], best[2]) if best else None)
    result.timings = {'flatten_enumerate_s': t1 - t0, 'gpu_search_s': t2 - t1,
                      'decode_columns_s': time.perf_counter() - t2}
    if headroom:
        result.timings['headroom_s'] = out.headroom_s
    if misses:
        result.timings['misses_s'] = out.misses_s
    result._searched = cluster_signature(gpu_cluster, problem.type_names)
    result._flat_inputs = (gpu_cluster, model_config, args.gbs, args.max_profiled_tp_degree,
                           args.max_profiled_batch_size, [tuple(s) for s in node_sequences], tuple(corrected))
    result._norm_source = norm_source(profile_data)
    return result


def norm_source(profile_data) -> Optional[Tuple[str, np.ndarray]]:
    """What flatten.norm_layer_duration reads (model/load_balancer.py:22-27, quirk Q3): the profile's first-listed
    entry's name and a copy of its tp1_bs1 layer-computes, or None when it has none."""
    try:
        first = next(iter(profile_data))
        return first, np.array(profile_data[first]['tp1_bs1']['time']['layer-computes'], dtype=np.float64)
    except (StopIteration, KeyError, TypeError, ValueError):
        return None


def _one_search(problem, space, seqs, dev, rank: int, world: int, headroom: bool, misses: bool):
    """The space in one metis_het_search on the cached engine: (search, multi-rank gather of its output, (output,
    summary) -> (candidates, ranker)).  The candidates keep the detail rows on the device."""
    from . import search
    stride = 3 * int(space.blocks['num_stage'].max()) + 1
    dp, searcher = _engine(problem, space, dev, rank, world, stride)
    searcher.set_outputs(headroom, misses)
    dp.upload()

    def gather(out, counts):
        return search.gather_records(out, searcher, want_rank=False, counts=counts)

    def candidates(out, summary):
        # the row blob of the engine is rewritten by the next call: a lazy result keeps its own copy (a few MB, on the GPU)
        cand = search.Candidates(out.records, out.detail, space, seqs, detail_dev=out.detail_dev,
                                 rows_dev=dp.rows_device().clone(), problem=problem,
                                 headroom=np.array(out.headroom) if headroom else None,   # the pinned buffer is reused
                                 misses=out.misses if misses else None)   # a fresh array (HetSearcher.run)
        return cand, search.make_ranker(searcher, out.records_dev) if len(out.records) else None
    return searcher.run, gather, candidates


def _window_search(problem, windows, seqs, dev, rank: int, world: int, headroom: bool, misses: bool):
    """cost_het_cluster() for a space larger than one search: flatten.plan_windows' windows, searched in ordinal order
    (search.search_windows), merged on the host.  Returns like _one_search; the candidates keep the records only
    (search.WindowSegment)."""
    from . import search
    searcher = None

    def run():
        nonlocal searcher
        merged, _dp, searcher = search.search_windows(problem, windows, dev, rank, world, headroom=headroom,
                                                      misses=misses)
        return merged

    def candidates(merged, summary):
        cand = search.window_candidates(merged, windows, problem, seqs, searcher)
        return cand, search.make_window_ranker(searcher, merged.records, summary) if len(merged.records) else None
    return run, (lambda merged, _counts: search.gather_window_records(merged, dev)), candidates


# A space whose search needs less device memory than this (and is within the 32-bit limits of one search) is searched
# in one window without asking the device how much memory is free.
_ONE_SEARCH_BYTES = 1 << 31
# Below this budget a windowed search is refused: its windows would be so small that reloading them dominates.
_MIN_WINDOW_BYTES = 1 << 30


# A space of more compositions than this is listed on the GPU (metis_b200.listing): the host then holds one window's
# composition records at a time instead of the whole space's, and spends milliseconds instead of seconds listing them.
# Below it the host enumerator lists them (metis_enum_compositions), which is as fast for spaces of this size.
_DEVICE_LISTING_COMPS = 1 << 18


def _device_listing(args, gpu_cluster, num_node_sequences: int, dev):
    """The device listing of the space of ``args`` when it has more than _DEVICE_LISTING_COMPS compositions, else
    None (also when a composition has more merged groups than the row kernel handles: the host path decides then)."""
    from . import listing as listing_mod
    num_devices = gpu_cluster.get_total_num_devices()
    cap = min(num_devices, args.num_layers)
    if cap < 1 or cap > native.METIS_MAX_STAGES:
        return None
    variance, mpl = args.min_group_scale_variance, args.max_permute_len
    try:
        comps = flatten.count_compositions(num_devices, cap, variance, mpl)
    except native.MetisNativeError:                           # beyond the counting table (more than 8192 GPUs)
        return None
    if comps <= _DEVICE_LISTING_COMPS:
        return None
    listing = listing_mod.DeviceListing(num_devices, cap, variance, mpl, dev, max_ranges=num_node_sequences * cap + 1)
    return listing if listing.max_groups <= native.METIS_MAX_PERMUTE_GROUPS else None


def _listed_windows(problem, space, listing, dev, rank: int, world: int):
    """_het_windows for a space listed on the device: its windows (flatten.plan_listed_windows), a single one when the
    whole space is searched at once."""
    num_recs, _ = listing.size(flatten.whole_space_ranges(space))
    windows = _het_windows(problem, space, dev, rank, world, num_recs=num_recs,
                           plan=lambda budget, *model: flatten.plan_listed_windows(space, budget, *model, listing=listing))
    if windows is None:
        windows = flatten.plan_listed_windows(space, float('inf'), listing=listing)
    return windows


def _engine_bytes(key) -> int:
    """Device bytes held by the cached one-search engine ``key`` (reusable by the search being planned)."""
    eng = _ENGINES.get(key)
    if eng is None:
        return 0
    dp, searcher = eng
    held = dp._dev.numel()
    for t in (searcher.workspace, searcher.records, searcher.detail, searcher._sort_ws):
        if t is not None:
            held += t.numel() * t.element_size()
    return held


def _het_windows(problem, space, dev, rank: int, world: int, num_recs: Optional[int] = None, plan=None):
    """None when ``space`` is searched by one metis_het_search call (today's path, the cached engine untouched), else
    its windows (flatten.plan_windows, or ``plan(budget, per plan, per row byte, per record)``), sized from the device
    memory free for them.  Every rank takes the smallest budget of all ranks, so that all ranks make the same choice
    and cut the same windows.  ``num_recs``: the space's composition records when it does not hold them itself."""
    from . import search
    if space.comp_recs is None and num_recs is None:          # host rows: build_plan_space kept its limits
        return None
    if num_recs is None:
        num_recs = len(space.comp_recs)
    per_plan, per_row, per_rec, fixed = search.window_cost_model(problem)
    shard = -(-space.num_plans // world) + 128                # plans of one rank's shard, with a tile of slack
    need = shard * per_plan + int(space.rows_total_bytes) * per_row + num_recs * per_rec
    if flatten.fits_one_search(space) and need + fixed < _ONE_SEARCH_BYTES:
        return None
    key = (dev.index if dev.index is not None else -1, rank, world)
    held = _engine_bytes(key)
    if flatten.fits_one_search(space) and need + fixed <= held and world == 1:
        return None                                           # the cached engine already holds such a search
    # the cached engine's buffers are reused by a one-window search and freed for a windowed one: both count as free
    budget = search.agree_budget(search.window_budget(dev, fixed) + held, dev)
    if flatten.fits_one_search(space) and need <= budget:
        return None
    if budget < _MIN_WINDOW_BYTES:
        raise native.MetisNativeError(
            f'{max(budget, 0) / 2 ** 20:.0f} MiB of device memory are free for a search of {space.num_plans} plans; '
            f'searching it in windows needs at least {_MIN_WINDOW_BYTES >> 20} MiB')
    _ENGINES.pop(key, None)
    import torch
    torch.cuda.empty_cache()
    # a rank searches 1/world of each window's plans; the rows and composition records are whole on every rank
    if plan is not None:
        return plan(budget, per_plan / world, per_row, per_rec)
    return flatten.plan_windows(space, budget, per_plan / world, per_row, per_rec)


def cost_homo_cluster(args: argparse.Namespace, gpu_cluster, cost_estimator: HomoCostEstimator,
                      device_type: Optional[str] = None, device=None) -> List[Tuple[UniformPlan, float]]:
    """cost_homo_cluster.py:21-37 on the GPU: every gbs-matching UniformPlan is costed by
    homo_cost_kernel; plans whose profile key is missing are skipped like ``except KeyError``."""
    from . import search
    plans, problem, table, type_id = _homo_inputs(args, gpu_cluster, cost_estimator, device_type)
    cost, status = search.homo_costs(problem, type_id, table, device)
    return [(p, float(c)) for p, c, s in zip(plans, cost, status) if s != 1]


@dataclass
class HomoBreakdown:
    """What HomoCostEstimator.get_cost computes besides the cost (model/cost_estimator.py:98-138), for the plans of
    cost_homo_cluster() in its order.  ``terms[:, k]`` is search.TERM_NAMES[k]; summed left to right they give the
    plan's cost."""
    plans: List[UniformPlan]
    terms: np.ndarray                     # float64 [n, 6]
    stage_memory: np.ndarray              # float64 [n, largest pp]: sum of the profiled memory of each stage, NaN past pp
    stage_memory_str: List[List[str]]     # the reference's f'{round(m/1024/1024/1024, 2)}GB' per stage
    oom: np.ndarray                       # bool [n]: _detect_oom_occurrence


def cost_homo_breakdown(args: argparse.Namespace, gpu_cluster, cost_estimator: HomoCostEstimator,
                        device_type: Optional[str] = None, device=None) -> HomoBreakdown:
    """The cost terms, per-stage memory and OOM flag of exactly the plans cost_homo_cluster() returns, on the GPU
    (homo_breakdown_kernel)."""
    from . import search
    plans, problem, table, type_id = _homo_inputs(args, gpu_cluster, cost_estimator, device_type)
    terms, mem, status = search.homo_breakdown(problem, type_id, table, device)
    keep = status != 1
    mem = mem[keep]
    pp = table[keep, 1]
    strs = [[f'{round(float(m) / 1024 / 1024 / 1024, 2)}GB' for m in row[:k]] for row, k in zip(mem, pp.tolist())]
    return HomoBreakdown([p for p, k in zip(plans, keep) if k], terms[keep], mem, strs, status[keep] == 2)


def _homo_inputs(args, gpu_cluster, cost_estimator: HomoCostEstimator, device_type: Optional[str]):
    """(gbs-matching UniformPlans, flattened problem, their (dp, pp, tp, mbs, gbs) table, type id) of
    cost_homo_cluster()."""
    from copy import copy
    profile_data = cost_estimator.profile_data
    if device_type is None:
        device_type = next(k for k in profile_data if k.startswith('DeviceType.')).split('.', 1)[1]
    for key in profile_data[f'DeviceType.{device_type}']:
        tp = int(key[2:].split('_bs')[0])
        if tp & (tp - 1):
            raise NotImplementedError(f'profile key {key}: non power-of-two tp is not supported on the GPU path')
    plans = [copy(p) for p in UniformPlanGenerator(num_devices=gpu_cluster.get_total_num_devices(),
                                                   max_tp=args.max_profiled_tp_degree, max_gbs=args.gbs)
             if p.gbs == args.gbs]
    max_tp = max([p.tp for p in plans] + [1])
    max_bs = max([p.mbs for p in plans] + [1])
    cluster_types = [t.name for t in gpu_cluster.get_device_types()]
    problem = flatten.build_problem(profile_data, gpu_cluster, cost_estimator.model_config, args.gbs,
                                    max_tp, max_bs, [tuple(dict.fromkeys(cluster_types))])
    if device_type not in problem.type_names:
        raise KeyError(f'DeviceType.{device_type}')
    table = np.array([[p.dp, p.pp, p.tp, p.mbs, p.gbs] for p in plans], dtype=np.int32).reshape(-1, 5)
    return plans, problem, table, problem.type_names.index(device_type)
