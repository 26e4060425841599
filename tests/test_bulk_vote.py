"""The vote of balance_run (the bulk round's and the replay kernels' layer balancer) against the oracle.

balance_run takes the stage of a forward sub-layer from the interval ends fe[] and the placed skipped sub-layers
(lstk), and reads the per-sub-layer map in subw only for the middle block.  On the families of tests/balancer_cases.py
every partition (or fatal code) must equal the oracle's: on the CPU in the Serial form of the host build, on the GPU
in the Serial and Lockstep forms of the device build in every scratch tier.  The notes of the first form must show
that the inputs reach the interval-end vote, the middle block (subw) and the irregular leftovers.
"""
import collections
import functools

import pytest

import balancer_cases as bc
import devsim_util as ds

VOTE_ENDS = 6              # BalancerPath kPathVoteEnds (metis_eval.cuh)


@functools.lru_cache(maxsize=None)
def expected(tier):
    cases, _stats = bc.all_cases(tier)
    return cases, [[bc.oracle(L, lc, capa) for capa in rows] for _f, L, lc, rows, _t in cases]


def check_vote(tier, run, policies):
    cases, wants = expected(tier)
    seen = collections.Counter()
    for (family, L, lc, rows, _target), want in zip(cases, wants):
        for policy in policies:
            got = run(policy, rows, lc, L)
            for i, (part, rc) in enumerate(want):
                assert (got.part[i], got.rc[i]) == (part, rc), (policy, tier, family, L, len(rows[i]))
            if policy == policies[0]:
                seen['rows'] += len(rows)
                seen['vote_ends'] += sum(bool(n >> VOTE_ENDS & 1) for n in got.notes)
                seen['middle'] += sum(got.took('middle'))
                seen['irregular'] += sum(got.took('irregular'))
                seen['both'] += sum(bool(n >> VOTE_ENDS & 1) and bool(n >> ds.PATHS['middle'] & 1) for n in got.notes)
    for path in ('vote_ends', 'middle', 'irregular', 'both'):
        assert seen[path] > 0, (tier, dict(seen))
    return seen


@pytest.mark.parametrize('tier', ds.TIERS)
def test_bulk_vote_on_host(tier):
    """balance_run in the Serial form of the host build against the oracle."""
    check_vote(tier, lambda pol, rows, lc, L: ds.host_balance(pol, tier, rows, lc, L), ('serial',))


@pytest.mark.gpu
@pytest.mark.parametrize('tier', ds.TIERS)
def test_bulk_vote_on_gpu(tier):
    """balance_run in the Lockstep form (32 rows per warp, as in het_first_kernel) and the Serial form on the GPU."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    check_vote(tier, lambda pol, rows, lc, L: ds.device_balance(pol, tier, rows, lc, L), ('lockstep', 'serial'))
