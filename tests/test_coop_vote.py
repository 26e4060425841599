"""The vote of the chain kernel's balancer run (CoopEvaluator::balance_coop) at the boundaries of how it divides the
layers: each lane takes a block of ceil(L / 32) consecutive layers, searches the interval ends once for the block's
first sub-layer and walks on from there.  L on both sides of the multiples of 32 where the block length changes, L
that leaves trailing lanes without layers, S on both sides of the multiples of 32; rows whose stages end inside,
beyond and in the middle block / reserved tail.

Every partition must equal the oracle's: on the host build on one lane (blocks visited forward and in reverse), on the
GPU on WarpCoop in every scratch tier.
"""
import collections
import random

import pytest

import balancer_cases as bc
import devsim_util as ds

SHAPES_L = (31, 32, 33, 40, 64, 65, 96, 97, 160, 224, 225, 255)
SHAPES_S = (4, 31, 32, 33, 34, 63, 64, 65, 95, 96, 97, 127, 128)
FORWARD_SHARE = 0.9        # rows of >= 4 stages whose forward state comes from the predicted pass


def vote_cases(tier, seed=31):
    """Per L: rows of every S in SHAPES_S that fits the tier and L.  Kind 0: random capacities at 0.97 / 1.0 / 1.05
    of the demand; kind 1: the same with up to three stages 10-50 times their neighbours' size (long intervals that
    cross several blocks); kind 2: under-subscribed (0.6), which leaves a middle block and the tail."""
    rng = random.Random(seed)
    out = []
    for L in SHAPES_L:
        if L > tier[1]:
            continue
        lc = bc.rand_lc(rng, L)
        rows = []
        for S in SHAPES_S:
            if S > min(L, tier[0]):
                continue
            for kind in range(3):
                capa = [rng.random() + 0.05 for _ in range(S)]
                if kind == 1:
                    for s in rng.sample(range(S - 1), min(S - 1, 3)):
                        capa[s] *= rng.choice([10, 30, 50])
                scale = 0.6 if kind == 2 else rng.choice([0.97, 1.0, 1.05])
                rows.append([c * scale for c in bc.normalise(capa)])
        out.append((L, lc, rows))
    return out


def check_vote(tier, run, policies):
    """Oracle parity of every row under each policy, and the paths the first policy took."""
    seen = collections.Counter()
    for L, lc, rows in vote_cases(tier):
        want = [bc.oracle(L, lc, capa) for capa in rows]
        for policy in policies:
            got = run(policy, rows, lc, L)
            for i, (part, rc) in enumerate(want):
                assert (got.part[i], got.rc[i]) == (part, rc), (policy, tier, L, len(rows[i]))
            if policy == policies[0]:
                for i, capa in enumerate(rows):
                    if len(capa) >= 4:
                        seen['rows'] += 1
                        seen['forward'] += not (got.took('seq_forward')[i] or got.took('verify_failed')[i])
                for path in ('middle', 'tail'):
                    seen[path] += sum(got.took(path))
    assert seen['forward'] >= FORWARD_SHARE * seen['rows'], dict(seen)
    assert seen['middle'] > 0 and seen['tail'] > 0, dict(seen)


@pytest.mark.parametrize('tier', ds.TIERS)
def test_vote_blocks_on_host(tier):
    """balance_coop on one lane, blocks forward and in reverse, and the serial form, against the oracle."""
    check_vote(tier, lambda pol, rows, lc, L: ds.host_balance(pol, tier, rows, lc, L), ('coop', 'coop_reverse', 'serial'))


@pytest.mark.gpu
@pytest.mark.parametrize('tier', ds.TIERS)
def test_vote_blocks_on_gpu(tier):
    """balance_coop on WarpCoop in scratch tier `tier` against the oracle."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    check_vote(tier, lambda pol, rows, lc, L: ds.device_balance(pol, tier, rows, lc, L), ('coop',))
