"""Seeded inputs of LayerComputeBalancer.run built to take the balancer's rarely taken paths, shared by the CPU and
GPU tests of the balancer forms (tests/test_balancer_forms.py).

A case is (family, L, lc, rows, target): `lc` holds the normalised layer weights (its length is norm_len, which may
differ from L), `rows` the capacity rows, `target` the BalancerPath (tests/devsim_util.PATHS) the family is built to
reach, or None.  Every generator is deterministic for a given seed and tier (MAXS, MAXL).
"""
import math
import random

from oracle import metis_oracle as orc

H = 7
INDEX, SCRATCH = 3, 5            # METIS_FATAL_INDEX, METIS_FATAL_SCRATCH (include/metis_b200.h)
SHAPES_S = (1, 2, 3, 4, 5, 31, 32, 33, 34, 63, 64, 65, 66, 95, 96, 97, 127, 128)
SHAPES_L = (2, 3, 7, 8, 36, 37, 127, 128, 129, 254, 255)


def normalise(v):
    t = sum(v)
    return [x / t for x in v]


def rand_lc(rng, L):
    return normalise([0.01 + rng.random() for _ in range(L)])


def demands(lc, L):
    """expand_lc_demand: the demand of every sub-layer, lc[j // 7] / 7."""
    return [lc[j // H] / H for j in range(H * L)]


def close(c, d, a, lim):
    """Where the reference's forward compare-and-subtract chain closes a stage of capacity c that starts at a:
    (first sub-layer not taken, residual capacity)."""
    j = a
    while j < lim and c > d[j]:
        c -= d[j]
        j += 1
    return j, c


def rand_rows(rng, n, smin, smax, scale=1.0):
    rows = []
    for _ in range(n):
        S = rng.randint(smin, smax)
        capa = [rng.random() ** rng.choice([1, 3]) + 1e-3 for _ in range(S)]
        rows.append([c * scale for c in normalise(capa)])
    return rows


def knife_row(rng, S, d, lim, stats):
    """Every stage but the last gets the demands of an interval [a, b] added up in reverse (d[b] + ... + d[a]), nudged
    by -2 .. +2 ulps: whether the reference's chain closes the stage at b or one sub-layer earlier or later is decided
    by the last bits, where the running-sum prediction of the forward pass is least reliable.  The last stage gets
    the rest.  `stats` counts the stages the reference closes at b, before b (the capacity falls short) and after b
    (it goes on), and the closing compares that met a residual exactly equal to the demand."""
    a, caps = 0, []
    for s in range(S - 1):
        if a >= lim - 1:
            caps.append(d[lim - 1] * rng.choice([0.5, 1.0, 2.0]))
            continue
        span = max(1, 2 * (lim - a) // (S - 1 - s))
        b = min(a + rng.randint(0, span), lim - 1)
        c = d[b]
        for j in range(b - 1, a - 1, -1):
            c += d[j]
        k = rng.choice([-2, -1, 0, 0, 1, 2])
        for _ in range(abs(k)):
            c = math.nextafter(c, math.inf if k > 0 else -math.inf)
        caps.append(c)
        j, rest = close(c, d, a, lim)
        if j < lim:
            stats['at' if j == b else 'early' if j < b else 'late'] += 1
            stats['eq'] += rest == d[j]
            a = j + 1
        else:
            a = lim
    caps.append(max(1e-3, 1.0 - sum(caps)))
    return caps


def knife_cases(tier, seed=21, per=40):
    rng = random.Random(seed)
    stats = {'at': 0, 'early': 0, 'late': 0, 'eq': 0}
    out = []
    for L in (24, 96, min(200, tier[1] - 1)):
        lc = rand_lc(rng, L)
        d = demands(lc, L)
        rows = [knife_row(rng, rng.randint(4, min(L, tier[0])), d, H * L - 1 - H, stats) for _ in range(per)]
        out.append(('knife', L, lc, rows, 'verify_failed'))
    return out, stats


def irregular_cases(tier, seed=22, per=40):
    """Stages with an empty forward interval: capacity 0.0 / -0.0, exactly the first demand the stage meets (c > d
    fails at once), or below it; single stages and runs of them, at the first and the last stage too."""
    rng = random.Random(seed)
    out = []
    for L in (12, 64, min(150, tier[1] - 1)):
        lc = rand_lc(rng, L)
        d = demands(lc, L)
        lim = H * L - 1 - H
        rows = []
        for r in range(per):
            S = rng.randint(3, min(L, tier[0]))
            capa = [c * rng.choice([1.0, 1.0, 0.97, 1.05]) for c in normalise([rng.random() + 0.05 for _ in range(S)])]
            empty = set()
            if r % 4 == 0:
                empty.update(range(rng.randint(1, max(1, S // 3))))                 # run at the first stage
            if r % 4 == 1:
                empty.update(range(S - rng.randint(1, max(1, S // 3)), S))          # run ending at the last stage
            for _ in range(rng.randint(1, 3)):
                a = rng.randrange(S)
                empty.update(range(a, min(S, a + rng.randint(1, 4))))
            a = 0
            for s in range(S):
                if s in empty:
                    kind = rng.choice(['zero', 'negzero', 'exact', 'below'])
                    dj = d[min(a, lim - 1)]
                    capa[s] = {'zero': 0.0, 'negzero': -0.0, 'exact': dj, 'below': dj * 0.5}[kind]
                if s < S - 1 and a < lim:
                    j, _ = close(capa[s], d, a, lim)
                    a = j + 1 if j < lim else lim
            rows.append(capa)
        out.append(('irregular', L, lc, rows, 'irregular'))
    return out


def tie_cases(tier, seed=23, per=40):
    """Equal capacities (ties in the middle block and at the skipped sub-layers' picks), +0.0 against -0.0, capacities
    that go negative in an under-subscribed middle block, and one dominant layer next to many tiny ones (a long
    middle block)."""
    rng = random.Random(seed)
    out = []
    for L in (16, min(120, tier[1] - 1), min(255, tier[1] - 1)):
        uniform = [1.0 / L] * L
        heavy = [0.3 / (L - 1)] * L
        heavy[L // 3] = 0.7
        for lc in (uniform, normalise(heavy)):
            rows = []
            for r in range(per):
                S = rng.randint(2, min(L, tier[0]))
                scale = rng.choice([1.0, 0.97, 0.9, 0.75, 0.6])
                if r % 3 == 0:
                    capa = [scale / S] * S
                elif r % 3 == 1:
                    capa = [c * scale for c in normalise([rng.choice([1.0, 2.0]) for _ in range(S)])]
                else:
                    capa = [c * scale for c in normalise([rng.random() + 0.05 for _ in range(S)])]
                    for s in rng.sample(range(S), min(S, 3)):
                        capa[s] = rng.choice([0.0, -0.0])
                rows.append(capa)
            out.append(('ties', L, lc, rows, 'middle'))
    return out


def zero_demand_cases(tier, seed=24, per=30):
    """Layers of weight 0.0 (first, last, single and in runs): repeated entries of the running sum and `c > 0.0`
    compares."""
    rng = random.Random(seed)
    out = []
    for L in (9, 48, min(130, tier[1] - 1)):
        lc = [0.01 + rng.random() for _ in range(L)]
        lc[0] = lc[-1] = 0.0
        for _ in range(max(1, L // 8)):
            a = rng.randrange(L)
            for r in range(a, min(L, a + rng.randint(1, 5))):
                lc[r] = 0.0
        lc = normalise(lc)
        rows = rand_rows(rng, per, 1, min(L, tier[0]))
        d = demands(lc, L)
        rows += [knife_row(rng, rng.randint(4, min(L, tier[0])), d, H * L - 1 - H,
                           dict.fromkeys(('at', 'early', 'late', 'eq'), 0)) for _ in range(per // 2)]
        out.append(('zero_demand', L, lc, rows, None))
    return out


def shape_cases(tier, seed=25):
    """S x L across the 32-lane bases of the skipped sub-layers' carry and the group boundaries of first_ge, within
    the tier; norm_len below L (every form must raise IndexError's code) and above it."""
    rng = random.Random(seed)
    out = []
    for L in SHAPES_L:
        if L > tier[1] - 1 and L > 255:
            continue
        if L > tier[1]:
            continue
        lc = rand_lc(rng, L)
        rows = []
        for S in SHAPES_S:
            if S <= tier[0]:
                rows += rand_rows(rng, 2, S, S, rng.choice([1.0, 0.97, 1.05]))
        out.append(('shapes', L, lc, rows, 'seq_forward'))
    for L in (8, 37, min(129, tier[1])):
        rows = rand_rows(rng, 6, 1, min(L, tier[0]))
        out.append(('norm_len_short', L, rand_lc(rng, L - 1), rows, None))
        out.append(('norm_len_long', L, rand_lc(rng, L + 3), rows, None))
    return out


def subscription_cases(tier, seed=26, per=40):
    """Capacities summing to 0.97, 1.0 and 1.05 of the demand, and rows whose first stages take everything up to the
    reserved tail with stages to spare."""
    rng = random.Random(seed)
    out = []
    for L in (20, min(100, tier[1] - 1), min(254, tier[1] - 1)):
        lc = rand_lc(rng, L)
        rows = []
        for scale in (0.97, 1.0, 1.05):
            rows += rand_rows(rng, per // 2, 1, min(L, tier[0]), scale)
        for _ in range(per // 2):
            S = rng.randint(3, min(L, tier[0]))
            capa = [rng.random() * 0.01 for _ in range(S)]
            capa[rng.randrange(S - 1)] = rng.choice([1.0, 1.5, 3.0])
            rows.append(capa)
        out.append(('subscription', L, lc, rows, 'tail'))
    return out


def lockstep_cases(tier, seed=27):
    """Warps of 32 rows with one stage count each (the bulk round sorts its lists by stage count), mixing knife-edge
    rows, empty stages, rows that run into the reserved tail and under-subscribed rows with a middle block."""
    rng = random.Random(seed)
    out = []
    for L in (40, min(127, tier[1] - 1)):
        lc = rand_lc(rng, L)
        d = demands(lc, L)
        lim = H * L - 1 - H
        rows = []
        for S in (4, 9, 33, min(L, tier[0])):
            for lane in range(32):
                kind = lane % 4
                if kind == 0:
                    rows.append(knife_row(rng, S, d, lim, dict.fromkeys(('at', 'early', 'late', 'eq'), 0)))
                elif kind == 1:
                    capa = normalise([rng.random() + 0.05 for _ in range(S)])
                    for s in rng.sample(range(S), min(S - 1, 2)):
                        capa[s] = 0.0
                    rows.append(capa)
                elif kind == 2:
                    capa = [0.002] * S
                    capa[0] = 2.0
                    rows.append(capa)
                else:
                    rows.append([c * 0.8 for c in normalise([rng.random() + 0.05 for _ in range(S)])])
        out.append(('lockstep_mix', L, lc, rows, 'middle'))
    return out


def all_cases(tier):
    knife, stats = knife_cases(tier)
    return knife + irregular_cases(tier) + tie_cases(tier) + zero_demand_cases(tier) + shape_cases(tier) + \
        subscription_cases(tier) + lockstep_cases(tier), stats


def oracle(L, lc, capa):
    """(partition, 0) from the oracle, or (None, METIS_FATAL_*) for the exception the reference raises."""
    try:
        return orc.layer_compute_balance(len(capa), L, list(capa), lc), 0
    except IndexError:
        return None, INDEX
    except TypeError:                   # get_proper_stage found no stage: range(lo, hi + 1) empty, capa[None]
        return None, SCRATCH
