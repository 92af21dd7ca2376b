"""The references the multi-rank GPU tests (tests/test_gpu_multi_rank.py) pin the merge to, worked on the CPU.

1. The integer MEAN after a merge (ranks.rank_order_mean): every rank's exact sum rounded once to f64, added in gather
   order from +0.0, over the count. Hand cases where that one rounding per rank moves the result off fl(S / n).
2. k_merge_m2 restated in f64: every rank's pass-1 shift c_r = fl(S_r) / n_r, its sums of d = x - c_r and d^2, and
   Chan's merge with each rank's mean taken relative to the shift of the first rank holding the cell. It meets the exact
   M2 on the M2 arenas of the GPU tests, while the same merge on absolute means c_r + sum(d) / n_r misses 1e-9 on the
   arena near 2^63: that arena is hard for the merge, as test_gpu_variance's ill-conditioned arena is for one rank."""
import math
from fractions import Fraction

import numpy as np
import pytest

from cnosdb_b200 import cabi
from tests.ranks import layouts, rank_order_mean
from tests.test_gpu_multi_rank import far_apart_values, ill_conditioned_values, near_2_63_values
from tests.variance_reference import as_f64, exact_m2

TWO53 = 2**53


# ---- 1. the integer MEAN ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sums,n,want,exact", [
    # three ranks of 2^53 + 1: each rounds to 2^53 (to even), so the ranks' f64 sum is 3 * 2^53, not 3 * 2^53 + 3
    ([TWO53 + 1] * 3, 5, 5404319552844595.0, Fraction(3 * TWO53 + 3, 5)),
    ([TWO53 + 1] * 3, 7, 3860228252031853.5, Fraction(3 * TWO53 + 3, 7)),
    # cancellation across ranks: 2^60 + 1 rounds to 2^60 and the +1 is gone
    ([2**60 + 1, -2**60], 1, 0.0, Fraction(1)),
    ([2**60 + 1, -2**60], 3, 0.0, Fraction(1, 3)),
])
def test_rank_order_integer_mean(sums, n, want, exact):
    got = rank_order_mean(sums, n)
    assert got == want
    assert float(exact) != got  # fl(S / n), what one rank gives, differs ...
    err = abs(Fraction(got) - exact)
    assert err <= sum(abs(Fraction(float(s)) - s) for s in sums) / n + Fraction(math.ulp(got)) / 2
    # ... by the ranks' rounding of their sums over n plus the final rounding: here 0.8, 0.64, 1 and 1/3
    assert float(err) == pytest.approx({5: 0.8, 7: 9 / 14, 1: 1.0, 3: 1 / 3}[n])


def test_rank_order_follows_the_gather_order_and_empty_ranks_add_zero():
    sums = [2**60 + 1, -2**60, 7]
    assert rank_order_mean(sums, 1) == 7.0  # (2^60 - 2^60) + 7
    assert rank_order_mean(sums[::-1], 1) == 0.0  # 7 - 2^60 rounds to -2^60 (an ulp there is 256): the 7 is lost
    assert rank_order_mean([0, TWO53 + 1, 0], 2) == rank_order_mean([TWO53 + 1], 2) == 2.0**52
    assert math.copysign(1, rank_order_mean([0, 0], 1)) == 1  # +0.0, as the merge starts from +0.0


def test_layouts():
    ids = np.arange(20, dtype=np.uint32)
    for n in (3, 4, 8):
        lay = layouts(ids, n, unselected=[5, 11])
        for name, (shards, order) in lay.items():
            assert len(shards) == n and sorted(order) == list(range(n)), name
            assert np.array_equal(np.sort(np.concatenate(shards)), ids), name  # every series on exactly one rank
        assert lay["uneven"][0][0].size == 1 and lay["uneven"][0][1].size == 20 - (n - 1)
        assert lay["empty"][0][0].size == 0 and lay["unselected"][0][0].tolist() == [5, 11]
        assert lay["reversed"][1] == list(range(n))[::-1]
    assert list(layouts(ids, 1)) == ["whole"]


# ---- 2. the Chan merge in f64 ----------------------------------------------------------------------------------------
def rank_partials(xs_f64, exact_sum):
    """One rank's (n, shift, sum(d), sum(d^2)) of one cell: the shift is the pass-1 mean, fl(S) / n (S exact for an
    integer column, the f64 sum otherwise); d = x - shift, summed in f64."""
    n = len(xs_f64)
    if not n:
        return 0, 0.0, 0.0, 0.0
    c = float(exact_sum) / n
    sd = sd2 = 0.0
    for x in xs_f64:
        d = x - c
        sd += d
        sd2 += d * d
    return n, c, sd, sd2


def chan_merge(parts, relative=True):
    """k_merge_m2 on the ranks' partials: relative=True takes each rank's mean relative to the shift c of the first rank
    holding the cell; relative=False uses the absolute means c_r + sum(d) / n_r."""
    held = [p for p in parts if p[0]]
    c = held[0][1] if relative else 0.0
    n = sum(p[0] for p in held)
    mu = 0.0
    for nr, cr, sd, _ in held:
        mu += (cr - c) * nr + sd
    mu /= n
    acc = 0.0
    for nr, cr, sd, sd2 in held:
        dm = (cr - c) + sd / nr - mu
        acc += (sd2 - sd * sd / nr) + nr * dm * dm
    return acc


def cell_partials(ranks, pt):
    """ranks: every rank's raw values of one cell (i64 / u64 / f64 arrays) -> (partials, every value as f64)."""
    parts, allx = [], []
    for v in ranks:
        x = [float(e) for e in as_f64(pt, np.asarray(v).view(np.uint64))] if len(v) else []
        s = sum(int(e) for e in v) if pt != cabi.TSKV_PT_F64 else sum(x)
        parts.append(rank_partials(x, s))
        allx += x
    return parts, allx


def rel_err(got, exact):
    return abs(got - exact) / exact


def arena_cells():
    """(name, pt, [values of rank r], rtol): cells like those of the GPU tests' M2 arenas."""
    rng = np.random.default_rng(5)
    out = []
    for k in range(4):
        out.append(("steps", cabi.TSKV_PT_F64, [far_apart_values(rng, r, 12, "steps") for r in range(8)], 1e-9))
        out.append(("alternating", cabi.TSKV_PT_F64, [far_apart_values(rng, r % 2, 12, "alternating") for r in range(4)],
                    1e-9))
        for pt in (cabi.TSKV_PT_U64, cabi.TSKV_PT_I64):
            ranks = [near_2_63_values(rng, r, 25, pt) for r in range(4)]
            out.append(("near 2^63", pt, ranks, 1e-9))
            out.append(("near 2^63, rank 0 empty", pt, [ranks[0][:0]] + ranks[1:], 1e-9))
        out.append(("ill-conditioned", cabi.TSKV_PT_F64,
                    [ill_conditioned_values(rng, int(rng.integers(1, 4))) for _ in range(8)], 1e-6))
    return out


@pytest.mark.parametrize("name,pt,ranks,rtol", arena_cells())
def test_relative_chan_merge_meets_the_exact_m2(name, pt, ranks, rtol):
    parts, allx = cell_partials(ranks, pt)
    exact = exact_m2(allx)
    assert rel_err(chan_merge(parts), exact) <= rtol, name
    if name.startswith("near 2^63"):
        assert min(abs(c) for n, c, _, _ in parts if n) > 2.0**62  # every rank's mean is near 2^63 in magnitude
        assert rel_err(chan_merge(parts, relative=False), exact) > 1e-9  # absolute means lose the digits
    if name in ("steps", "alternating"):  # the between-rank term is nearly all of M2
        within = sum(sd2 - sd * sd / n for n, _, sd, sd2 in parts if n)
        assert within < 1e-6 * exact


def test_one_rank_merge_is_the_plain_m2():
    """With one rank the merge leaves sd2 - sd^2 / n, which is what k_finalize computes."""
    rng = np.random.default_rng(8)
    x = list(1e9 + rng.normal(0, 1e-3, 17))
    n, c, sd, sd2 = rank_partials(x, sum(x))
    assert chan_merge([(n, c, sd, sd2)]) == sd2 - sd * sd / n
