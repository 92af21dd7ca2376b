"""tests/mode_reference.py against the reference's mode.slt and approx_distinct.slt answers (tests/golden/mode_slt.json), a
collections.Counter brute force on random inputs, its tie rule, and f64 -0.0 / +0.0,
NaN payloads and infinities under bit equality."""
from collections import Counter

import numpy as np

from cnosdb_b200 import cabi
from tests.mode_reference import golden_cases, golden_refused, mode_bits, order_key

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64


def f64(bits):
    return np.uint64(bits).view(np.float64)


def test_random_against_counter():
    rng = np.random.default_rng(7)
    for trial in range(300):
        pt = (I64, U64, F64)[trial % 3]
        n = int(rng.integers(0, 40))
        pool = rng.integers(-5, 6, size=8)
        vals = [float(x) / 2 if pt == F64 else (int(x) if pt == I64 else int(x) & 0xFFFFFFFFFFFFFFFF)
                for x in rng.choice(pool, size=n)]
        m, d = mode_bits(vals, pt)
        bits = [int(np.float64(v).view(np.uint64)) if pt == F64 else int(v) & 0xFFFFFFFFFFFFFFFF for v in vals]
        c = Counter(bits)
        assert d == len(c)
        if not n:
            assert m is None
            continue
        assert c[m] == max(c.values())


def test_ties_take_the_smallest_value():
    assert mode_bits([3, -2, 3, -2, 7], I64) == ((-2) & 0xFFFFFFFFFFFFFFFF, 3)
    assert mode_bits([2**63, 5, 2**63, 5], U64) == (5, 2)
    assert mode_bits([1.5, -1.5], F64) == (int(np.float64(-1.5).view(np.uint64)), 2)
    assert mode_bits([9], I64) == (9, 1)
    assert mode_bits([], F64) == (None, 0)


def test_f64_specials_by_bits():
    pz, nz = 0x0000000000000000, 0x8000000000000000
    nan_a, nan_b, nnan = 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000
    pinf, ninf = 0x7FF0000000000000, 0xFFF0000000000000
    # -0.0 and +0.0 are two values; -0.0 orders first
    assert mode_bits([f64(pz), f64(nz)], F64) == (nz, 2)
    assert mode_bits([f64(pz), f64(pz), f64(nz)], F64) == (pz, 2)
    # NaNs are equal only with equal bits; a negative NaN orders before everything
    assert mode_bits([f64(nan_a), f64(nan_b), f64(nan_a)], F64) == (nan_a, 2)
    assert mode_bits([f64(nan_a), f64(nnan), f64(ninf), f64(pinf)], F64) == (nnan, 4)
    assert order_key(ninf, F64) < order_key(nz, F64) < order_key(pz, F64) < order_key(pinf, F64) < order_key(nan_a, F64)


def test_reference_reproduces_the_goldens():
    """mode.slt's func_tbl / func_tb3 answers and approx_distinct.slt's distinct counts, from the rows the slt files
    insert (mode.slt's ties do not arise: each answer is a unique mode)."""
    cases = golden_cases()
    assert len(cases) == 8
    for c in cases:
        got = []
        for vals in c.groups().values():
            m, d = mode_bits(vals, c.pt)
            got.append(d if c.kind == "distinct" else bits_to_value(m, c.pt))
        assert got == c.expected, (c.what, got, c.expected)
    assert {t for _, t, _ in golden_refused()} == {"TIME", "BOOLEAN", "STRING", "GEOMETRY"}


def bits_to_value(bits, pt):
    if pt == F64:
        return float(f64(bits))
    if pt == I64:
        return bits - (1 << 64) if bits >> 63 else bits
    return bits
