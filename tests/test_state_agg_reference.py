"""tests/state_agg_reference.py against the reference's compact_state_agg answers (tests/golden/compact_state_agg_slt.json:
duration_in.slt on the states table, the DurationStates unit fixture of state_agg_data.rs) and against a split of the rows
into random batches, as the accumulator's update_batch receives them."""
import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import PushedAggregate, QueryOption, duration_in
from tests.helpers import random_arena
from tests.state_agg_reference import exact_state_maps, fold, load_golden, selected_points, update_batch_reference


def test_golden_slt_answers():
    g = load_golden()
    rows = [(r["time"], r["code"]) for r in g["states"]["rows"]]
    m = fold(sorted(rows))
    assert len(g["answers"]) == 2
    for a in g["answers"]:
        assert duration_in(m, a["code"]) == a["expected"], a["src"]
    assert duration_in(m, 99) == 0  # an absent state


def test_golden_unit_fixture():
    u = load_golden()["unit"]
    m = fold([(t, s) for t, s in u["points"]])
    assert m == {s: d for s, d in u["durations"]} == {111: 1003, 222: 97, 333: 800}


def test_fold_edges():
    assert fold([]) == {}
    assert fold([(5, 7)]) == {7: 0}  # finalize: the last state's 0 entry
    assert fold([(5, None), (9, 1)]) == {None: 4, 1: 0}  # NULL is a state
    assert fold([(0, 1), (3, 2), (4, 1)]) == {1: 3, 2: 1}  # the last state has an entry already
    assert fold([(0, 1), (0, 2)]) == {1: 0, 2: 0}  # a pair of equal times still makes an entry


@pytest.mark.parametrize("seed", range(20))
def test_random_batch_splits(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 60))
    t = rng.choice(np.arange(10_000), n, replace=False)
    states = rng.integers(0, 4, n)
    rows = [(int(a) if rng.random() > 0.1 else None, (int(s) if s else None)) for a, s in zip(t, states)]
    cuts = sorted({0, n, *rng.integers(0, n + 1, 4).tolist()})
    expect = fold(sorted(((a, s) for a, s in rows if a is not None), key=lambda r: r[0]))
    assert update_batch_reference(rows, cuts) == expect
    perm = rng.permutation(n)
    assert update_batch_reference([rows[i] for i in perm], cuts) == expect  # the input order does not matter


def test_selection_keeps_nulls():
    rng = np.random.default_rng(3)
    _, _, truth = random_arena(rng, n_series=3, n_points=50, fields=((1, cabi.TSKV_PT_I64),), null_frac=0.3)
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, ["compact_state_agg"])], width=0, n_buckets=1,
                    group_by_series=True)
    pts = selected_points(truth, q, 1, cabi.TSKV_PT_I64)
    for slot, sid in enumerate(sorted(truth)):
        ts, cols = truth[sid][0]
        v, ok = cols[1]
        assert pts[slot] == [(int(a), int(x) if k else None) for a, x, k in zip(ts, v, ok)]
    maps = exact_state_maps(truth, q, 1, cabi.TSKV_PT_I64, 3)
    for slot in range(3):
        assert sum(maps[slot].values()) == pts[slot][-1][0] - pts[slot][0][0]
