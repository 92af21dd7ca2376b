"""The exact reference of tests/helpers.py for GROUP BY tags: group g's cells are exact_aggregate of the same query with
series_ids = g's members (the selected series whose slot maps to g), so every grouped result is computed from the
generated arrays like the ungrouped ones - nothing is shared with the oracle or the kernels."""
import copy

import numpy as np

from tests.helpers import ExactResult, exact_aggregate


def exact_aggregate_grouped(truth, query, group_ids, n_groups, tombstones=None, files=None):
    """ExactResult of `query` (GROUP BY bucket, not by series) with group_ids[slot] in [0, n_groups) the group of the
    slot-th selected series (series_ids order, or every series of `truth` in ascending id order). Cell c = group *
    n_buckets + bucket; a group without members reads like an empty bucket. FIRST / LAST keep the keys of the whole
    selection (ties to the lower slot, which the members keep in their order); tombstones / files: as in
    exact_aggregate."""
    assert not query.group_by_series
    slots = np.asarray(query.series_ids if query.series_ids is not None else sorted(truth), dtype=np.uint32)
    gid = np.asarray(group_ids)
    assert gid.shape == slots.shape and (gid < n_groups).all()
    nb = query.n_buckets
    res = ExactResult(query, n_groups)
    for g in range(n_groups):
        sub = copy.copy(query)
        sub.series_ids = slots[gid == g]
        sub._keep = None
        e = exact_aggregate(truth, sub, tombstones=tombstones, files=files, key_slots=slots.size)
        cells = slice(g * nb, (g + 1) * nb)
        res.values[:, cells] = e.values
        res.validity[:, cells] = e.validity
        for j in e.center:
            res.center.setdefault(j, np.zeros(n_groups * nb))[cells] = e.center[j]
            res.bound.setdefault(j, np.zeros(n_groups * nb))[cells] = e.bound[j]
        for c, sums in e.exact_sums.items():
            res.exact_sums.setdefault(c, {}).update({g * nb + k: v for k, v in sums.items()})
    return res
