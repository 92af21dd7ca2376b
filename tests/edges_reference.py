"""The exact reference of tests/helpers.py with explicit time-bucket edges (tskvgpu_scan_prepare_edges): bucket b is
[edges[b], edges[b + 1]), a row's bucket is searchsorted(edges, t, 'right') - 1, and the FIRST / LAST key budget is
bits(longest bucket) + slot bits.

exact_aggregate depends on the bucket grid in two places only: bucket_index (a row's bucket) and first_last_rel_bits
(the key budget). The functions below swap those two rules of tests.helpers for the edge rules while the call runs, so
that FIRST / LAST runs and ties, tombstones, the overlap merge and tag groups stay exactly the ones the tumbling scans
are checked against."""
import contextlib

import numpy as np

from tests import helpers
from tests.group_reference import exact_aggregate_grouped


def edge_bucket_index(t, edges):
    """Bucket of every timestamp (int64 array) and whether it has one: [edges[b], edges[b + 1]), floor at every time."""
    e = np.asarray(edges, dtype=np.int64)
    idx = np.searchsorted(e, np.asarray(t, dtype=np.int64), side="right") - 1
    return idx, (idx >= 0) & (idx < e.size - 1)


def edge_rel_bits(edges):
    """Bits of the time part of the FIRST / LAST tie-break keys: rel = t - edges[b] + 1 <= the longest bucket."""
    return helpers.bits_for(max(int(b) - int(a) for a, b in zip(edges[:-1], edges[1:])))


@contextlib.contextmanager
def _edge_rules(query, edges):
    e = np.asarray(edges, dtype=np.int64)
    assert query.n_buckets == e.size - 1 and query.width == 0
    saved = helpers.bucket_index, helpers.first_last_rel_bits
    helpers.bucket_index = lambda t, _query: edge_bucket_index(t, e)
    helpers.first_last_rel_bits = lambda _truth, _query: edge_rel_bits(e)
    try:
        yield
    finally:
        helpers.bucket_index, helpers.first_last_rel_bits = saved


def exact_aggregate_edges(truth, query, edges, tombstones=None, files=None, key_slots=None):
    """helpers.exact_aggregate over the buckets of `edges` (query.n_buckets = len(edges) - 1, query.width 0)."""
    with _edge_rules(query, edges):
        return helpers.exact_aggregate(truth, query, tombstones=tombstones, files=files, key_slots=key_slots)


def exact_aggregate_grouped_edges(truth, query, group_ids, n_groups, edges, tombstones=None, files=None):
    """group_reference.exact_aggregate_grouped over the buckets of `edges`."""
    with _edge_rules(query, edges):
        return exact_aggregate_grouped(truth, query, group_ids, n_groups, tombstones=tombstones, files=files)
