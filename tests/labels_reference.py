"""The exact reference of tests/helpers.py with labelled time buckets (tskvgpu_scan_prepare_labels): edge bucket b is
[edges[b], edges[b + 1]) and aggregates into output bucket labels[b], so a row's output bucket is
labels[searchsorted(edges, t, 'right') - 1]; query.n_buckets is the number of output buckets.

exact_aggregate depends on the bucket grid through bucket_index (a row's bucket) and first_last_rel_bits (the FIRST /
LAST key budget). The functions below swap bucket_index for the labelled rule while the call runs, as
tests/edges_reference.py does for edges, so that tombstones, the overlap merge and tag groups stay exactly the code the
other scans are checked against. FIRST / LAST are refused (TSKV_ERR_UNSUPPORTED), as the scan refuses them."""
import contextlib

import numpy as np

from cnosdb_b200 import cabi
from tests import helpers
from tests.edges_reference import edge_bucket_index
from tests.group_reference import exact_aggregate_grouped


def label_bucket_index(t, edges, labels):
    """Output bucket of every timestamp (int64 array) and whether it has one: labels[b] of its edge bucket b."""
    idx, ok = edge_bucket_index(t, edges)
    lab = np.asarray(labels, dtype=np.int64)
    return np.where(ok, lab[np.clip(idx, 0, lab.size - 1)], 0), ok


@contextlib.contextmanager
def _label_rules(query, edges, labels):
    e = np.asarray(edges, dtype=np.int64)
    lab = np.asarray(labels, dtype=np.int64)
    assert query.width == 0 and lab.size == e.size - 1 and (lab < query.n_buckets).all()
    if any(c.agg_mask & (cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST) for c in query.columns):
        raise helpers.ReferenceError(cabi.TSKV_ERR_UNSUPPORTED)
    saved = helpers.bucket_index
    helpers.bucket_index = lambda t, _query: label_bucket_index(t, e, lab)
    try:
        yield
    finally:
        helpers.bucket_index = saved


def exact_aggregate_labels(truth, query, edges, labels, tombstones=None, files=None):
    """helpers.exact_aggregate over the output buckets of `labels` (query.n_buckets output buckets, query.width 0)."""
    with _label_rules(query, edges, labels):
        return helpers.exact_aggregate(truth, query, tombstones=tombstones, files=files)


def exact_aggregate_grouped_labels(truth, query, group_ids, n_groups, edges, labels, tombstones=None, files=None):
    """group_reference.exact_aggregate_grouped over the output buckets of `labels`."""
    with _label_rules(query, edges, labels):
        return exact_aggregate_grouped(truth, query, group_ids, n_groups, tombstones=tombstones, files=files)
