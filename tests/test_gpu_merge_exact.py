"""The overlap merge of chunk files (merge_kernels.cuh) against the exact reference (tests/helpers.py), bit for bit, on
the merge arena of tests/exact_arenas.py: 2 to 8 files per series with duplicate times inside chunks (a run of 320),
overlap chains, touching and just-separated chunks, a newest chunk without a column or with NULLs, raw "memcache"
chunks, merged NULL rows on bucket starts / ends, times at the i64 limits; with predicates, row and column tombstones,
by bucket, by series, by tags, unbucketed, sliding windows, a host-resident page set and a two-shard exchange."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import exact_arenas as ea
from tests.helpers import assert_matches_exact
from tests.ranks import sharded_scans

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def merge_set():
    arena, descs, truth, files = ea.merge_arena()
    return arena, descs, truth, files, ea.merge_tombstones(truth)


def _scan(engine, pages, q, extra):
    return engine.scan_aggregate(pages, q, slide=extra.get("slide"), group_ids=extra.get("group_ids"),
                                 n_groups=extra.get("n_groups"))


@pytest.mark.parametrize("tombstoned", [False, True])
def test_merge_matches_the_exact_reference(engine, merge_set, tombstoned):
    arena, descs, truth, files, tombs = merge_set
    tombs = tombs if tombstoned else None
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    host = engine.upload_pages(arena, descs, host_resident=True)
    host.set_chunk_files(files)
    if tombstoned:
        pages.set_tombstones(tombs)
        host.set_tombstones(tombs)
    queries = ea.merge_queries(truth) + ([] if tombstoned else [("sliding",) + ea.merge_sliding_query()])
    for name, q, extra in queries:
        what = "%s tombstones=%s" % (name, tombstoned)
        exp = ea.expected(truth, q, extra, tombstones=tombs, files=files)
        assert_matches_exact(_scan(engine, pages, q, extra), exp, what=what)
        if not (extra or q.predicates or tombstoned):  # (as in test_gpu_overlap_merge.py)
            _, pts = orc.scan_aggregate(arena, descs, q, chunk_files=files, tombstones=tombs, return_points=True)
            assert engine.counters()["points_decoded"] == pts, what
        assert_matches_exact(_scan(engine, host, q, extra), exp, what=what + " host-resident")
    host.close()
    pages.close()


def test_merge_through_a_two_shard_exchange(engine, merge_set):
    arena, descs, truth, files, tombs = merge_set
    for name, q, _ in ea.merge_queries(truth)[:2]:
        ids = q.series_ids
        for tb in (None, tombs):
            exp = ea.expected(truth, q, {}, tombstones=tb, files=files)
            for got in sharded_scans(engine, arena, descs, q, (ids[ids % 2 == 0], ids[ids % 2 == 1]), files=files,
                                     tombstones=tb):
                assert_matches_exact(got, exp, what="%s tombstones=%s 2-shard exchange" % (name, tb is not None),
                                     int_mean=False)
