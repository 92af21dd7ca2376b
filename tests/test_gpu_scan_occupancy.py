"""Resident CTAs per SM of the fused scan kernels on the bench's C4 shape. The kernels are built for 4 CTAs of 4 warps
per SM (__launch_bounds__(128, 4): at most 128 registers per thread), so registers allow 4 CTAs per SM; what a CTA
takes in shared memory (the per-CTA partial table, each warp's staging rings and flush staging area, the lanes'
tombstone lists) must not cut that. C4's table is 1512 words, and its simple8b-timestamp bins hold two staging rings
per warp: they are the tightest fit. The scan prints each bin's resident CTAs per SM with TSKV_DEBUG_BINS=1."""
import re

import pytest

import bench
from cnosdb_b200 import cabi, datagen
from cnosdb_b200.parallel import select_tag_subset

pytestmark = pytest.mark.gpu

REGISTER_LIMITED_CTAS = 4  # SCAN_MIN_BLOCKS in scan_kernels.cuh
C4_BINS = {9, 10, 11, 12}  # RLE ts + simple8b, simple8b ts + simple8b, RLE ts + Gorilla, simple8b ts + Gorilla values
LINE = re.compile(r"\[tskv\] bin (\d+)( \(coop\))? grid (\d+), (\d+) CTAs/SM")


@pytest.mark.parametrize("tombstones", [False, True])
def test_c4_bins_reach_register_limited_occupancy(engine, tombstones, capfd, monkeypatch):
    n_series = 20_000
    g = bench.generate_shard(n_series, 0, 1)
    pages = engine.upload_pages(g.arena, g.descs)
    if tombstones:  # the lanes' tombstone lists take 2 KB more per CTA
        pages.set_tombstones(cabi.tombstones([(0, None, datagen.TSBS_T0, datagen.TSBS_T0 + 60 * datagen.TSBS_STEP)]))
    monkeypatch.setenv("TSKV_DEBUG_BINS", "1")
    capfd.readouterr()
    res = engine.scan_aggregate(pages, bench.make_query(select_tag_subset(n_series, 10)))
    err = capfd.readouterr().err
    occ = {int(m.group(1)): int(m.group(4)) for m in LINE.finditer(err) if not m.group(2)}
    assert set(occ) == C4_BINS, err
    for b, ctas in sorted(occ.items()):
        assert ctas >= REGISTER_LIMITED_CTAS, "bin %d: %d CTAs per SM\n%s" % (b, ctas, err)
    assert res.validity.any()
    pages.close()
