"""TSKV_UPLOAD_VERIFY_ON_READ for pages resident in HBM: every scan re-checks the CRC32 of the pages it reads (the
reference's Page::crc_validation on every read, tsm/reader.rs:259), in front of each bin's fused kernel; a mismatch
outranks whatever the decoders made of the corrupt page."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption, TskvError
from oracle import pyoracle as orc
from tests.helpers import assert_results_equal, bucket_spec

pytestmark = pytest.mark.gpu


def test_verify_on_read_in_hbm(engine):
    g = datagen.generate(3000, n_fields=2, n_points=600, value_kind=datagen.MIXED, seed=21, jitter_permille=300, jitter_max=999_999,
                         null_page_permille=100, null_row_permille=50)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1_000_000, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP + 1_000_000, w)
    sel = np.arange(0, 3000, 3, dtype=np.uint32)
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, ["count", "sum", "min", "max", "mean"]),
                     PushedAggregate(3, cabi.TSKV_PT_F64, ["count", "sum", "max"])],
                    series_ids=sel, width=w, first_bucket_start=fbs, n_buckets=nb)
    exp = orc.scan_aggregate(g.arena, g.descs, q, n_threads=8)
    pages = engine.upload_pages(g.arena, g.descs, verify_crc=True, verify_on_read=True)
    scan = engine.prepare(pages, q)
    for _ in range(4):  # the second enqueue onwards replays the captured graph (CRC checks on the bin streams inside it)
        scan.enqueue()
        assert_results_equal(scan.finalize(), exp, what="verify on read, clean pages")
    scan.close()
    pages.close()
    # corruption that the upload did not look at (verify_crc=False) is caught by the first scan that reads the page -
    # in a value stream (the decoder may also choke on it: the CRC error wins) and in a time page
    for kind, series in (("value", 6), ("time", 9)):
        arena = g.arena.copy()
        pt = cabi.TSKV_PT_TIME if kind == "time" else cabi.TSKV_PT_I64
        victim = next(i for i, d in enumerate(g.descs) if d["series_id"] == series and d["phys_type"] == pt)
        arena[int(g.descs[victim]["offset"]) + int(g.descs[victim]["size"]) - 5] ^= 0x5A
        bad = engine.upload_pages(arena, g.descs, verify_crc=False, verify_on_read=True)
        with pytest.raises(TskvError) as e:
            engine.scan_aggregate(bad, q)
        assert e.value.status == cabi.TSKV_ERR_CRC_MISMATCH and e.value.page == victim
        # a series the scan does not select is not read, so its corruption goes unnoticed (like the reference)
        q_other = QueryOption(q.columns, series_ids=np.array([1, 2, 4, 5], dtype=np.uint32), width=w, first_bucket_start=fbs, n_buckets=nb)
        engine.scan_aggregate(bad, q_other)
        bad.close()
