"""Multi-rank scans on one device: every rank's series shard is its own page set, scanned with the global query, and the
ranks' partial states are merged as a multi-GPU run merges them.

  RankScans.gather     the all-gather merge: the ranks' exchange regions concatenated in a given rank order (what one
                       ncclAllGather hands every rank), then tskvgpu_scan_merge_gathered and finalize on every rank.
  RankScans.allreduce  the all-reduce contract of parallel.allreduce_sections, restated on host copies of every rank's
                       tskvgpu_scan_partials sections: snapshot the FIRST / LAST keys, wrap-add the integer sums, add the
                       f64 sums in rank order from +0.0 (k_merge_gathered's order), MIN / MAX the keys, write the reduced
                       sections back, mask the values whose key lost, sum them, finalize.

A rank whose shard holds no page (zero descriptors) takes part like any other. Layouts (lists of series ids per rank,
plus the gather order) are built by `layouts`."""
import copy

import numpy as np

from cnosdb_b200 import cabi, parallel


def with_series(q, ids):
    q = copy.copy(q)
    q.series_ids = np.asarray(ids, dtype=np.uint32)
    q._keep = None
    return q


def multi_rank(q):
    q = copy.copy(q)
    q.multi_rank = True
    q._keep = None
    return q


def layouts(all_ids, n, unselected=()):
    """{name: (shards, gather order)} of n ranks over the series `all_ids`; n == 1 gives the one layout "whole".
      contiguous  parallel.shard_range over all_ids (what bench.py does)
      mod         id % n
      uneven      rank 0 holds one series, ranks 2.. one each, rank 1 the rest
      unselected  rank 0 holds only the series of `unselected` (none the query selects), the others contiguous shares
                  of the rest (only with `unselected`)
      empty       rank 0 holds no page at all, the others contiguous shares
      reversed    the contiguous shards, gathered in reverse rank order"""
    ids = np.asarray(sorted(all_ids), dtype=np.uint32)
    if n == 1:
        return {"whole": ([ids], [0])}

    def contiguous(x, k):
        return [x[slice(*parallel.shard_range(x.size, r, k))] for r in range(k)]
    fwd = list(range(n))
    out = {
        "contiguous": (contiguous(ids, n), fwd),
        "mod": ([ids[ids % n == r] for r in range(n)], fwd),
        "uneven": ([ids[:1], ids[n - 1:]] + [ids[r - 1:r] for r in range(2, n)], fwd),
        "empty": ([ids[:0]] + contiguous(ids, n - 1), fwd),
        "reversed": (contiguous(ids, n), fwd[::-1]),
    }
    if len(unselected):
        un = np.isin(ids, np.asarray(unselected, dtype=np.uint32))
        out["unselected"] = ([ids[un]] + contiguous(ids[~un], n - 1), fwd)
    return out


def rank_order_mean(rank_sums, n):
    """The integer MEAN of a cell after a multi-rank merge: every rank's exact sum rounded once to f64 (k_export_pairs;
    Python's float(int) rounds to nearest even as it does), added in gather order from +0.0 (k_merge_gathered), over
    the count (k_finalize). A rank without a value of the cell adds +0.0."""
    acc = 0.0
    for s in rank_sums:
        acc += float(s)
    return acc / n


class RankScans:
    """One prepared scan per shard of `shards` (lists of series ids, or boolean masks over the descriptors that keep
    whole column groups: a series split over ranks by time): the shard's descriptors uploaded as its own page set
    (none for an empty shard), the column groups' chunk files (`files`, one per column group in descriptor order) and
    the tombstones set as on the whole arena, and `q` prepared with multi_rank=True and the same group map, edges,
    labels and slide on every rank (`prep`: Engine.prepare's keyword arguments)."""

    def __init__(self, engine, arena, descs, q, shards, files=None, tombstones=None, **prep):
        self.engine = engine
        self.query = multi_rank(q)
        self.pages, self.scans = [], []
        time_page = descs["phys_type"] == cabi.TSKV_PT_TIME
        try:
            for ids in shards:
                ids = np.asarray(ids)
                mine = ids if ids.dtype == bool else np.isin(descs["series_id"], ids)
                pages = engine.upload_pages(arena, descs[mine])
                self.pages.append(pages)
                if files is not None:
                    pages.set_chunk_files(np.asarray(files)[mine[time_page]])
                if tombstones is not None:
                    pages.set_tombstones(tombstones)
                self.scans.append(engine.prepare(pages, self.query, **prep))
        except BaseException:
            self.close()
            raise

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def close(self):
        for s in self.scans:
            s.close()
        for p in self.pages:
            p.close()
        self.scans, self.pages = [], []

    def run(self):
        """One pass on every rank -> every rank's reader counters. Keeps a copy of every rank's exchange region, so that
        each merge below starts from the same partials (a pass adds f64 sums with atomics: a second pass may differ in
        their last bits)."""
        import torch
        dev = torch.device("cuda", self.engine.device)
        out, self.regions = [], []
        for s in self.scans:
            s.run()
            out.append(self.engine.counters())
            ptr, words = s.exchange_view()
            self.regions.append(parallel.device_tensor(ptr, words, torch.int64, dev).clone())
        torch.cuda.synchronize()
        return out

    def restore(self):
        """Every rank's exchange region as the last pass left it."""
        import torch
        dev = torch.device("cuda", self.engine.device)
        for s, saved in zip(self.scans, self.regions):
            ptr, words = s.exchange_view()
            parallel.device_tensor(ptr, words, torch.int64, dev).copy_(saved)
        torch.cuda.synchronize()

    def words(self):
        return [s.exchange_view()[1] for s in self.scans]

    def finalize(self):
        return [s.finalize() for s in self.scans]

    def gather(self, order=None):
        """The all-gather merge in rank order `order` (default 0 .. N-1) -> every rank's finalized result."""
        import torch
        order = range(len(self.scans)) if order is None else order
        self.restore()
        gathered = torch.cat([self.regions[r] for r in order])
        torch.cuda.synchronize()
        for s in self.scans:
            s.merge_gathered(gathered.data_ptr(), len(order))
        out = self.finalize()
        del gathered  # (finalize synchronised the engine stream: the merge has read it)
        return out

    def allreduce(self, order=None):
        """The all-reduce path in rank order `order` -> every rank's finalized result."""
        import torch
        dev = torch.device("cuda", self.engine.device)
        order = list(range(len(self.scans)) if order is None else order)

        def sections(s):
            v = s.partials()
            return {k: parallel.device_tensor(getattr(v, k + "_ptr"), getattr(v, k + "_len"), torch.int64, dev)
                    for k in ("sum_i64", "sum_f64", "min_i64", "max_i64", "sel_val")}

        self.restore()
        for s in self.scans:
            s.snapshot_keys()
        torch.cuda.synchronize()
        secs = [sections(s) for s in self.scans]
        host = [{k: t.cpu().numpy() for k, t in sec.items()} for sec in secs]
        red = {
            "sum_i64": np.sum([h["sum_i64"].view(np.uint64) for h in host], axis=0, dtype=np.uint64).view(np.int64),
            "min_i64": np.minimum.reduce([h["min_i64"] for h in host]),
            "max_i64": np.maximum.reduce([h["max_i64"] for h in host]),
        }
        acc = np.zeros(host[0]["sum_f64"].size, dtype=np.float64)
        for r in order:
            acc = acc + host[r]["sum_f64"].view(np.float64)
        red["sum_f64"] = acc.view(np.int64)
        for sec in secs:
            for k, v in red.items():
                if v.size:
                    sec[k].copy_(torch.from_numpy(np.ascontiguousarray(v)))
        torch.cuda.synchronize()
        for s in self.scans:
            s.mask_values()
        torch.cuda.synchronize()
        vals = [sec["sel_val"].cpu().numpy().view(np.uint64) for sec in secs]
        total = np.sum(vals, axis=0, dtype=np.uint64).view(np.int64)
        if total.size:
            for sec in secs:
                sec["sel_val"].copy_(torch.from_numpy(np.ascontiguousarray(total)))
        torch.cuda.synchronize()
        return self.finalize()


def sharded_scans(engine, arena, descs, q, shards, files=None, tombstones=None, order=None, **prep):
    """The shards' scans merged through the all-gather in rank order `order` -> every rank's finalized result."""
    with RankScans(engine, arena, descs, q, shards, files=files, tombstones=tombstones, **prep) as rs:
        rs.run()
        return rs.gather(order)
