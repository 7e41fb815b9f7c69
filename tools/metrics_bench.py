"""
Measuring top-100 lists with ten ranking metrics at the synthetic ML-25M shape (``data.ML25M_SHAPE``): every one of
the 162,541 users with a rating, about 20 % of each user's ratings held out as the test set (at least one), the bias scorer trained on the rest,
and each user's top 100 over the items outside their training ratings (``engine.offset_scores``, the kernel behind
``BiasScorer.recommend_batch``).  The metrics: NDCG, NDCG@10, DCG, RBP, RecipRank, Hit@10, Precision@10, Recall@10,
AveragePrecision and MeanPopRank.
Reported as median, min and max of ``--reps`` runs, the three device timings alternated:
* ``kernel_ms``: ``engine.rank_metrics`` alone between CUDA events (the table upload and ``lk_rank_metrics``);
* ``measure_topn_ms``: the whole ``measure_topn`` call from the kernel's ``idx`` / ``cnt`` on the host clock,
  synchronised (the test CSR, the tables, the launch, the copy back and the summaries);
* ``measure_batch_ms``: the whole ``measure_batch`` call on the same lists as ``ItemList``s;
* ``host_ms_per_list``: the reference's per-list path (``measure_lists_host``: every metric's ``measure_list``) on
  ``--host-lists`` sampled lists, and that time extrapolated to every list (``host_extrapolated_s``: not measured
  at full scale).  The sampled lists' device values are checked against the host's, bit for bit.
The card name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.
    python tools/metrics_bench.py [--host-lists 2000] [--reps 3] [--out result.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
import warnings
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from lkpy_b200 import _lib, data, engine  # noqa: E402
from lkpy_b200 import metrics as lm  # noqa: E402
from lkpy_b200.basic import BiasScorer  # noqa: E402
from lkpy_b200.components import Dataset, ItemList  # noqa: E402
from lkpy_b200.data import Interactions  # noqa: E402


def _card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)  # fmt: skip
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _log(msg: str) -> None:
    print(msg, file=sys.stderr, flush=True)


def _spread(xs: list[float]) -> dict:
    return {"median": float(np.median(xs)), "min": float(min(xs)), "max": float(max(xs)), "n": len(xs)}


def _wall(fn) -> float:
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def _events(fn) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def ten_metrics(ds) -> list:
    return [lm.NDCG(), lm.NDCG(10), lm.DCG(), lm.RBP(), lm.RecipRank(), lm.Hit(10), lm.Precision(10), lm.Recall(10),
            lm.AveragePrecision(), lm.MeanPopRank(ds)]  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--host-lists", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = _lib.require_device()
    card = _card()
    _log(f"card: {card}")
    t = time.perf_counter()
    it = data.synth_interactions(**data.ML25M_SHAPE)
    _log(f"synthetic ML-25M shape: {it.n_users} users, {it.n_items} items, {it.nnz} ratings "
         f"({time.perf_counter() - t:.1f} s to generate)")  # fmt: skip
    test = np.random.default_rng(31).random(it.nnz) < 0.2
    # every user keeps at least one test item (AveragePrecision divides by the test length)
    rated = np.bincount(it.users, minlength=it.n_users) > 0
    none = np.flatnonzero(rated & (np.bincount(it.users[test], minlength=it.n_users) == 0))
    test[np.searchsorted(it.users, none)] = True
    users = np.flatnonzero(rated)  # the users with a test set: a user without ratings has none to measure
    tr = Interactions(it.users[~test], it.items[~test], it.ratings[~test], it.n_users, it.n_items)
    ds = Dataset(tr)
    scorer = BiasScorer()
    scorer.train(ds)
    # each user's training items, excluded from their list (users without ratings have empty rows: dropped)
    excl_indptr = np.searchsorted(tr.users, np.append(users, it.n_users)).astype(np.int64)
    excl_indptr, excl_items = torch.from_numpy(excl_indptr).to(dev), torch.from_numpy(tr.items.astype(np.int32)).to(dev)
    idx, _val, cnt = engine.offset_scores(scorer._device_base(), len(users), None, args.n, excl_indptr, excl_items)
    tptr = np.searchsorted(it.users[test], np.arange(it.n_users + 1))
    titems = ds.items.ids(it.items[test])
    tests = [ItemList(item_ids=titems[tptr[u] : tptr[u + 1]]) for u in users]
    idx_h, cnt_h = idx.cpu().numpy(), cnt.cpu().numpy()
    lists = [ItemList(item_ids=ds.items.ids(idx_h[b, : cnt_h[b]]), item_nums=idx_h[b, : cnt_h[b]], vocabulary=ds.items,
                      ordered=True) for b in range(len(users))]  # fmt: skip
    ms = ten_metrics(ds)
    B = len(lists)

    # the kernel's own inputs, captured from one measure_topn call
    captured = {}
    real = engine.rank_metrics

    def capture(*a, **kw):
        captured["args"] = (a, kw)
        return real(*a, **kw)

    engine.rank_metrics = capture
    got = lm.measure_topn(ms, ds.items, idx, cnt, tests)
    engine.rank_metrics = real
    a, kw = captured["args"]

    # warm-up of every timed call, and the two device paths agree
    other = lm.measure_batch(ms, lists, tests)
    for c in got.list_metrics.columns:
        assert np.array_equal(got.list_metrics[c].to_numpy(), other.list_metrics[c].to_numpy(), equal_nan=True), c
    real(*a, **kw)

    times = {"kernel_ms": [], "measure_topn_ms": [], "measure_batch_ms": []}
    for _ in range(args.reps):
        times["kernel_ms"].append(_events(lambda: real(*a, **kw)))
        times["measure_topn_ms"].append(_wall(lambda: lm.measure_topn(ms, ds.items, idx, cnt, tests)))
        times["measure_batch_ms"].append(_wall(lambda: lm.measure_batch(ms, lists, tests)))

    rng = np.random.default_rng(2)
    sample = np.sort(rng.choice(B, min(args.host_lists, B), replace=False))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        t = time.perf_counter()
        host = lm.measure_lists_host(ms, [lists[b] for b in sample], [tests[b] for b in sample])
        host_s = time.perf_counter() - t
    for c in host.list_metrics.columns:
        d, h = got.list_metrics[c].to_numpy()[sample], host.list_metrics[c].to_numpy()
        assert np.array_equal(np.isnan(d), np.isnan(h)) and np.array_equal(d[~np.isnan(d)].view(np.int64),
                                                                           h[~np.isnan(h)].view(np.int64)), c  # fmt: skip
    per_list = host_s * 1e3 / len(sample)
    res = {
        "card": card, "shape": {"n_users": it.n_users, "n_items": it.n_items, "nnz": it.nnz}, "users": it.n_users, "lists": B,
        "list_length": args.n, "test_items": int(test.sum()), "metrics": [m.label for m in ms],
        **{k: _spread(v) for k, v in times.items()},
        "host_ms_per_list": per_list, "host_sample": len(sample), "host_extrapolated_s": per_list * B / 1e3,
        "summary": {k: v for k, v in got.summary_metrics.items() if k.endswith(".mean")},
    }  # fmt: skip
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
