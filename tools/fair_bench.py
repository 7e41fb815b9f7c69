"""
FAIRReranker's ``rank_scores`` on the synthetic ML-25M shape (``data.ML25M_SHAPE``): a factor scorer's item-major
score matrix (``engine.als_recommend``'s score mode, k = 64, the path of ``FactorScorer.score_matrix``) for ``--users``
queries, passed as its transpose without a copy, each query's history excluded, for ``N`` (``candidates``) of 100 and
1000 and ``n`` of 10 and 100.  About a third of the items are protected.

Reported per configuration, as median, min and max of ``--reps`` runs with the configurations alternated:

* ``engine_ms``: ``engine.fair_rerank`` alone between CUDA events (the exclusion sort and the fused kernel);
* ``call_ms``: the whole ``rank_scores`` call on the host clock, synchronised (exclusions, the launch, the copy back
  and the ``ItemList``s);
* ``bytes``: the score matrix the kernel reads (4 bytes per score), and that over ``engine_ms`` as a share of the data
  sheet's 3.35 TB/s; ``not_copied_bytes``: the score matrix a host path would copy to the host;
* ``host_ms_per_query``: the host path on ``--host-users`` queries (the score column copied to the host, the history
  set to NaN, argtopn's top N by ``oracle.argtopn``, the C restatement of the reference's heap, and
  ``FAIRReranker.__call__``), and that time extrapolated to every query.  Those queries' device lists are checked
  against the host's.

The card name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.

    python tools/fair_bench.py [--users 32768] [--host-users 64] [--reps 3] [--out result.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import oracle  # noqa: E402
from lkpy_b200 import _lib, data, engine  # noqa: E402
from lkpy_b200.batch import history_csr  # noqa: E402
from lkpy_b200.components import Dataset, ItemList, RecQuery  # noqa: E402
from lkpy_b200.reranking import FAIRReranker  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


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


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--host-users", type=int, default=64)
    ap.add_argument("--k", type=int, default=64)
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
    rng = np.random.default_rng(1)
    ds = Dataset(it, item_attributes={"protected": rng.random(it.n_items) < 0.3})
    sel = np.sort(rng.choice(it.n_users, args.users, replace=False))
    lo, hi = np.searchsorted(it.users, sel), np.searchsorted(it.users, sel + 1)
    queries = [RecQuery(int(u), ItemList(item_nums=it.items[a:b], vocabulary=ds.items)) for u, a, b in zip(sel, lo, hi)]
    q = torch.from_numpy((rng.standard_normal((it.n_items, args.k)) * 0.1).astype(np.float32)).to(dev)
    x = torch.from_numpy((rng.standard_normal((args.users, args.k)) * 0.1).astype(np.float32)).to(dev)
    S = engine.als_recommend(q, x)  # [n_items, B], as FactorScorer.score_matrix returns it
    M = S.T
    B, L = M.shape
    res = {"card": card, "shape": {"n_users": it.n_users, "n_items": it.n_items, "nnz": it.nnz}, "queries": B,
           "k": args.k, "configs": {}}  # fmt: skip

    rerankers = {}
    for n in (10, 100):
        rerankers[n] = FAIRReranker(n=n, p=0.5, alpha=0.1)
        rerankers[n].train(ds)
    configs = [(N, n) for N in (100, 1000) for n in (10, 100)]
    excl = history_csr(queries, ds.items, dev)[1:]
    flags = rerankers[10].protected_attributes

    def engine_call(c):
        N, n = c
        return lambda: engine.fair_rerank(rerankers[n].m_list, n, flags, scores=M, candidates=N, excl_indptr=excl[0],
                                          excl_items=excl[1])  # fmt: skip

    for c in configs:  # warm-up of every shape
        rerankers[c[1]].rank_scores(M, queries, ds.items, candidates=c[0])
    times = {c: {"engine_ms": [], "call_ms": []} for c in configs}
    for _ in range(args.reps):
        for c in configs:
            times[c]["engine_ms"].append(_events(engine_call(c)))
            times[c]["call_ms"].append(_wall(lambda: rerankers[c[1]].rank_scores(M, queries, ds.items, candidates=c[0])))

    for c in configs:
        N, n = c
        r = rerankers[n]
        got = r.rank_scores(M, queries, ds.items, candidates=N)
        by = 4 * B * L
        eng = float(np.median(times[c]["engine_ms"]))
        entry = {k: _spread(v) for k, v in times[c].items()}
        entry["bytes"] = by
        entry["share_of_3.35TB/s"] = by / (eng * 1e-3) / PEAK_BYTES_PER_S
        entry["not_copied_bytes"] = 4 * B * L
        host_ms = []
        for j in range(args.host_users):
            t = time.perf_counter()
            row = S[:, j].cpu().numpy()
            row[queries[j].query_items.numbers()] = np.nan
            top = oracle.argtopn(row, N)
            want = r(ItemList(item_nums=top, vocabulary=ds.items, scores=row[top], ordered=True))
            host_ms.append((time.perf_counter() - t) * 1e3)
            assert np.array_equal(got[j].numbers(), want.numbers()), (c, j)
            assert np.array_equal(got[j].scores().view(np.int32), want.scores().view(np.int32)), (c, j)
        entry["host_ms_per_query"] = _spread(host_ms)
        entry["host_ms_extrapolated"] = float(np.median(host_ms)) * B
        entry["host_checked_queries"] = args.host_users
        res["configs"][f"N={N} n={n}"] = entry
        _log(f"N={N} n={n}: {entry}")
    out = json.dumps(res)
    print(out)
    if args.out:
        Path(args.out).write_text(out + "\n")


if __name__ == "__main__":
    main()
