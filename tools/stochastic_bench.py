"""
StochasticTopNRanker on the synthetic ML-25M shape (``data.ML25M_SHAPE``): a factor scorer's item-major score matrix
(``engine.als_recommend``'s score mode, k = 64, the path of ``FactorScorer.score_matrix``) for ``--users`` queries,
ranked by ``rank_scores`` with ``exclude="query"`` (each query a user's history), top-100 and top-500, with each
transform, and with ``rng`` an int (one shared stream) and ``(seed, "user")`` (a generator per user).

Reported per configuration, as median, min and max of ``--reps`` runs with the configurations alternated:

* ``engine_ms``: ``engine.stochastic_topn`` alone between CUDA events (the three kernels and the exclusion sort);
* ``call_ms``: the whole ``rank_scores`` call on the host clock, synchronised (seeding, exclusions, the launches, the
  copy back and the ``ItemList``s);
* ``seed_ms``: the host seeding of the per-user generators alone (``(seed, "user")`` only);
* ``bytes`` counted from the shapes (the score matrix read twice; for softmax and linear the compacted scores
  written once and read twice), and their rate over ``engine_ms`` as a share of the data sheet's 3.35 TB/s;
* ``host_ms_per_query``: the reference's per-query path on ``--host-users`` queries (the score column copied to the
  host, the candidate list, the key statements of tests/stochastic_oracle.py and a NumPy argsort standing in for
  argtopn), and that time extrapolated to every query.

The card name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.

    python tools/stochastic_bench.py [--users 32768] [--host-users 16] [--reps 3] [--out result.json]
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
sys.path.insert(0, str(ROOT / "tests"))

import stochastic_oracle as so  # noqa: E402
from lkpy_b200 import _lib, data, engine  # noqa: E402
from lkpy_b200.batch import history_csr  # noqa: E402
from lkpy_b200.components import Dataset, ItemList, RecQuery  # noqa: E402
from lkpy_b200.stochastic import StochasticTopNRanker  # noqa: E402

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


def counted_bytes(B: int, L: int, transform) -> int:
    reads = 2 * 4 * B * L  # the prepare pass and the key pass each read every score
    return reads + (3 * 4 * B * L if transform is not None else 0)  # compacted: written, summed, read for the keys


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--host-users", type=int, default=16)
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
    ds = Dataset(it)
    rng = np.random.default_rng(1)
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

    configs = [(n, tf, rs) for n in (100, 500) for tf in ("softmax", "linear", None) for rs in ("int", "user")]
    rankers = {c: StochasticTopNRanker(n=c[0], transform=c[1], rng=42 if c[2] == "int" else (42, "user")) for c in configs}
    excl = history_csr(queries, ds.items, dev)[1:]

    def engine_call(c):
        r = rankers[c]
        states, shared, _gen = r._streams(queries)
        return lambda: engine.stochastic_topn(M, c[0], transform=c[1], scale=1.0, states=states, shared=shared,
                                              excl_indptr=excl[0], excl_items=excl[1])  # fmt: skip

    for c in configs:  # warm-up of every shape
        rankers[c].rank_scores(M, queries, ds.items)
    times = {c: {"engine_ms": [], "call_ms": [], "seed_ms": []} for c in configs}
    for _ in range(args.reps):
        for c in configs:
            times[c]["engine_ms"].append(_events(engine_call(c)))
            times[c]["call_ms"].append(_wall(lambda: rankers[c].rank_scores(M, queries, ds.items)))
            if c[2] == "user":
                t = time.perf_counter()
                rankers[c]._streams(queries)
                times[c]["seed_ms"].append((time.perf_counter() - t) * 1e3)

    host = S[:, : args.host_users].T.cpu().numpy()  # only for the checks below
    for c in configs:
        n, tf, rs = c
        by = counted_bytes(B, L, tf)
        eng = float(np.median(times[c]["engine_ms"]))
        entry = {k: _spread(v) for k, v in times[c].items() if v}
        entry["bytes"] = by
        entry["share_of_3.35TB/s"] = by / (eng * 1e-3) / PEAK_BYTES_PER_S
        # the reference's per-query path on a few queries
        host_ms = []
        gen = np.random.default_rng(7)
        for j in range(args.host_users):
            t = time.perf_counter()
            col = S[:, j].cpu().numpy()
            cand = np.setdiff1d(np.arange(L), queries[j].query_items.numbers())
            s = col[cand]
            valid = np.isfinite(s)
            k = so.keys(s[valid], tf, 1.0, gen)
            cand[valid][np.argsort(-k)[:n]]
            host_ms.append((time.perf_counter() - t) * 1e3)
        entry["host_ms_per_query"] = _spread(host_ms)
        entry["host_ms_extrapolated"] = float(np.median(host_ms)) * B
        res["configs"][f"n={n} transform={tf} rng={rs}"] = entry
        _log(f"n={n} transform={tf} rng={rs}: {entry}")
    del host
    out = json.dumps(res)
    print(out)
    if args.out:
        Path(args.out).write_text(out + "\n")


if __name__ == "__main__":
    main()
