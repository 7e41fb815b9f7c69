"""
NMFScorer on the synthetic ML-25M shape (``data.ML25M_SHAPE``): the ``nndsvda`` initialisation (randomized SVD and
NNDSVD), then per iteration with CUDA events the ``lk_spmm`` products, the Grams, the sweeps and the violation sums,
then the whole ``train`` (host clock, synchronised), and ``recommend_batch`` top-100 for 32,768 users with
``exclude="query"``; each timed step ``--reps`` times, reported as median, min and max.  ``--host-iters N`` also times N iterations of scikit-learn's coordinate descent on the host.

The card name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.

    python tools/nmf_bench.py [--k 64] [--max-iter 200] [--host-iters 0] [--out result.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
import warnings
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from lkpy_b200 import _lib, data, engine, nmf  # noqa: E402
from lkpy_b200.components import Dataset, ItemList, RecQuery, TrainingOptions  # noqa: E402


def _card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)  # fmt: skip
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _log(msg: str) -> None:
    print(msg, file=sys.stderr, flush=True)


class _Stages:
    """``stage(name)``: CUDA events around each step, summed per name."""

    def __init__(self):
        self.events = defaultdict(list)

    def __call__(self, name):
        stages = self

        class _Ctx:
            def __enter__(self):
                self.s, self.e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                self.s.record()

            def __exit__(self, *_a):
                self.e.record()
                stages.events[name].append((self.s, self.e))

        return _Ctx()

    def totals_ms(self) -> dict:
        torch.cuda.synchronize()
        return {k: sum(s.elapsed_time(e) for s, e in v) for k, v in self.events.items()}


def _spread(xs: list[float]) -> dict:
    return {"median": float(np.median(xs)), "min": float(min(xs)), "max": float(max(xs)), "n": len(xs)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=64)
    ap.add_argument("--max-iter", type=int, default=200)
    ap.add_argument("--iters", type=int, default=10, help="iterations timed stage by stage")
    ap.add_argument("--reps", type=int, default=3, help="repetitions of each timed step: median, min and max")
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--host-iters", type=int, default=0, help="iterations of scikit-learn on the host (0: skip)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = _lib.require_device()
    res = {"card": _card(), "k": args.k}
    it = data.synth_interactions(**data.ML25M_SHAPE)
    ds = Dataset(it)
    res["shape"] = {"users": it.n_users, "items": it.n_items, "nnz": int(it.nnz)}
    _log(f"data ready: {res['shape']}")
    x = nmf.indicator_operand(it.users, it.items, it.n_users, it.n_items, dev)

    # the initialisation, twice (the first loads modules and lets cuSOLVER pick its algorithms)
    for _rep in range(2):
        np.random.seed(0)
        st = _Stages()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        W, H = nmf.initialize(x, args.k, st)
        torch.cuda.synchronize()
        res["init_s"] = time.perf_counter() - t0
        res["init_stages_ms"] = st.totals_ms()

    # iterations, stage by stage (a warm-up iteration first), --reps windows of --iters iterations
    d = engine.NmfDescent(x, W, H.T.contiguous())
    d.iteration()
    its, stages = [], []
    for _rep in range(args.reps):
        st = _Stages()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            d.iteration(st)
        torch.cuda.synchronize()
        its.append((time.perf_counter() - t0) * 1e3 / args.iters)
        stages.append({k: v / args.iters for k, v in st.totals_ms().items()})
        _log(f"iteration: {its[-1]:.2f} ms {stages[-1]}")
    res["iteration_ms"] = _spread(its)
    res["iteration_stages_ms"] = {k: _spread([s[k] for s in stages]) for k in stages[0]}

    # whole train, --reps times
    m = nmf.NMFScorer(embedding_size=args.k, max_iter=args.max_iter)
    trains = []
    for _rep in range(args.reps):
        np.random.seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m.train(ds, TrainingOptions(retrain=True))
        torch.cuda.synchronize()
        trains.append(time.perf_counter() - t0)
        _log(f"train: {trains[-1]:.2f} s, {m.n_iter_} iterations")
    res["train_s"] = _spread(trains)
    res["train_n_iter"] = m.n_iter_
    _log("building queries")

    # recommend_batch top-100, excluding each user's history
    users = np.sort(np.random.default_rng(3).choice(it.n_users, min(args.users, it.n_users), replace=False))
    lo = np.searchsorted(it.users, users.astype(it.users.dtype))
    hi = np.searchsorted(it.users, (users + 1).astype(it.users.dtype))
    queries = [RecQuery(ds.users.id(u), ItemList(item_nums=it.items[a:b], vocabulary=ds.items))
               for u, a, b in zip(users, lo, hi)]  # fmt: skip
    m.recommend_batch(queries[:8], 100, exclude="query")
    recs_s = []
    for _rep in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        recs = m.recommend_batch(queries, 100, exclude="query")
        torch.cuda.synchronize()
        recs_s.append(time.perf_counter() - t0)
        assert all(len(r) == 100 for r in recs)
    res["recommend_s"] = _spread(recs_s)

    if args.host_iters:
        from scipy import sparse as sps
        from sklearn.decomposition._nmf import _update_coordinate_descent

        X = sps.csr_matrix((np.ones(it.nnz, np.float32), (it.users, it.items)), shape=(it.n_users, it.n_items))
        Wh, Hth = W.cpu().numpy(), np.ascontiguousarray(H.T.cpu().numpy())
        t0 = time.perf_counter()
        for _ in range(args.host_iters):
            _update_coordinate_descent(X, Wh, Hth, 0.0, 0.0, False, None)
            _update_coordinate_descent(X.T, Hth, Wh, 0.0, 0.0, False, None)
        res["host_iteration_s"] = (time.perf_counter() - t0) / args.host_iters

    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
