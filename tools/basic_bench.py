"""
BiasScorer and PopScorer on the synthetic ML-25M shape (``data.ML25M_SHAPE``):

* the bias model: ``lk_bias_learn`` (CUDA events around the kernels; with only the item pass and only the user pass
  as well, beside the longest entity of each, whose f64 chain is the floor of its pass), the whole device
  ``basic.learn`` (host clock, synchronised, with the upload and the CSR build), and the host ``BiasModel.learn`` —
  device and host runs alternated, and their results compared bit for bit;
* ``recommend_batch`` top-100 with ``exclude="query"`` for ``--users`` queries (each a user id with that user's
  history), both scorers, against the host per-query path (``compute_for_items`` or ``item_scores``, exclusion,
  ``argtopn`` as the host heap of ``oracle``) on ``--host-users`` of them.

Each timed step runs ``--reps`` times, reported as median, min and max.  The card name and power limit are read in
the same run.  Needs a GPU; there is no CPU fallback.

    python tools/basic_bench.py [--users 32768] [--host-users 16] [--reps 3] [--out result.json]
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

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import oracle  # noqa: E402
from lkpy_b200 import _lib, basic, data, engine  # noqa: E402
from lkpy_b200.basic import BiasModel  # noqa: E402
from lkpy_b200.components import Dataset, ItemList, RecQuery  # noqa: E402
from lkpy_b200.prep import coo_to_csr_pair  # noqa: E402


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


def same(a: BiasModel, b: BiasModel) -> bool:
    return (a.global_bias == b.global_bias and np.array_equal(a.item_biases.view(np.int32), b.item_biases.view(np.int32))
            and np.array_equal(a.user_biases.view(np.int32), b.user_biases.view(np.int32)))  # fmt: skip


def host_recommend(scorer, q: RecQuery, all_items: ItemList, n: int) -> np.ndarray:
    """The reference's per-query path: ``__call__`` over every item, the query's items left out, ``argtopn``."""
    if isinstance(scorer, basic.BiasScorer):
        m = scorer.model
        s = np.full(len(all_items), m.global_bias, dtype=np.float32)
        s[all_items.numbers()] += m.item_biases[all_items.numbers()]
        uno = scorer.users.number(q.user_id, missing="none")
        if uno is not None:
            s += m.user_biases[uno]
    else:
        s = scorer(all_items).scores().copy()
    s[q.query_items.numbers(vocabulary=scorer.items, missing="negative")] = np.nan
    return oracle.argtopn(s, n)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--host-users", type=int, default=16)
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--damping", type=float, default=5.0)
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
    counts_i, counts_u = np.bincount(it.items, minlength=it.n_items), np.bincount(it.users, minlength=it.n_users)
    res = {"card": card, "shape": {"n_users": it.n_users, "n_items": it.n_items, "nnz": it.nnz},
           "longest_item": int(counts_i.max()), "longest_user": int(counts_u.max()), "damping": args.damping}  # fmt: skip

    # --- kernels alone on resident inputs
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    users, items, ratings = up(it.users), up(it.items), up(it.ratings)
    ui, iu, _ = coo_to_csr_pair(users, items, ratings, it.n_users, it.n_items)
    d = (args.damping, args.damping)
    kernel = lambda **kw: engine.bias_learn(ratings, items, ui.indptr, iu.indptr, iu.values, d, **kw)  # noqa: E731
    variants = {"both": {}, "item_pass_only": {"user_pass": False}, "user_pass_only": {"item_pass": False},
                "mean_only": {"item_pass": False, "user_pass": False}}  # fmt: skip
    for kw in variants.values():
        kernel(**kw)  # warm-up
    kt = {k: [] for k in variants}
    for _ in range(args.reps):
        for k, kw in variants.items():
            kt[k].append(_events(lambda: kernel(**kw)))
    res["kernel_ms"] = {k: _spread(v) for k, v in kt.items()}
    _log(f"lk_bias_learn: {res['kernel_ms']}")

    # --- device learn against the host learn, alternated
    dev_ms, host_ms = [], []
    dm = basic.learn(ds, args.damping)  # warm-up
    for _ in range(args.reps):
        dev_ms.append(_wall(lambda: basic.learn(ds, args.damping)))
        t = time.perf_counter()
        hm = BiasModel.learn(it, d, np.float32)
        host_ms.append((time.perf_counter() - t) * 1e3)
    res["learn_device_ms"], res["learn_host_ms"] = _spread(dev_ms), _spread(host_ms)
    res["learn_bit_identical"] = same(dm, hm)
    _log(f"learn: device {res['learn_device_ms']}, host {res['learn_host_ms']}, identical {res['learn_bit_identical']}")
    del users, items, ratings, ui, iu

    # --- recommend_batch against the host per-query path
    rng = np.random.default_rng(1)
    sel = np.sort(rng.choice(it.n_users, args.users, replace=False))
    lo, hi = np.searchsorted(it.users, sel), np.searchsorted(it.users, sel + 1)
    bs, ps = basic.BiasScorer(damping=args.damping), basic.PopScorer(score="quantile")
    bs.train(ds)
    ps.train(ds)
    queries = [RecQuery(int(u), ItemList(item_nums=it.items[a:b], vocabulary=ds.items)) for u, a, b in zip(sel, lo, hi)]
    all_items = ItemList(item_nums=np.arange(it.n_items, dtype=np.int32), vocabulary=ds.items)
    res["recommend"] = {}
    for name, sc in (("BiasScorer", bs), ("PopScorer", ps)):
        recs = sc.recommend_batch(queries, args.n)  # warm-up, and the lists checked below
        dev_ms = [_wall(lambda: sc.recommend_batch(queries, args.n)) for _ in range(args.reps)]
        host_ms = []
        ok = True
        for j in range(args.host_users):
            t = time.perf_counter()
            want = host_recommend(sc, queries[j], all_items, args.n)
            host_ms.append((time.perf_counter() - t) * 1e3)
            ok &= bool(np.array_equal(recs[j].numbers(), want))
        per_q = float(np.median(host_ms))
        res["recommend"][name] = {
            "device_ms": _spread(dev_ms), "host_ms_per_query": _spread(host_ms),
            "host_ms_extrapolated": per_q * args.users, "lists_match_host": ok,
        }  # fmt: skip
        _log(f"{name}: {res['recommend'][name]}")
    out = json.dumps(res)
    print(out)
    if args.out:
        Path(args.out).write_text(out + "\n")


if __name__ == "__main__":
    main()
