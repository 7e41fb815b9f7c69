"""
Batched ALS recommendation at the ML-25M shape (162,541 users x 59,047 items, 25 M ratings, synthetic; ImplicitMF
k = 64 trained for 2 epochs), top-100: the fused kernel (``lk_als_recommend_batch``) against the previous path,
a cuBLAS fp32 GEMM into the [items x users] score matrix followed by ``topn_columns``.

1. rank mode against GEMM + ``topn_columns`` for 32,768 users, nothing excluded: kernel time (CUDA events around
   each path's device work) and whole ``recommend_batch``-style calls (host clock around synchronised work);
2. score mode against the GEMM alone at the same shape;
3. all 162,541 users in one ``recommend_batch(..., exclude="query")`` call, each excluding its training items:
   time and peak device memory;
4. the achieved FP32 rate of the dot products (2 n_items B k over the rank-mode kernel time) against the data
   sheet's 67 TFLOP/s;
5. how many of the 32,768 fused and unfused top-100 lists differ, and the largest difference between the two
   score matrices (the summation orders differ).

Paths alternate; medians of ``--samples`` runs.  Prints one JSON object, and writes it to ``--out`` when given.
"""

from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from lkpy_b200 import _lib, data, engine  # noqa: E402
from lkpy_b200.als import ImplicitMFScorer  # noqa: E402
from lkpy_b200.components import Dataset, ItemList, RecQuery, TrainingOptions  # noqa: E402

FP32_PEAK_TFLOPS = 67.0  # H100 SXM data sheet, dense FP32


def gpu_info() -> dict:
    out = subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
        capture_output=True, text=True, check=False,
    ).stdout.strip()  # fmt: skip
    name, _, power = out.partition(",")
    return {"name": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip()}


def stats(v: list[float]) -> dict:
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3), "samples": len(v)}


def device_ms(fn) -> float:
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1])


def host_ms(fn) -> float:
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def unfused_recommend(model, queries, n):
    """The previous ``ALSBase.recommend_batch``: GEMM into the score matrix, then ``topn_columns``."""
    X, scorable, _user_nums, _fold = model.embed_batch(queries)
    S = model._device_items() @ X.T
    idx, val, cnt = engine.topn_columns(S, n)
    idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy()
    return [
        ItemList(item_ids=model.items.ids(idx[b, : cnt[b]]), item_nums=idx[b, : cnt[b]].copy(), vocabulary=model.items,
                 scores=val[b, : cnt[b]].copy())
        for b in range(len(queries))
    ]  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    dev = _lib.require_device()
    res: dict = {"gpu": gpu_info(), "shape": data.ML25M_SHAPE, "k": 64, "n": args.n}

    inter = data.synth_interactions(**data.ML25M_SHAPE)
    ds = Dataset(inter)
    model = ImplicitMFScorer(features=64, epochs=2, user_embeddings="prefer")
    model.train(ds, TrainingOptions(rng=7))
    Q = model._device_items()
    n_items, k = Q.shape
    n_users = model.user_embeddings.shape[0]
    rng = np.random.default_rng(11)
    users = np.sort(rng.choice(n_users, args.batch, replace=False))
    X = torch.from_numpy(model.user_embeddings[users]).to(dev)
    n = args.n

    # 1/2: kernels, alternated (warm both shapes first)
    paths = {
        "rank": lambda: engine.als_recommend(Q, X, n),
        "gemm_topn": lambda: engine.topn_columns(Q @ X.T, n),
        "score": lambda: engine.als_recommend(Q, X, None),
        "gemm": lambda: Q @ X.T,
    }
    for fn in paths.values():
        fn()
    times: dict[str, list[float]] = {name: [] for name in paths}
    for _ in range(args.samples):
        for name, fn in paths.items():
            times[name].append(device_ms(fn))
    res["kernel_ms"] = {name: stats(v) for name, v in times.items()}
    flop = 2.0 * n_items * args.batch * k
    for name in ("rank", "score", "gemm"):
        tf = flop / (statistics.median(times[name]) * 1e-3) / 1e12
        res.setdefault("dot_product_fp32", {})[name] = {
            "tflops": round(tf, 2), "share_of_67_tflops": round(tf / FP32_PEAK_TFLOPS, 3)}  # fmt: skip
    res["dot_product_gflop"] = round(flop / 1e9, 1)

    # whole calls through the component (queries by user id, nothing excluded)
    ids = model.users.ids(users)
    queries = [RecQuery(user_id=u) for u in ids]
    calls = {"fused": lambda: model.recommend_batch(queries, n), "unfused": lambda: unfused_recommend(model, queries, n)}
    for fn in calls.values():
        fn()
    ctimes: dict[str, list[float]] = {name: [] for name in calls}
    for _ in range(args.samples):
        for name, fn in calls.items():
            ctimes[name].append(host_ms(fn))
    res["call_ms"] = {name: stats(v) for name, v in ctimes.items()}

    # 5: fused vs unfused lists and scores
    fi, fv, fc = (t.cpu().numpy() for t in engine.als_recommend(Q, X, n))
    S_fma = engine.als_recommend(Q, X, None)
    S_gemm = Q @ X.T
    res["max_abs_score_diff"] = float((S_fma - S_gemm).abs().max().item())
    del S_fma
    ui, uv, uc = (t.cpu().numpy() for t in engine.topn_columns(S_gemm, n))
    del S_gemm
    differ = int(np.sum(np.any(fi != ui, axis=1) | (fc != uc)))
    res["lists_differing"] = {"count": differ, "of": args.batch}

    # 3: all users, each excluding its training items, in one call
    R = inter.coo().tocsr()
    all_ids = model.users.ids(np.arange(n_users))
    all_q = [
        RecQuery(user_id=all_ids[u], query_items=ItemList(item_nums=R.indices[R.indptr[u] : R.indptr[u + 1]],
                                                           vocabulary=model.items))
        for u in range(n_users)
    ]  # fmt: skip
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t_all = [host_ms(lambda: model.recommend_batch(all_q, n, exclude="query")) for _ in range(2)]
    res["all_users_exclude_query"] = {
        "users": n_users, "call_ms": stats(t_all),
        "peak_extra_device_mb": round((torch.cuda.max_memory_allocated() - base) / 2**20, 1),
        "kernel_ms_no_exclusion": round(device_ms(lambda: engine.als_recommend(
            Q, torch.from_numpy(model.user_embeddings).to(dev), n)), 2),
    }  # fmt: skip

    line = json.dumps(res)
    print(line)
    if args.out is not None:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
