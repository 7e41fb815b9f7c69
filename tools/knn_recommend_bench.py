"""
Batched kNN recommendation at the ML-25M shape (162,541 users x 59,047 items, 25 M ratings, synthetic), the
fused path (``KnnScorerState.recommend``: scoring and top-n selection in one kernel, n entries written per
query) against the unfused device path (``score_all_items`` writing full score and count rows, the offsets and
the exclusion mask, the transpose, ``topn_columns``):

1. item-kNN as in ``bench.py`` (explicit feedback, save_nbrs 20, max_nbrs 20): top-100 with ``exclude="query"``
   for every user, in batches of 16,384;
2. user-kNN: 4,096 known users in batches of 256, neighbours found once per batch and shared by both paths
   (a user id alone excludes nothing), top-100.

For each: the kernel time of each path (sum of the CUDA kernels' device time from ``torch.profiler``, one
profiled pass), the whole pass timed with a host clock around synchronised work (warmed up, the two paths
alternated, 5 samples each), the bytes each path writes, and a bit-for-bit comparison of both outputs
(items, score bits, neighbour counts, list lengths) on every batch.

Prints one JSON object, and also writes it to ``--out`` when that is given.
"""

from __future__ import annotations

import argparse
import gc
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
from lkpy_b200.components import Dataset  # noqa: E402
from lkpy_b200.knn import ItemKNNScorer  # noqa: E402
from lkpy_b200.knn_user import UserKNNScorer  # noqa: E402


def gpu_info() -> dict:
    out = subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
        capture_output=True, text=True, check=False,
    ).stdout.strip()  # fmt: skip
    name, _, power = out.partition(",")
    return {"name": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip()}


def kernel_ms(fn) -> tuple[float, dict]:
    """Summed device time of every CUDA kernel fn() launches, and the time per kernel name."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per: dict[str, float] = {}
    for ev in prof.events():
        if getattr(ev, "device_type", None) != torch.autograd.DeviceType.CUDA:
            continue
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        per[ev.name] = per.get(ev.name, 0.0) + t / 1000.0
    return sum(per.values()), {k[:80]: round(v, 2) for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:6]}


def alternate(paths: dict, samples: int) -> dict:
    times = {k: [] for k in paths}
    for _ in range(samples):
        for name, fn in paths.items():
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t1) * 1e3)
    return {f"{k}_ms": {"median": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1),
                        "samples": len(v)} for k, v in times.items()}  # fmt: skip


def unfused(st, ref_ptr, ref_items, ref_vals, max_nbrs, n, item_offset=None, query_offset=None, excl=None):
    """The device path without the ranking mode: full rows, offsets, exclusion mask, transpose, topn_columns."""
    sc, ct = st.score_all_items(ref_ptr, ref_items, ref_vals, max_nbrs, 1)
    if item_offset is not None:
        sc.add_(item_offset[None, :])
    if query_offset is not None:
        sc.add_(query_offset[:, None])
    if excl is not None:
        e_ptr, e_items = excl
        rows = torch.repeat_interleave(torch.arange(sc.shape[0], device=sc.device), e_ptr[1:] - e_ptr[:-1])
        ok = e_items >= 0
        sc[rows[ok], e_items[ok].long()] = float("nan")
    idx, val, cnt = engine.topn_columns(sc.T.contiguous(), n)
    nbrs = torch.gather(ct, 1, idx.long().clamp_min(0)) * (idx >= 0)
    return idx, val, nbrs.to(torch.int32), cnt


def same(a, b) -> bool:
    (i1, v1, n1, c1), (i2, v2, n2, c2) = a, b
    return bool(
        torch.equal(i1, i2) and torch.equal(v1.view(torch.int32), v2.view(torch.int32)) and torch.equal(n1, n2)
        and torch.equal(c1, c2)
    )


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--batch", type=int, default=16384)
    ap.add_argument("--users", type=int, default=0, help="item-kNN users to recommend for (0: all)")
    ap.add_argument("--user-knn-users", type=int, default=4096)
    ap.add_argument("--user-knn-batch", type=int, default=256)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    dev = _lib.require_device()
    res = {"gpu": gpu_info(), "shape": data.ML25M_SHAPE, "n": args.n}
    t0 = time.perf_counter()
    inter = data.synth_interactions(**data.ML25M_SHAPE)
    ds = Dataset(inter)
    R = inter.coo().tocsr()
    n_users, n_items = R.shape

    # 1. item-kNN, every user (or --users), exclude="query"
    m = ItemKNNScorer(max_nbrs=20, min_sim=1e-6, save_nbrs=20)
    m.train(ds)
    st = m._device_state()
    means = torch.from_numpy(m.item_means).to(dev)
    res["setup_s"] = round(time.perf_counter() - t0, 1)
    U = n_users if args.users <= 0 else min(args.users, n_users)
    rv_all = (R.data - m.item_means[R.indices]).astype(np.float32)
    batches = []
    for u0 in range(0, U, args.batch):
        u1 = min(u0 + args.batch, U)
        a0, a1 = int(R.indptr[u0]), int(R.indptr[u1])
        ptr_ = torch.from_numpy((R.indptr[u0 : u1 + 1] - a0).astype(np.int64)).to(dev)
        ri = torch.from_numpy(R.indices[a0:a1].astype(np.int32)).to(dev)
        batches.append((ptr_, ri, torch.from_numpy(rv_all[a0:a1]).to(dev)))

    def fused_item(b):
        p, ri, rv = b
        return st.recommend(p, ri, rv, 20, 1, args.n, item_offset=means, excl_indptr=p, excl_items=ri)

    def unfused_item(b):
        p, ri, rv = b
        return unfused(st, p, ri, rv, 20, args.n, item_offset=means, excl=(p, ri))

    ok = True
    for b in batches:  # warm-up, and the two paths must agree bit for bit on every batch
        ok = same(fused_item(b), unfused_item(b)) and ok
        torch.cuda.empty_cache()
    k_f, k_f_names = kernel_ms(lambda: [fused_item(b) for b in batches])
    k_u, k_u_names = kernel_ms(lambda: [unfused_item(b) for b in batches])
    B = U
    res["item_knn"] = {
        "users": U, "batch": args.batch, "batches": len(batches), "outputs_bit_identical": ok,
        "kernel_ms": {"fused": round(k_f, 1), "unfused": round(k_u, 1)},
        "kernels": {"fused": k_f_names, "unfused": k_u_names},
        # fused: n x (item, score, count) + the list length; unfused: score_all_items' f32 + int32 rows, the
        # transposed copy of the scores, topn_columns' n x (item, score) + length
        "output_bytes": {"fused": B * args.n * 12 + B * 4,
                         "unfused": B * n_items * 8 + B * n_items * 4 + B * args.n * 8 + B * 4},
        **alternate({"fused": lambda: [fused_item(b) for b in batches],
                     "unfused": lambda: [unfused_item(b) for b in batches]}, args.samples),
    }  # fmt: skip
    print(json.dumps({"item_knn": res["item_knn"]}), file=sys.stderr, flush=True)
    # the user-mode contribution pool of a 256-query batch takes ~45 GB at this shape: free the item-kNN state
    del batches, m, st, means
    gc.collect()
    torch.cuda.empty_cache()
    res["allocated_GB_before_user_knn"] = round(torch.cuda.memory_allocated() / 1e9, 2)

    # 2. user-kNN, known users (a user id alone excludes nothing)
    um = UserKNNScorer()  # explicit feedback, min_sim 1e-6, max_nbrs 20
    um.train(ds)
    ust, ns = um._device_state(), um._neighbour_state()
    rng = np.random.default_rng(0)
    users = np.sort(rng.choice(n_users, args.user_knn_users, replace=False))
    ubatches = []
    for b0 in range(0, len(users), args.user_knn_batch):
        ub = users[b0 : b0 + args.user_knn_batch]
        ip, rows, sims = ns.neighbours(ns.known_queries(ub), um.config.min_sim)
        ubatches.append((ip, rows, sims, torch.from_numpy(um.user_means[ub].astype(np.float32)).to(dev)))

    def fused_user(b):
        ip, rows, sims, qoff = b
        return ust.recommend(ip, rows, sims, 20, 1, args.n, query_offset=qoff)

    def unfused_user(b):
        ip, rows, sims, qoff = b
        return unfused(ust, ip, rows, sims, 20, args.n, query_offset=qoff)

    uok = True
    for b in ubatches:
        uok = same(fused_user(b), unfused_user(b)) and uok
    k_f, k_f_names = kernel_ms(lambda: [fused_user(b) for b in ubatches])
    k_u, k_u_names = kernel_ms(lambda: [unfused_user(b) for b in ubatches])
    B = len(users)
    res["user_knn"] = {
        "users": B, "batch": args.user_knn_batch, "outputs_bit_identical": uok,
        "neighbours": int(sum(int(b[0][-1].item()) for b in ubatches)),
        "kernel_ms": {"fused": round(k_f, 1), "unfused": round(k_u, 1)},
        "kernels": {"fused": k_f_names, "unfused": k_u_names},
        "output_bytes": {"fused": B * args.n * 12 + B * 4,
                         "unfused": B * n_items * 8 + B * n_items * 4 + B * args.n * 8 + B * 4},
        **alternate({"fused": lambda: [fused_user(b) for b in ubatches],
                     "unfused": lambda: [unfused_user(b) for b in ubatches]}, args.samples),
    }  # fmt: skip
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")
    return 0 if ok and uok else 1


if __name__ == "__main__":
    sys.exit(main())
