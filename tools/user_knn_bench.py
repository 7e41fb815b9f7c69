"""
User-kNN neighbour search at the ML-25M shape (162,541 users x 59,047 items, 25 M ratings, synthetic):

1. ``lk_uknn_search`` for 4,096 known users in batches (kernel time from the CUDA profiler, whole call from
   CUDA events), products/s and algorithmic GB/s (12 B per product read from VT + 8 B per neighbour
   written) against the H100 SXM data sheet's 3.35 TB/s, for both accumulator geometries (1 and 2 CTAs/SM);
   a probe of short-history users gives the fixed per-unit cost (the threshold scan of a whole tile);
2. the host path it replaces, SciPy's ``user_vectors @ x`` and mask, for 64 of those users;
3. ``UserKNNScorer.score_batch``, 128 queries x 100 targets in batches of 8 (the user-mode contribution pool
   is ~16 B x 10 M per query at this shape), device search against the SciPy neighbours restated here, the
   two alternated, 5 samples each;
4. bit-identity of the neighbour lists of a sample of the timed users against SciPy.

Prints one JSON object, and also writes it to ``--out`` when that is given.
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
from lkpy_b200.components import Dataset, ItemList  # noqa: E402
from lkpy_b200.knn_user import UserKNNScorer  # noqa: E402

HBM_TBS = 3.35


def gpu_info() -> dict:
    out = subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
        capture_output=True, text=True, check=False,
    ).stdout.strip()  # fmt: skip
    name, _, power = out.partition(",")
    return {"name": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip()}


def search_kernel_ms(fn) -> float:
    """Device time of the lk_uknn_search kernels launched by fn()."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for ev in prof.events():
        if "uknn_search_kernel" in ev.name:
            tot += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return tot / 1000.0


def timed_search(ns, users, batch, min_sim):
    """(event ms of the whole calls, kernel ms, products, neighbours)."""
    prods = nbrs = 0
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run():
        nonlocal prods, nbrs
        prods = nbrs = 0
        for b in range(0, len(users), batch):
            qs = ns.known_queries(users[b : b + batch])
            ip, _r, _s = ns.neighbours(qs, min_sim)
            nbrs += int(ip[-1].item())
        return nbrs

    run()  # warm-up
    torch.cuda.synchronize()
    start.record()
    run()
    stop.record()
    torch.cuda.synchronize()
    call_ms = start.elapsed_time(stop)
    kern_ms = search_kernel_ms(run)
    for b in range(0, len(users), batch):
        prods += int(ns.query_cost(ns.known_queries(users[b : b + batch])).sum().item())
    return call_ms, kern_ms, prods, nbrs


def rates(ms, prods, nbrs):
    gb = (12 * prods + 8 * nbrs) / 1e9
    return {
        "ms": round(ms, 2), "products": prods, "neighbours": nbrs,
        "products_per_s": float(f"{prods / (ms / 1e3):.4g}"), "algorithmic_GB": round(gb, 2),
        "algorithmic_GBps": round(gb / (ms / 1e3), 1),
        "fraction_of_datasheet_3.35TBps": round(gb / (ms / 1e3) / (HBM_TBS * 1e3), 3),
    }  # fmt: skip


def host_neighbours(V, x, self_, min_sim):
    sims = V @ x
    if self_ is not None:
        sims[self_] = 0
    mask = sims >= min_sim
    return np.flatnonzero(mask).astype(np.int32), sims[mask].astype(np.float32)


def host_path_scores(m, st, queries, targets):
    """score_batch with the SciPy neighbour search it replaced (known-user queries only)."""
    dev = st.sim_cols.device
    V = m.user_vectors
    r_ptr, t_ptr, nbrs, sims, tgts, metas = [0], [0], [], [], [], []
    for q, items in zip(queries, targets):
        u = int(m.users.number(q))
        rr, ss = host_neighbours(V, V[[u], :].toarray()[0], u, m.config.min_sim)
        iidx = items.numbers(vocabulary=m.items, missing="negative").astype(np.int32)
        ki = iidx >= 0
        nbrs.append(rr)
        sims.append(ss)
        tgts.append(iidx[ki])
        metas.append((ki, float(m.user_means[u])))
        r_ptr.append(r_ptr[-1] + len(rr))
        t_ptr.append(t_ptr[-1] + int(ki.sum()))
    t = lambda a, dt: torch.from_numpy(np.asarray(a, dtype=dt)).to(dev)  # noqa: E731
    sc, _ = st.score(
        t(r_ptr, np.int64), t(np.concatenate(nbrs), np.int32), t(np.concatenate(sims), np.float32),
        t(t_ptr, np.int64), t(np.concatenate(tgts), np.int32), m.config.max_nbrs, m.config.min_nbrs,
    )  # fmt: skip
    sc = sc.cpu().numpy()
    out = []
    for i, items in enumerate(targets):
        full = np.full(len(items), np.nan, dtype=np.float32)
        ki, umean = metas[i]
        full[ki] = sc[t_ptr[i] : t_ptr[i + 1]] + np.float32(umean)
        out.append(full)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--host-users", type=int, default=64)
    ap.add_argument("--e2e-queries", type=int, default=128)
    ap.add_argument("--e2e-batch", type=int, default=8)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    dev = _lib.require_device()
    res = {"gpu": gpu_info(), "shape": data.ML25M_SHAPE}
    t0 = time.perf_counter()
    inter = data.synth_interactions(**data.ML25M_SHAPE)
    ds = Dataset(inter)
    m = UserKNNScorer()  # explicit feedback, min_sim 1e-6, max_nbrs 20
    m.train(ds)
    V = m.user_vectors
    res["setup_s"] = round(time.perf_counter() - t0, 1)
    min_sim = m.config.min_sim
    rng = np.random.default_rng(0)
    users = np.sort(rng.choice(V.shape[0], args.users, replace=False))

    # 1. device neighbour search, both geometries
    search = {}
    for ctas in (2, 1):
        ns = engine.UserNeighbourState.create(V, dev, ctas_per_sm=ctas)
        g = ns.geom
        call_ms, kern_ms, prods, nbrs = timed_search(ns, users, args.batch, min_sim)
        r = {"tile_users": g.warps * g.tile_cols, "tiles": g.n_halves,
             "tile_ptr_MB": round(V.shape[1] * (g.n_subtiles + 1) * 4 / 1e6, 1),
             "kernel": rates(kern_ms, prods, nbrs), "whole_calls_ms": round(call_ms, 2),
             "per_query_kernel_us": round(kern_ms * 1e3 / len(users), 1)}  # fmt: skip
        # fixed cost per unit: the users with the fewest (nonzero) products, one tile pass each
        cost = ns.query_cost(ns.known_queries(np.arange(V.shape[0]))).cpu().numpy()
        cheap = np.argsort(np.where(cost > 0, cost, np.iinfo(np.int64).max), kind="stable")[: args.users]
        p_call, p_kern, p_prods, p_nbrs = timed_search(ns, np.sort(cheap), args.batch, min_sim)
        units = len(cheap) * g.n_halves
        r["short_history_probe"] = {"products": p_prods, "kernel_ms": round(p_kern, 2), "units": units,
                                    "grid_us_per_unit": round(p_kern * 1e3 / units, 3)}  # fmt: skip
        # upper bound on the share of the per-unit fixed cost (scan + reset) in the timed run
        r["scan_share_estimate"] = round(min(1.0, p_kern / units * len(users) * g.n_halves / kern_ms), 3)
        if ctas == 2:
            r["products_median_per_query"] = int(np.median(cost[users]))
            r["products_max_per_query"] = int(cost[users].max())
            keep_ns = ns
        search[f"ctas_per_sm={ctas}"] = r
        del ns
        torch.cuda.empty_cache()
    res["search"] = search
    ns = keep_ns

    # 4. bit-identity at the timed size: a sample of the timed users, from the timed batch shape
    sample = users[: args.batch]
    ip, rows, sims = (t.cpu().numpy() for t in ns.neighbours(ns.known_queries(sample), min_sim))
    checked = mism = 0
    for q in range(0, len(sample), 8):
        rr, ss = host_neighbours(V, V[[int(sample[q])], :].toarray()[0], int(sample[q]), min_sim)
        lo, hi = ip[q], ip[q + 1]
        ok = np.array_equal(rows[lo:hi], rr) and np.array_equal(sims[lo:hi].view(np.int32), ss.view(np.int32))
        mism += 0 if ok else 1
        checked += 1
    res["bit_identity"] = {"queries_checked": checked, "mismatches": mism, "neighbours_checked": int(ip[-1])}

    # 2. host mat-vec on the CPU of the measured system (single call per query, SciPy)
    ht = []
    for u in users[: args.host_users]:
        x = V[[int(u)], :].toarray()[0]
        t1 = time.perf_counter()
        host_neighbours(V, x, int(u), min_sim)
        ht.append((time.perf_counter() - t1) * 1e3)
    res["host_matvec_ms_per_query"] = {"median": round(statistics.median(ht), 2), "max": round(max(ht), 2),
                                       "n": len(ht)}  # fmt: skip

    # 3. end to end score_batch, alternated with the restated host path
    st = m._device_state()
    qids = [ds.users.id(int(u)) for u in users[: args.e2e_queries]]
    tg = [ItemList(item_nums=rng.choice(V.shape[1], 100, replace=False).astype(np.int32), vocabulary=ds.items)
          for _ in qids]  # fmt: skip
    B = args.e2e_batch

    def dev_path():
        return [s.scores() for b in range(0, len(qids), B) for s in m.score_batch(qids[b : b + B], tg[b : b + B])]

    def host_path():
        return [s for b in range(0, len(qids), B) for s in host_path_scores(m, st, qids[b : b + B], tg[b : b + B])]

    a, h = dev_path(), host_path()  # warm-up, and the two paths must agree bit for bit
    same = all(np.array_equal(np.asarray(x, np.float32).view(np.int32), y.view(np.int32)) for x, y in zip(a, h))
    times = {"device": [], "host": []}
    for _ in range(args.samples):
        for name, fn in (("device", dev_path), ("host", host_path)):
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t1) * 1e3)
    res["score_batch_e2e"] = {
        "queries": len(qids), "targets_per_query": 100, "batch": B, "outputs_bit_identical": bool(same),
        **{f"{k}_ms": {"median": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1),
                       "samples": len(v)} for k, v in times.items()},
    }  # fmt: skip
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")
    return 0 if mism == 0 and same else 1


if __name__ == "__main__":
    sys.exit(main())
