"""
EASE training and recommendation at the ML-25M shape (``data.ML25M_SHAPE``).

Reports, as one JSON line (and ``--out``):
  * ``EASEScorer.train``, whole (host clock around a synchronised call) and per stage with CUDA events: the Gram
    (co-occurrence count, diagonal, dense sink, regularisation), ``torch.linalg.cholesky_ex``,
    ``torch.cholesky_inverse`` and the normalisation; plus the allocator's peak over the whole call;
  * ``recommend_batch`` top-100 with ``exclude="query"`` for ``--users`` users: the kernel alone (CUDA events) and
    the whole call, with the algorithmic bytes 4 * n_items * sum |H_q|;
  * the unfused device baseline: dense 0/1 query vectors times W with cuBLAS (f32, TF32 off) in batches of
    ``--batch`` users, the history set to NaN, then ``lk_topn_columns``;
  * the reference's host statement ``q_vec @ weights`` (NumPy) on ``--host-sample`` users, when the host has room
    for a copy of W.
Medians over ``--reps`` runs; the kernel and the whole call are alternated.  The card name and power limit are
read in the same run.  Needs a GPU; there is no CPU fallback.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from lkpy_b200 import _lib, data, engine  # noqa: E402
from lkpy_b200.batch import history_csr  # noqa: E402
from lkpy_b200 import ease as ease_mod  # noqa: E402
from lkpy_b200.components import Dataset, ItemList  # noqa: E402
from lkpy_b200.ease import EASEScorer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)  # fmt: skip
    return {"card": q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"}


def _time(fn) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def _log(msg: str) -> None:
    print(msg, file=sys.stderr, flush=True)


def _train_stages(it, dev, reg: float = 1.0) -> dict:
    """The steps of ``EASEScorer.train``, one CUDA-event window each."""
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    out, t = {}, {}

    def gram():
        plan = engine.CoocPlan.create(it.n_users, it.n_items, up(it.users), up(it.items))
        indptr, cols, counts = plan.count(full_rows=False)
        g = plan.dense(indptr, cols, counts, plan.diagonal())
        g.diagonal().add_(reg)
        out["g"] = g

    t["gram_ms"] = _time(gram)
    g = out.pop("g")
    with torch.inference_mode():
        t["cholesky_ms"] = _time(lambda: out.setdefault("l", torch.linalg.cholesky_ex(g)))
        decomp, info = out.pop("l")
        assert int(info.item()) == 0
        t["inverse_ms"] = _time(lambda: torch.cholesky_inverse(decomp, out=g))
        del decomp
    t["normalise_ms"] = _time(lambda: ease_mod._normalise(g))
    del g
    return t


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--host-sample", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = _lib.require_device()
    torch.backends.cuda.matmul.allow_tf32 = False
    res = _card()
    it = data.synth_interactions(**data.ML25M_SHAPE)
    n_items = it.n_items
    ds = Dataset(it)
    _log("data ready")

    # training: the whole call and the staged statements, alternated
    whole, stages, peaks = [], [], []
    m = EASEScorer()
    for _rep in range(args.reps):
        m.__dict__.pop("_state", None)  # the previous weights must not count towards this call's peak
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        m.train(ds)
        torch.cuda.synchronize()
        whole.append(time.perf_counter() - t0)
        peaks.append(torch.cuda.max_memory_allocated())
        _log(f"train: {whole[-1]:.2f} s, peak {peaks[-1] / 1e9:.1f} GB")
        st = m._device_state()
        m.__dict__.pop("_state")  # the staged run below needs the room; the last state is kept aside
        torch.cuda.empty_cache()
        stages.append(_train_stages(it, dev))
        _log(f"stages: {stages[-1]}")
        m._state = st
        del st
    res["train"] = {"whole_s": float(np.median(whole)), "peak_allocated_GB": max(peaks) / 1e9,
                    **{k: float(np.median([s[k] for s in stages])) for k in stages[0]}}  # fmt: skip
    st = m._device_state()
    W = st.weights

    rng = np.random.default_rng(0)
    users = np.sort(rng.choice(it.n_users, min(args.users, it.n_users), replace=False))
    lo = np.searchsorted(it.users, users.astype(it.users.dtype))
    hi = np.searchsorted(it.users, (users + 1).astype(it.users.dtype))
    hist = [ItemList(item_nums=it.items[a:b], vocabulary=ds.items) for a, b in zip(lo, hi)]
    _has, h_ptr, h_items = history_csr(hist, ds.items, dev, unique=True)
    rows = int(h_items.numel())
    alg = 4 * n_items * rows
    _log(f"{len(users)} queries, {rows} history rows, {alg / 1e12:.3f} TB to read")
    _time(lambda: st.recommend(h_ptr, h_items, 100, h_ptr, h_items))  # warm-up
    m.recommend_batch(hist[:8], 100)
    kt, wt = [], []
    for _rep in range(args.reps):
        kt.append(_time(lambda: st.recommend(h_ptr, h_items, 100, h_ptr, h_items)))
        t0 = time.perf_counter()
        m.recommend_batch(hist, 100, exclude="query")
        wt.append(time.perf_counter() - t0)
        _log(f"recommend: kernel {kt[-1]:.1f} ms, whole call {wt[-1]:.2f} s")
    kms = float(np.median(kt))
    res["recommend"] = {"users": len(users), "n": 100, "history_rows": rows, "kernel_ms": kms,
                        "whole_call_s": float(np.median(wt)), "algorithmic_bytes": alg,
                        "GB_per_s": alg / kms / 1e6, "hbm_bound_ms": alg / HBM_BYTES_PER_S * 1e3}  # fmt: skip

    # unfused baseline: S^T = W^T X^T with cuBLAS per batch, history -> NaN, lk_topn_columns
    h_ptr_h, h_items_h = h_ptr.cpu().numpy(), h_items.cpu().numpy().astype(np.int64)

    def baseline():
        for b0 in range(0, len(users), args.batch):
            b1 = min(b0 + args.batch, len(users))
            a, z = int(h_ptr_h[b0]), int(h_ptr_h[b1])
            cols = torch.from_numpy(np.repeat(np.arange(b1 - b0), np.diff(h_ptr_h[b0 : b1 + 1]))).to(dev)
            r = torch.from_numpy(h_items_h[a:z]).to(dev)
            xt = torch.zeros((n_items, b1 - b0), dtype=torch.float32, device=dev)
            xt[r, cols] = 1.0
            s = W.t() @ xt
            s[r, cols] = float("nan")
            engine.topn_columns(s, 100)

    _time(baseline)  # warm-up
    bt = [_time(baseline) for _ in range(max(1, args.reps - 1))]
    res["unfused_baseline"] = {"batch": args.batch, "ms": float(np.median(bt))}
    _log(f"baseline: {res['unfused_baseline']}")

    # the reference's host statement, when the host can hold W
    need = 4 * n_items * n_items
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail > 2 * need:
        Wh = W.cpu().numpy()
        ht = []
        for k in range(args.host_sample):
            q_vec = np.zeros(n_items, dtype=np.float32)
            q_vec[h_items_h[int(h_ptr_h[k]) : int(h_ptr_h[k + 1])]] = 1.0
            t0 = time.perf_counter()
            _ = q_vec @ Wh
            ht.append(time.perf_counter() - t0)
        res["host_q_vec_matmul_per_query_ms"] = 1e3 * float(np.median(ht))
        res["host_queries"] = len(ht)
        del Wh
    else:
        res["host_q_vec_matmul_per_query_ms"] = None  # not measured: no room for a host copy of W
        res["host_available_GB"] = avail / 1e9
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
