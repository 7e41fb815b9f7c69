"""
Co-occurrence counting and association recommendation at the ML-25M shape (``data.ML25M_SHAPE``).

Reports, as one JSON line (and ``--out``):
  * the whole ``CoocPlan.count`` call (row costs, schedule, count kernel, pool -> CSR gather) for the strict upper
    triangle (``count_cooc``'s device part) and for full rows with the lift values (``AssociationScorer.train``'s),
    medians of alternated runs, with the nnz produced and the algorithmic
    bytes (4 B per pair update for the column reads, 8 B per entry written);
  * the whole ``AssociationScorer.train``;
  * ``recommend_batch`` top-100 with ``exclude="query"`` for ``--users`` users: the kernel alone and the whole call,
    with the algorithmic bytes (8 B per association entry read);
  * the host path (``__call__``'s dense rows and ``np.mean`` restated) on ``--host-sample`` queries.
The card name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.
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

from lkpy_b200 import _lib, data, engine  # noqa: E402
from lkpy_b200.association import AssociationScorer  # noqa: E402
from lkpy_b200.components import Dataset, ItemList  # noqa: E402


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


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--host-sample", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = _lib.require_device()
    res = _card()
    it = data.synth_interactions(**data.ML25M_SHAPE)
    _log("data ready")
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    plan = engine.CoocPlan.create(it.n_users, it.n_items, up(it.users), up(it.items))
    counts = np.bincount(it.items, minlength=it.n_items).astype(np.int32)
    d_counts = up(counts)
    upd = {False: int(plan.row_cost(False).sum()), True: int(plan.row_cost(True).sum())}
    nnz, t = {}, {False: [], True: []}
    for _rep in range(args.reps + 1):  # the first round warms up
        for full in (False, True):
            kw = dict(method=_lib.LK_ASSOC_LIFT, item_count=d_counts) if full else {}
            out = {}
            t[full].append(_time(lambda: out.setdefault("r", plan.count(full_rows=full, **kw))))  # noqa: B023
            nnz[full] = int(out["r"][0][-1])
            del out
            _log(f"count full_rows={full}: {t[full][-1]:.1f} ms, nnz {nnz[full]}")
    for full, name in ((False, "count_upper"), (True, "count_full_lift")):
        ms = float(np.median(t[full][1:]))
        res[name] = {"ms_whole_count_call": ms, "pair_updates": upd[full], "nnz": nnz[full],
                     "algorithmic_bytes": 4 * upd[full] + 8 * nnz[full],
                     "GB_per_s": (4 * upd[full] + 8 * nnz[full]) / ms / 1e6}  # fmt: skip
    del plan
    torch.cuda.empty_cache()

    ds = Dataset(it)
    m = AssociationScorer(method="lift")
    t0 = time.perf_counter()
    m.train(ds)
    torch.cuda.synchronize()
    res["train_s"] = time.perf_counter() - t0
    _log(f"train: {res['train_s']:.2f} s")
    st = m._device_state()

    rng = np.random.default_rng(0)
    users = np.sort(rng.choice(it.n_users, min(args.users, it.n_users), replace=False))
    # the users' histories from one vectorised search (Dataset.user_history searches per call with a type promotion
    # that copies the whole user column each time)
    lo = np.searchsorted(it.users, users.astype(it.users.dtype))
    hi = np.searchsorted(it.users, (users + 1).astype(it.users.dtype))
    hist = [ItemList(item_nums=it.items[a:b], vocabulary=ds.items) for a, b in zip(lo, hi)]
    refs = [h.numbers() for h in hist]
    _log("histories ready")
    r_ptr = up(np.concatenate([[0], np.cumsum([len(r) for r in refs])]).astype(np.int64))
    r_items = up(np.concatenate(refs).astype(np.int32))
    h_ip = st.indptr.cpu().numpy()
    entries = int(sum(int((h_ip[r + 1] - h_ip[r]).sum()) for r in refs))
    _log(f"{len(users)} queries ready, {entries} association entries to read")
    _time(lambda: st.recommend(r_ptr, r_items, 0, 100, r_ptr, r_items))  # warm-up
    _log("warm-up done")
    kt, wt = [], []
    for _rep in range(args.reps):
        kt.append(_time(lambda: st.recommend(r_ptr, r_items, 0, 100, r_ptr, r_items)))
        t0 = time.perf_counter()
        m.recommend_batch(hist, 100, exclude="query")
        wt.append(time.perf_counter() - t0)
        _log(f"recommend: kernel {kt[-1]:.1f} ms, whole call {wt[-1]:.2f} s")
    kms = float(np.median(kt))
    res["recommend"] = {"users": len(users), "n": 100, "kernel_ms": kms, "whole_call_s": float(np.median(wt)),
                        "assoc_entries_read": entries, "algorithmic_bytes": 8 * entries,
                        "GB_per_s": 8 * entries / kms / 1e6}  # fmt: skip

    # host path: __call__'s dense rows (assoc_scores[ref_items, :].todense()) and np.mean, on rows copied out of the
    # device matrix beforehand
    ht = []
    for r in refs[: args.host_sample]:
        rows = [(st.cols[int(h_ip[x]) : int(h_ip[x + 1])].cpu().numpy(), st.vals[int(h_ip[x]) : int(h_ip[x + 1])].cpu().numpy())
                for x in r]  # fmt: skip
        t0 = time.perf_counter()
        dense = np.zeros((len(r), it.n_items), dtype=np.float32)
        for k, (c, v) in enumerate(rows):
            dense[k, c] = v
        s = np.mean(dense, axis=0)
        s[r] = np.nan
        _ = np.argsort(-s, kind="stable")[:100]
        ht.append(time.perf_counter() - t0)
    res["host_path_per_query_ms"] = 1e3 * float(np.median(ht))
    res["host_path_queries"] = len(ht)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
