"""
SLIM training and recommendation on one GPU.

Reports, as one JSON line (and ``--out``):
  * the whole ``SLIMScorer.train`` at the ML-25M shape (``data.ML25M_SHAPE``) with fsSLIM ``max_nbrs=100``,
    ``max_iters=10``;
  * the whole ``SLIMScorer.train`` of full SLIM (the defaults) on ml-latest-small;
  * full SLIM on a fixed cost-stratified sample of target items at the ML-25M shape (the most expensive item
    included): ``SlimPlan.train`` on the device against the C restatement (``tests/slim_oracle.c``, OpenMP on every
    CPU thread) on the same sample, with a bit-for-bit comparison;
  * ``recommend_batch`` top-100 with ``exclude="query"`` for ``--users`` users at the ML-25M shape (fsSLIM weights):
    the scoring kernel alone and the whole call.
The card name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.
"""

from __future__ import annotations

import argparse
import importlib.util
import json
import os
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
from lkpy_b200.slim import SLIMScorer  # noqa: E402

#: positions in the descending-cost order of the sampled target items
SAMPLE_RANKS = [0, 1, 10, 100, 1000, 5000, 20000, 40000]


def _card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)  # fmt: skip
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _oracle():
    spec = importlib.util.spec_from_file_location("slim_oracle", ROOT / "tests" / "slim_oracle.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t) * 1000.0


def _log(msg: str) -> None:
    print(msg, file=sys.stderr, flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = _lib.require_device()
    so = _oracle()
    res: dict = {"card": _card(), "cpu_threads": os.cpu_count()}

    small = data.load_ml_small()
    m = SLIMScorer()
    m.train(Dataset(small))  # warm-up: module load, allocator
    _m, res["ml_small_full_train_ms"] = _wall(lambda: SLIMScorer().train(Dataset(small)))
    _log(f"ml-small full SLIM: {res['ml_small_full_train_ms']:.1f} ms")

    it = data.synth_interactions(**data.ML25M_SHAPE, ratings=False)
    fs = SLIMScorer(max_nbrs=100, max_iters=10)
    _r, res["ml25m_fsslim100_train_ms"] = _wall(lambda: fs.train(Dataset(it)))
    res["ml25m_fsslim100_nnz"] = int(fs._state.indptr[-1].item())
    _log(f"ML-25M fsSLIM k=100, 10 iterations: {res['ml25m_fsslim100_train_ms']:.1f} ms")

    ui = so.structure(it.n_users, it.users, it.items)
    iu = so.structure(it.n_items, it.items, it.users)
    cost = np.bincount(it.items, weights=np.diff(ui[0])[it.users], minlength=it.n_items)
    cols = np.argsort(-cost, kind="stable")[SAMPLE_RANKS]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    plan = engine.SlimPlan.create(it.n_users, it.n_items, t(ui[0]), t(ui[1]), t(iu[0]), t(iu[1]), 1.0, 1.0, 100, None,
                                  columns=t(cols))  # fmt: skip
    got, res["sample_full_gpu_ms"] = _wall(plan.train)
    tc = time.perf_counter()
    want = so.train(it.n_users, it.n_items, ui, iu, 1.0, 1.0, 100, None, columns=cols)
    res["sample_full_cpu_ms"] = (time.perf_counter() - tc) * 1000.0
    ip, c, v = (x.cpu().numpy() for x in got)
    res["sample_items"] = [int(x) for x in cols]
    res["sample_nnz"] = int(want.nnz)
    res["sample_bit_exact"] = bool(np.array_equal(ip, want.indptr) and np.array_equal(c, want.indices)
                                   and np.array_equal(v.view(np.int32), want.data.view(np.int32)))  # fmt: skip
    _log(f"sample full SLIM: GPU {res['sample_full_gpu_ms']:.1f} ms, CPU {res['sample_full_cpu_ms']:.1f} ms")

    rng = np.random.default_rng(0)
    users = np.sort(rng.choice(it.n_users, size=min(args.users, it.n_users), replace=False))
    starts = np.searchsorted(it.users, users)
    ends = np.searchsorted(it.users, users, side="right")
    hists = [it.items[a:b] for a, b in zip(starts, ends)]
    st = fs._device_state()
    r_ptr = torch.from_numpy(np.concatenate([[0], np.cumsum([len(h) for h in hists])]).astype(np.int64)).to(dev)
    r_items = torch.from_numpy(np.concatenate(hists).astype(np.int32)).to(dev)
    st.recommend(r_ptr, r_items, 2, 100, r_ptr, r_items)  # warm-up
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    st.recommend(r_ptr, r_items, 2, 100, r_ptr, r_items)
    e.record()
    e.synchronize()
    res["recommend_top100_kernel_ms"] = s.elapsed_time(e)
    qs = [ItemList(item_nums=h, vocabulary=fs.items) for h in hists]
    fs.recommend_batch(qs[:64], 100)
    _r, res["recommend_top100_call_ms"] = _wall(lambda: fs.recommend_batch(qs, 100))
    res["recommend_users"] = len(qs)
    # algorithmic bytes of scoring: 8 B (column, value) per weight entry of every history row read
    nnz_row = np.diff(st.indptr.cpu().numpy())
    res["recommend_bytes"] = int(8 * nnz_row[np.concatenate(hists)].sum())
    _log(f"recommend top-100, {len(qs)} users: kernel {res['recommend_top100_kernel_ms']:.1f} ms, "
         f"call {res['recommend_top100_call_ms']:.1f} ms")  # fmt: skip

    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
