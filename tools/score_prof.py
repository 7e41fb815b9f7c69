#!/usr/bin/env python
"""Diagnostic: one batch of all-items scoring on the ML-25M-shaped kNN model (run under ncu)."""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
import torch

from lkpy_b200 import _lib, data, engine, prep

n_q = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
dev = _lib.require_device()
inter = data.synth_interactions_cached(__import__("os").environ.get("LK_BENCH_DATA_CACHE"), **data.ML25M_SHAPE)
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
ui, iu, means = prep.knn_item_matrices_device(t(inter.users), t(inter.items), t(inter.ratings), inter.n_users, inter.n_items, True)
plan = engine.KnnBuildPlan.create(ui, iu)
cols, vals, cnt = plan.build_topk(1e-6, 20)
indptr, c, v = engine.topk_rows_to_csr(cols, vals, cnt)
st = engine.KnnScorerState.create(inter.n_items, indptr, c, v, dev)
R = inter.coo().tocsr()
a1 = int(R.indptr[n_q])
ref_ptr = t(R.indptr[: n_q + 1].astype(np.int64))
ri = t(R.indices[:a1].astype(np.int32))
rv = t((R.data[:a1] - means.cpu().numpy()[R.indices[:a1]]).astype(np.float32))
for ctas in ([int(x) for x in sys.argv[2].split(",")] if len(sys.argv) > 2 else [-1]):
    _lib.set_option("LK_KNN_SCORE_CTAS", ctas)
    for rep in range(2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        sc, ct = st.score_all_items(ref_ptr, ri, rv, 20, 1)
        e1.record()
        torch.cuda.synchronize()
        print(f"score_all_items {n_q} users, CTAs/SM option {ctas}: {e0.elapsed_time(e1):.2f} ms, scored fraction "
              f"{torch.isfinite(sc).float().mean().item():.4f}", flush=True)
        del sc, ct
