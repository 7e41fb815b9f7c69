"""
BiasedSVD training and recommendation at the ML-25M shape (``data.ML25M_SHAPE``, the generator's ratings), k = 64,
n_iter = 5.

Reports, as one JSON line (and ``--out``):
  * ``BiasedSVDScorer.train``, whole (host clock around a synchronised call), and per stage: the bias model and the
    device residual matrix (host clock, synchronised), then with CUDA events the power-iteration products, the LUs,
    the QR, the projection product, the SVD, the sign flip and the final transform ``X @ components_.T``;
  * ``lk_spmm`` alone at W = k + 10 for both orientations (median of ``--reps``), with its rate by counted bytes
    ``nnz * (8 + 4 W) + rows * 4 W`` (indices, values and one gathered row of D per nonzero, one written row of Y per
    row).  The gathered operand is reused from L2 (the 59k-row D is 17.5 MB, inside the 50 MB L2), so this is a
    rate over counted bytes, not a share of HBM bandwidth;
  * scikit-learn's ``TruncatedSVD`` on the same residual matrix on the host, one run from the same global NumPy
    state, and the device result's singular values and sampled users' scores against it ("not available" without
    scikit-learn, skipped with ``--no-host``);
  * ``recommend_batch`` top-100 with ``exclude="query"`` for ``--users`` users, whole call.
The card name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from lkpy_b200 import _lib, data, engine, svd  # noqa: E402
from lkpy_b200.basic import BiasModel  # noqa: E402
from lkpy_b200.components import Dataset, ItemList, RecQuery  # noqa: E402


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


class _Stages:
    """``stage(name)`` for ``engine.randomized_svd``: CUDA events around each step, summed per name."""

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
        return {f"{k}_ms": sum(s.elapsed_time(e) for s, e in v) for k, v in self.events.items()} | {
            f"{k}_count": len(v) for k, v in self.events.items()
        }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=64)
    ap.add_argument("--n-iter", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--users", type=int, default=32768)
    ap.add_argument("--no-host", action="store_true", help="skip scikit-learn's host run")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = _lib.require_device()
    torch.backends.cuda.matmul.allow_tf32 = False
    res = _card() | {"k": args.k, "n_iter": args.n_iter}
    it = data.synth_interactions(**data.ML25M_SHAPE)
    ds = Dataset(it)
    k, W = args.k, args.k + svd.N_OVERSAMPLES
    res["shape"] = {"users": it.n_users, "items": it.n_items, "nnz": int(it.nnz)}
    _log(f"data ready: {res['shape']}")

    # whole train (a warm-up first: cuSOLVER and the module load)
    m = svd.BiasedSVDScorer(embedding_size=k, n_iter=args.n_iter)
    np.random.seed(0)
    m.train(ds)
    whole = []
    for _rep in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        np.random.seed(0)
        m.train(ds)
        torch.cuda.synchronize()
        whole.append(time.perf_counter() - t0)
        _log(f"train: {whole[-1]:.2f} s")
    res["train_whole_s"] = float(np.median(whole))

    # staged train
    staged = []
    for _rep in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        bias = BiasModel.learn(it, 5.0, np.float32)
        t1 = time.perf_counter()
        x = svd.residual_operand(bias, it, dev)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        np.random.seed(0)
        q0 = np.random.normal(size=(min(it.n_users, it.n_items), W)).astype(np.float32)
        d_q0 = torch.from_numpy(q0).to(dev)
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        st = _Stages()
        vt, s = engine.randomized_svd(x, d_q0, k, args.n_iter, st)
        with st("transform"):
            uc = x.mul(vt.T.contiguous())
        r = {"bias_s": t1 - t0, "residuals_s": t2 - t1, "start_matrix_s": t3 - t2} | st.totals_ms()
        staged.append(r)
        _log(f"stages: {r}")
    res["train_stages"] = {key: float(np.median([r[key] for r in staged])) for key in staged[0]}

    # lk_spmm alone at width W, both orientations
    rng = np.random.default_rng(1)
    spmm = {}
    for name, csr, order in (("ui", x.rows, x.rows_order), ("iu", x.cols, x.cols_order)):
        d = torch.from_numpy(rng.standard_normal((csr.shape[1], W)).astype(np.float32)).to(dev)
        engine.spmm(csr, order, d)
        ms = float(np.median([_time(lambda: engine.spmm(csr, order, d)) for _ in range(max(args.reps, 5))]))
        counted = csr.nnz * (8 + 4 * W) + csr.shape[0] * 4 * W
        spmm[name] = {"rows": csr.shape[0], "W": W, "ms": ms, "counted_bytes": counted, "GB_per_s": counted / ms / 1e6}
        _log(f"lk_spmm {name}: {spmm[name]}")
    res["spmm"] = spmm

    # scikit-learn on the host, from the same global state
    sample_users = np.sort(rng.choice(it.n_users, 64, replace=False))
    if args.no_host:
        res["sklearn"] = "not measured"
    else:
        try:
            from sklearn.decomposition import TruncatedSVD
        except ImportError:
            TruncatedSVD = None
        if TruncatedSVD is None:
            res["sklearn"] = "not available"
        else:
            import scipy.sparse as sps

            X = sps.csr_array((x.rows.values.cpu().numpy(), x.rows.indices.cpu().numpy(), x.rows.h_indptr),
                              shape=x.shape)  # fmt: skip
            np.random.seed(0)
            t0 = time.perf_counter()
            f = TruncatedSVD(k, algorithm="randomized", n_iter=args.n_iter)
            xt = f.fit_transform(X)
            host_s = time.perf_counter() - t0
            ours = uc[torch.from_numpy(sample_users).to(dev)].cpu().numpy().astype(np.float64) @ vt.cpu().numpy()
            theirs = xt[sample_users].astype(np.float64) @ f.components_
            res["sklearn"] = {
                "version": __import__("sklearn").__version__,
                "fit_transform_s": host_s,
                "singular_values_max_rel": float(np.abs(s.cpu().numpy() / f.singular_values_ - 1).max()),
                "sampled_scores_rel_frobenius": float(np.linalg.norm(ours - theirs) / np.linalg.norm(theirs)),
                "sampled_users": len(sample_users),
            }  # fmt: skip
        _log(f"sklearn: {res['sklearn']}")

    # recommend_batch top-100, exclude="query"
    users = np.sort(rng.choice(it.n_users, min(args.users, it.n_users), replace=False))
    lo = np.searchsorted(it.users, users.astype(it.users.dtype))
    hi = np.searchsorted(it.users, (users + 1).astype(it.users.dtype))
    queries = [RecQuery(ds.users.id(u), ItemList(item_nums=it.items[a:b], vocabulary=ds.items))
               for u, a, b in zip(users, lo, hi)]  # fmt: skip
    m.recommend_batch(queries[:8], 100, exclude="query")
    wt = []
    for _rep in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.recommend_batch(queries, 100, exclude="query")
        torch.cuda.synchronize()
        wt.append(time.perf_counter() - t0)
        _log(f"recommend: whole call {wt[-1]:.2f} s")
    res["recommend"] = {"users": len(users), "n": 100, "exclude": "query", "whole_call_s": float(np.median(wt))}

    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
