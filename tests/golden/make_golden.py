#!/usr/bin/env python
"""
Generate the committed golden fixtures in this directory.

Run with ``LENSKIT_REFERENCE_SRC`` naming a LensKit source checkout; nothing at test,
smoke or bench time reads the reference tree.  The reference package cannot be
imported as a whole here (its Rust extension ``lenskit._accel`` is not built and
several Python dependencies are absent), so the pure-Python reference functions
that restate the hot-path arithmetic are *executed from the reference's own
source*: each function's source segment is pulled out of the reference file with
``ast`` and compiled in a namespace holding NumPy/SciPy.  No reference source is
copied into this repository; only the numbers they produce are.

Outputs
-------
ml_small.npz            ml-latest-small ratings, ids numbered by sorted unique id
item-item-preds.csv     the reference's own golden predictions
                        (tests/models/item-item-preds.csv, consumed by
                        tests/models/test_knn_item_item.py:413-453)
als_ref_rows.npz        per-row ALS solves from the reference's fold-in code
                        (_train_new_row als/_implicit.py:91-130, _implicit_otor
                        :177-184, _train_bias_row_cholesky als/_explicit.py:121-147,
                        solve_cholesky math/solve.py:17-41) on seeded inputs
knn_prep.npz            ItemKNNScorer._center_ratings / _normalize_rows
                        (knn/item.py:202-228) on the toy set of
                        tests/models/test_knn_item_item.py:30-49 and on
                        ml-latest-small (sha256 + leading values)
"""

from __future__ import annotations

import os
import ast
import hashlib
import shutil
import warnings
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pandas as pd
import scipy.sparse.linalg as spla
from scipy.linalg import cho_factor, cho_solve
from scipy.sparse import coo_array, sparray

REF = Path(os.environ["LENSKIT_REFERENCE_SRC"])  # a LensKit source checkout
OUT = Path(__file__).resolve().parent


def extract(path: Path, name: str, cls: str | None = None) -> str:
    src = path.read_text()
    tree = ast.parse(src)
    body = tree.body
    if cls is not None:
        (cnode,) = [n for n in body if isinstance(n, ast.ClassDef) and n.name == cls]
        body = cnode.body
    (fn,) = [n for n in body if isinstance(n, ast.FunctionDef) and n.name == name]
    fn.decorator_list = []
    fn.returns = None
    for a in fn.args.args + fn.args.kwonlyargs:
        a.annotation = None
    return ast.unparse(fn)


class _Quiet:
    def __getattr__(self, _name):
        return lambda *a, **k: None


def ref_namespace() -> dict:
    ns: dict = {
        "np": np,
        "spla": spla,
        "cho_factor": cho_factor,
        "cho_solve": cho_solve,
        "coo_array": coo_array,
        "sparray": sparray,
        "warnings": warnings,
        "DataWarning": UserWarning,
        "max_memory": lambda: "n/a",
        "NPMatrix": object,
        "NPVector": object,
    }
    src = REF / "src" / "lenskit"
    exec(extract(src / "math" / "solve.py", "solve_cholesky"), ns)
    exec(extract(src / "als" / "_implicit.py", "_implicit_otor"), ns)
    exec(extract(src / "als" / "_implicit.py", "_train_new_row", "ImplicitMFScorer"), ns)
    exec(extract(src / "als" / "_explicit.py", "_train_bias_row_cholesky"), ns)
    exec(extract(src / "knn" / "item.py", "_center_ratings", "ItemKNNScorer"), ns)
    exec(extract(src / "knn" / "item.py", "_normalize_rows", "ItemKNNScorer"), ns)
    return ns


def make_ml_small():
    r = pd.read_csv(REF / "data" / "ml-latest-small" / "ratings.csv")
    user_ids = np.sort(r.userId.unique())
    item_ids = np.sort(r.movieId.unique())
    users = np.searchsorted(user_ids, r.userId.values).astype(np.int16)
    items = np.searchsorted(item_ids, r.movieId.values).astype(np.int16)
    halves = np.rint(r.rating.values * 2).astype(np.uint8)
    assert np.all(halves * 0.5 == r.rating.values)
    np.savez_compressed(
        OUT / "ml_small.npz",
        users=users,
        items=items,
        rating_halves=halves,
        user_ids=user_ids.astype(np.int32),
        item_ids=item_ids.astype(np.int32),
    )
    shutil.copyfile(REF / "tests" / "models" / "item-item-preds.csv", OUT / "item-item-preds.csv")
    return users.astype(np.int32), items.astype(np.int32), halves.astype(np.float32) * 0.5


def make_als_rows(ns):
    rng = np.random.default_rng(20260924)
    dummy = SimpleNamespace(logger=_Quiet())
    out = {}
    cases = [(8, 5, 40), (32, 71, 200), (64, 3, 120), (64, 200, 400), (64, 1, 50), (128, 150, 220)]
    for ci, (k, n, c) in enumerate(cases):
        other = (rng.standard_normal((c, k)).astype(np.float32) * np.float32(0.1)).astype(np.float32)
        items = np.sort(rng.choice(c, size=n, replace=False)).astype(np.int32)
        # implicit: confidence values (already multiplied by weight)
        conf = (np.float32(40.0) * rng.choice([1.0, 2.5, 4.0], size=n)).astype(np.float32)
        reg = 0.1
        otor = ns["_implicit_otor"](other, reg)
        x_imp = ns["_train_new_row"](dummy, items, conf, other, otor)
        # explicit: bias-removed ratings
        rates = rng.standard_normal(n).astype(np.float32)
        x_exp = ns["_train_bias_row_cholesky"](items, rates, other, np.float32(reg))
        out[f"c{ci}_k"] = np.int32(k)
        out[f"c{ci}_other"] = other
        out[f"c{ci}_items"] = items
        out[f"c{ci}_conf"] = conf
        out[f"c{ci}_rates"] = rates
        out[f"c{ci}_reg"] = np.float64(reg)
        out[f"c{ci}_otor"] = np.asarray(otor, dtype=np.float32)
        out[f"c{ci}_x_implicit"] = np.asarray(x_imp, dtype=np.float32)
        out[f"c{ci}_x_explicit"] = np.asarray(x_exp, dtype=np.float32)
    out["n_cases"] = np.int32(len(cases))
    np.savez_compressed(OUT / "als_ref_rows.npz", **out)


def _prep(ns, rmat, explicit):
    dummy = SimpleNamespace(config=SimpleNamespace(explicit=explicit))
    log = _Quiet()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cmat, means = ns["_center_ratings"](dummy, log, None, rmat)
    nmat = ns["_normalize_rows"](dummy, log, None, cmat)
    ui = nmat.tocsr()
    ui.sort_indices()
    iu = nmat.T.tocsr()
    iu.sort_indices()
    return ui, iu, means


def make_knn_prep(ns, users, items, ratings):
    out = {}
    # toy data from the reference's test (user, item, rating)
    toy = np.array(
        [
            (1, 6, 4.0), (2, 6, 2.0), (1, 7, 3.0), (2, 7, 2.0), (3, 7, 5.0), (4, 7, 2.0),
            (1, 8, 3.0), (2, 8, 4.0), (3, 8, 3.0), (4, 8, 2.0), (5, 8, 3.0), (6, 8, 2.0),
            (1, 9, 3.0), (3, 9, 4.0),
        ]
    )  # fmt: skip
    tu = toy[:, 0].astype(np.int32) - 1
    ti = toy[:, 1].astype(np.int32) - 6
    tr = toy[:, 2].astype(np.float32)
    for tag, explicit in (("exp", True), ("imp", False)):
        vals = tr if explicit else np.ones_like(tr)
        ui, iu, means = _prep(ns, coo_array((vals, (tu, ti)), shape=(6, 4)).astype(np.float32), explicit)
        out[f"toy_{tag}_ui_indptr"] = ui.indptr.astype(np.int32)
        out[f"toy_{tag}_ui_indices"] = ui.indices.astype(np.int32)
        out[f"toy_{tag}_ui_data"] = ui.data.astype(np.float32)
        if means is not None:
            out[f"toy_{tag}_means"] = np.asarray(means, dtype=np.float32)

        vals = ratings if explicit else np.ones_like(ratings)
        nu, ni = users.max() + 1, items.max() + 1
        ui, iu, means = _prep(
            ns, coo_array((vals.astype(np.float32), (users, items)), shape=(nu, ni)).astype(np.float32), explicit
        )
        out[f"ml_{tag}_ui_sha256"] = np.array(
            hashlib.sha256(ui.data.astype(np.float32).tobytes()).hexdigest()
        )
        out[f"ml_{tag}_iu_sha256"] = np.array(
            hashlib.sha256(iu.data.astype(np.float32).tobytes()).hexdigest()
        )
        out[f"ml_{tag}_ui_head"] = ui.data[:4096].astype(np.float32)
        if means is not None:
            out[f"ml_{tag}_means"] = np.asarray(means, dtype=np.float32)
    out["toy_users"] = tu
    out["toy_items"] = ti
    out["toy_ratings"] = tr
    np.savez_compressed(OUT / "knn_prep.npz", **out)


if __name__ == "__main__":
    ns = ref_namespace()
    u, i, r = make_ml_small()
    make_als_rows(ns)
    make_knn_prep(ns, u, i, r)
    for f in sorted(OUT.iterdir()):
        print(f.name, f.stat().st_size)
