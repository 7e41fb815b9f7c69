"""
The function-level drop-in of INTEGRATION.md §1 checked against the reference's OWN classes: ``lenskit.training``,
``pipeline.components.Component``, ``data.matrix.SparseRowArray``, ``als._common`` / ``als._implicit`` and
``knn.item`` / ``knn.user`` run with ``lenskit._accel`` bound to ``lkpy_b200.accel``, and what they produce —
trained factors, the similarity matrix, scores, top-N order, wire format, the protocol names they use — is
compared with what this package computes on the same inputs.

The reference's side comes from one of two places.  With a lenskit/lkpy source checkout
(``LENSKIT_REFERENCE_SRC``, or a ``reference`` directory beside the repository; tests/ref_sandbox.py) it is
computed live, the classes are exercised end to end, and ``LK_RECORD_REFERENCE_GOLDEN=1`` rewrites the golden
files.  Without one it is read from ``tests/golden/reference_classes/``, recorded from that checkout (on a
machine without a GPU, where the device part of the two entry points is the oracle).
"""

import ast
import os
from pathlib import Path
import warnings

import numpy as np
import pytest
import scipy.sparse as sps
import torch

import oracle
import ref_sandbox
from helpers import implicit_init
from lkpy_b200 import accel, data

GOLD = Path(__file__).resolve().parent / "golden" / "reference_classes"
RECORD = os.environ.get("LK_RECORD_REFERENCE_GOLDEN") == "1"
ROWS_U = np.random.default_rng(0).choice(671, 120, replace=False)
ROWS_I = np.random.default_rng(1).choice(9066, 300, replace=False)


def _theirs(name: str, ref, live) -> dict:
    """The reference's values: ``live()`` run against the checkout when there is one, else the golden file."""
    if ref is None:
        with np.load(GOLD / f"{name}.npz") as z:
            return {k: z[k] for k in z.files}
    vals = {k: np.asarray(v) for k, v in live().items()}
    if RECORD:
        GOLD.mkdir(exist_ok=True)
        np.savez_compressed(GOLD / f"{name}.npz", **vals)
    return vals


@pytest.fixture(scope="module")
def ref():
    if not ref_sandbox.available():
        with pytest.MonkeyPatch.context() as mp:
            if not torch.cuda.is_available():
                _oracle_compute(mp)
            yield None
        return
    with ref_sandbox.reference_modules() as mods, warnings.catch_warnings(), pytest.MonkeyPatch.context() as mp:
        warnings.simplefilter("ignore")  # "not the short import path": the sandbox has no lenskit/__init__
        if not torch.cuda.is_available():
            _oracle_compute(mp)
        yield mods


def _oracle_compute(monkeypatch):
    """No GPU here: keep the entry points' own argument handling, swap the device part for the oracle."""

    def als_task(mode, matrix, this, other, otor, reg):
        this = accel._check_factor("this", this, writable=True)
        other = accel._check_factor("other", other)
        csr = accel.as_host_csr(matrix)  # the reference's SparseRowArray
        assert csr.shape == (this.shape[0], other.shape[0])

        def run(_task):
            if mode == accel._lib.LK_ALS_IMPLICIT:
                new, delta = oracle.als_half("implicit", csr, this, other, otor_mat=otor)
            else:
                new, delta = oracle.als_half("explicit", csr, this, other, reg=reg)
            this[...] = new  # in place, like implicit.rs:57-64
            return float(delta)

        return accel.AccelTask(run, total=this.shape[0])

    def compute_similarities(ui_ratings, iu_ratings, shape, min_sim, save_nbrs):
        nu, ni = shape
        ui, iu = accel.as_host_csr(ui_ratings, ni), accel.as_host_csr(iu_ratings, nu)
        assert ui.shape == (nu, ni) and iu.shape == (ni, nu)

        def run(_task):
            S = oracle.knn_build(ui, iu, min_sim, save_nbrs)
            out = data.InteractionCSR(S.indptr.astype(np.int64), S.indices, S.data, (ni, ni))
            return accel.csr_to_arrow_chunks(out, 2000)

        return accel.AccelTask(run, total=ni)

    class CpuScorerState:
        """``engine.KnnScorerState`` with the oracle behind ``score``: accel._score runs unchanged around it."""

        def __init__(self, n_items, indptr, cols, vals, user_mode):
            n_rows = len(indptr) - 1
            self.explicit = vals is not None
            v = np.asarray(vals) if vals is not None else np.ones(len(cols), np.float32)
            self.S = sps.csr_array((v, np.asarray(cols), np.asarray(indptr)), shape=(n_rows, n_items))
            self.user_mode = user_mode

        @classmethod
        def create(cls, n_items, indptr, cols, vals, _dev, user_mode=False):
            return cls(n_items, indptr, cols, vals, user_mode)

        def score(self, _ref_ptr, ref_items, ref_vals, _tgt_ptr, tgt_items, max_nbrs, min_nbrs):
            if self.user_mode:  # the "history" is the neighbour list and carries the weights (user_score.rs:21-98)
                sc, ct = oracle.user_score(self.S, ref_items.numpy(), ref_vals.numpy(), tgt_items.numpy(), max_nbrs,
                                           min_nbrs, explicit=self.explicit)  # fmt: skip
            else:
                sc, ct = oracle.knn_score(self.S, ref_items.numpy(), None if ref_vals is None else ref_vals.numpy(),
                                          tgt_items.numpy(), max_nbrs, min_nbrs)  # fmt: skip
            return torch.from_numpy(sc), torch.from_numpy(ct)

    def argtopn_batch(scores, n):
        return [oracle.argtopn(np.ascontiguousarray(row, dtype=np.float32), int(min(n, len(row)))) for row in np.asarray(scores)]

    monkeypatch.setattr(accel, "argtopn_batch", argtopn_batch)
    monkeypatch.setattr(accel, "_als_task", als_task)
    monkeypatch.setattr(accel.knn, "compute_similarities", compute_similarities)
    monkeypatch.setattr(accel._lib, "require_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(accel.engine, "KnnScorerState", CpuScorerState)


@pytest.fixture(scope="module")
def ml_small():
    return data.load_ml_small()


def _np_otor(other: np.ndarray, reg: float) -> np.ndarray:
    """OᵀO + reg·I in f32 NumPy arithmetic, as the reference's trainer forms it (als/_implicit.py:177-184): the
    first epochs from the tiny initial factors are ill-conditioned enough to amplify any other summation order."""
    o = other.T @ other
    o += np.eye(other.shape[1], dtype=other.dtype) * np.float32(reg)
    return o


def _tol():
    return 1e-4 if torch.cuda.is_available() else 1e-5


def test_reference_implicit_mf_trains_through_the_shim(ref, ml_small):
    """``ImplicitMFScorer.train`` (training.py:301-334 -> als/_common.py:209-256 -> als/_implicit.py:158-164):
    the reference's trainer builds R and Rᵀ as SparseRowArrays, initialises the factors (items first) and
    calls ``als.train_implicit_matrix`` once per half-epoch; the factors it ends with are those of the same
    half-steps computed directly from the same initialisation."""
    k, epochs = 16, 2

    def live():
        imp, training = ref["lenskit.als._implicit"], ref["lenskit.training"]
        m = imp.ImplicitMFScorer(embedding_size=k, epochs=epochs, regularization=0.1, weight=40)
        assert type(m).train is training.UsesTrainer.train  # the reference's epoch loop, not ours
        trainer = m.create_trainer(ref_sandbox.FakeDataset(ml_small), training.TrainingOptions(rng=42))
        assert isinstance(trainer, imp.ImplicitMFTrainer)
        assert type(trainer.ui_rates).__name__ == "SparseRowArray" and trainer.ui_rates.shape == (ml_small.n_users, ml_small.n_items)
        p0, q0 = m.user_embeddings.copy(), m.item_embeddings.copy()
        p_arr, q_arr = m.user_embeddings, m.item_embeddings
        for _ in range(epochs):
            metrics = trainer.train_epoch()
            assert set(metrics) == {"deltaP", "deltaQ"} and all(np.isfinite(v) and v > 0 for v in metrics.values())
        assert m.user_embeddings is p_arr and m.item_embeddings is q_arr  # mutated in place (TrainContext.left)
        trainer.finalize()
        assert m._OtOr.shape == (k, k)
        return {"p0": p0[ROWS_U], "q0": q0[ROWS_I], "p": p_arr[ROWS_U], "q": q_arr[ROWS_I]}

    theirs = _theirs("implicit_mf_train", ref, live)
    ui, iu = data.als_implicit_matrices(ml_small, 40.0)
    p, q = implicit_init(np.random.default_rng(42), ml_small.n_items, ml_small.n_users, k)
    assert np.array_equal(p[ROWS_U], theirs["p0"]) and np.array_equal(q[ROWS_I], theirs["q0"])  # the same init
    for _ in range(epochs):
        p, _ = oracle.als_half("implicit", ui, p, q, otor_mat=_np_otor(q, 0.1))
        q, _ = oracle.als_half("implicit", iu, q, p, otor_mat=_np_otor(p, 0.1))
    assert np.linalg.norm(theirs["p"] - p[ROWS_U]) <= _tol() * np.linalg.norm(p[ROWS_U])
    assert np.linalg.norm(theirs["q"] - q[ROWS_I]) <= _tol() * np.linalg.norm(q[ROWS_I])


def test_reference_item_knn_trains_through_the_shim(ref, ml_small):
    """``ItemKNNScorer.train`` (knn/item.py:121-199): the reference centres and normalises, hands two
    SparseRowArrays to ``knn.compute_similarities``, concatenates the returned chunks and wraps them with
    ``SparseRowArray.from_array`` — which only accepts an index field of the ``lenskit.sparse_index``
    extension type (data/matrix.py:530-546).  The model it stores is the oracle's, bit for bit."""

    def live():
        knn, training = ref["lenskit.knn.item"], ref["lenskit.training"]
        m = knn.ItemKNNScorer(max_nbrs=20, min_sim=1e-6, save_nbrs=20)
        m.train(ref_sandbox.FakeDataset(ml_small), training.TrainingOptions())
        sim = m.sim_matrix
        assert type(sim).__name__ == "SparseRowArray" and sim.type.dimension == ml_small.n_items
        got = sim.to_scipy()
        # the stored matrix goes back into the scoring entry points' ingest unchanged
        back = accel.as_host_csr(sim, len(sim))
        assert back.shape == (ml_small.n_items, ml_small.n_items) and np.array_equal(back.indices, got.indices)
        rows = [np.arange(got.indptr[r], got.indptr[r + 1]) for r in ROWS_I]
        sel = np.concatenate(rows)
        return {"indptr": got.indptr, "indices": got.indices[sel], "data": got.data[sel].astype(np.float32),
                "means": np.asarray(m.item_means, dtype=np.float32), "counts": np.asarray(m.item_counts)}  # fmt: skip

    theirs = _theirs("item_knn_train", ref, live)
    ui, iu, means = data.knn_item_matrices(ml_small, True)
    want = oracle.knn_build(ui, iu, 1e-6, 20)
    sel = np.concatenate([np.arange(want.indptr[r], want.indptr[r + 1]) for r in ROWS_I])
    assert np.array_equal(theirs["indptr"], want.indptr)
    assert np.array_equal(theirs["indices"], want.indices[sel])
    assert np.array_equal(theirs["data"].view(np.int32), want.data[sel].view(np.int32))
    assert np.array_equal(theirs["means"].view(np.int32), means.view(np.int32))
    assert np.array_equal(theirs["counts"], np.diff(want.indptr))


def test_result_index_field_is_the_reference_extension_type(ref):
    """Wire format of the ``index`` field: extension name and JSON metadata of ``SparseIndexType``
    (data/matrix.py:104-146), whether or not lenskit is loaded; it survives an IPC round trip."""
    import pyarrow as pa

    csr = data.InteractionCSR(np.array([0, 2, 2, 3], np.int64), np.array([1, 5, 0], np.int32),
                              np.array([0.5, 0.25, 1.0], np.float32), (3, 77))  # fmt: skip
    arr = pa.chunked_array(accel.csr_to_arrow_chunks(csr, 2)).combine_chunks()

    def live():
        matrix = ref["lenskit.data.matrix"]
        t_ref = accel.sparse_index_type(77)
        assert isinstance(t_ref, matrix.SparseIndexType) and t_ref.dimension == 77  # lenskit loaded: its own class
        wrapped = matrix.SparseRowArray.from_array(arr)  # no external dimension: it must come from the type
        assert wrapped.shape == (3, 77) and wrapped.to_scipy().nnz == 3
        return {"name": np.array(t_ref.extension_name), "meta": np.frombuffer(t_ref.__arrow_ext_serialize__(), np.uint8)}

    theirs = _theirs("index_field_type", ref, live)
    t = arr.type.value_type.field("index").type
    assert t.extension_name == str(theirs["name"])
    assert t.__arrow_ext_serialize__() == theirs["meta"].tobytes()
    sink = pa.BufferOutputStream()
    tbl = pa.table({"rows": arr})
    with pa.ipc.new_stream(sink, tbl.schema) as w:
        w.write_table(tbl)
    col = pa.ipc.open_stream(sink.getvalue()).read_all().column("rows").combine_chunks()
    field = col.type.value_type.field("index")
    if isinstance(field.type, pa.ExtensionType):  # lenskit loaded: its registered class comes back
        assert field.type.extension_name == str(theirs["name"]) and field.type.dimension == 77
    else:  # unregistered: int32 storage, the extension name and metadata travel with the field
        assert field.type == pa.int32()
        assert field.metadata[b"ARROW:extension:name"] == str(theirs["name"]).encode()
        assert field.metadata[b"ARROW:extension:metadata"] == theirs["meta"].tobytes()


@pytest.mark.parametrize("feedback", ["explicit", "implicit"])
def test_reference_item_knn_scores_through_the_shim(ref, ml_small, feedback):
    """``ItemKNNScorer.__call__`` (knn/item.py:230-295) with the reference's real ``ItemList`` / ``Vocabulary``:
    nullable Int32 / Float32 Arrow arrays in (unknown history items and unknown targets are nulls), nullable
    score and count arrays out, the means added back by the reference; equal to the oracle's accumulator."""
    explicit = feedback == "explicit"
    R = ml_small.coo().tocsr()
    u = int(np.argmax(np.diff(R.indptr)))
    nums = R.indices[R.indptr[u] : R.indptr[u + 1]]
    rates = R.data[R.indptr[u] : R.indptr[u + 1]].astype(np.float32)
    tgt_nums = np.arange(0, ml_small.n_items, 7)

    def live():
        knn, training, items_mod = ref["lenskit.knn.item"], ref["lenskit.training"], ref["lenskit.data._items"]
        ItemList = items_mod.ItemList
        m = knn.ItemKNNScorer(max_nbrs=20, min_sim=1e-6, save_nbrs=20, feedback=feedback)
        m.train(ref_sandbox.FakeDataset(ml_small), training.TrainingOptions())
        accel.clear_cache()
        unknown = int(ml_small.item_ids.max()) + 1000
        hist = ItemList(item_ids=np.concatenate([ml_small.item_ids[nums], [unknown]]), rating=np.concatenate([rates, [3.0]]))
        targets = ItemList(item_ids=np.concatenate([ml_small.item_ids[tgt_nums], [unknown + 1]]))
        out = m(hist, targets)
        got = out.scores("numpy")
        assert len(got) == len(tgt_nums) + 1 and np.isnan(got[-1])  # the unknown target has no score
        return {"scores": got[:-1].astype(np.float32), "counts": np.asarray(out.field("nbr_counts", "numpy")[:-1], dtype=np.float64)}

    theirs = _theirs(f"item_knn_score_{feedback}", ref, live)
    got, counts = theirs["scores"], theirs["counts"]
    ui, iu, means = data.knn_item_matrices(ml_small, explicit)
    S = oracle.knn_build(ui, iu, 1e-6, 20)
    rv = (rates - means[nums]).astype(np.float32) if explicit else None
    want, want_ct = oracle.knn_score(S, nums.astype(np.int32), rv, tgt_nums.astype(np.int32), 20, 1)
    ok = ~np.isnan(want)
    assert ok.sum() > 100 and np.array_equal(np.isnan(got), ~ok)
    if explicit:
        want = want + means[tgt_nums]
    assert np.array_equal(want[ok].astype(np.float32).view(np.int32), got[ok].view(np.int32))
    assert np.array_equal(counts[ok], want_ct[ok].astype(np.float64))


def test_reference_implicit_mf_scores_after_training_through_the_shim(ref, ml_small):
    """The model the reference's trainer leaves behind is the one its own ``ALSBase.__call__`` scores with
    (als/_common.py:133-175): known user -> P[u] . Q^T over the requested items."""
    tgt = np.array([0, 10, 200, 4000])

    def live():
        imp, training, items_mod = ref["lenskit.als._implicit"], ref["lenskit.training"], ref["lenskit.data._items"]
        m = imp.ImplicitMFScorer(embedding_size=8, epochs=1, regularization=0.1, weight=40)
        m.train(ref_sandbox.FakeDataset(ml_small), training.TrainingOptions(rng=7))
        assert m.trained_epochs == 1 and m.user_embeddings.dtype == np.float32
        out = m(ml_small.user_ids[5], items_mod.ItemList(item_ids=ml_small.item_ids[tgt]))
        scores = out.scores("numpy")
        assert np.allclose(scores, m.item_embeddings[tgt] @ m.user_embeddings[5], rtol=1e-5, atol=1e-7)
        return {"scores": scores}

    theirs = _theirs("implicit_mf_scores", ref, live)
    ui, iu = data.als_implicit_matrices(ml_small, 40.0)
    p, q = implicit_init(np.random.default_rng(7), ml_small.n_items, ml_small.n_users, 8)
    p, _ = oracle.als_half("implicit", ui, p, q, otor_mat=_np_otor(q, 0.1))
    q, _ = oracle.als_half("implicit", iu, q, p, otor_mat=_np_otor(p, 0.1))
    assert np.allclose(theirs["scores"], q[tgt] @ p[5], rtol=10 * _tol(), atol=1e-7)


def test_reference_biased_mf_trains_through_the_shim(ref, ml_small):
    """``BiasedMFScorer`` (als/_explicit.py:94-118): the reference learns its bias model, builds the residual
    matrices and calls ``als.train_explicit_matrix(matrix, this, other, reg)`` — the scalar ``reg`` (scaled by
    the row's nnz inside, explicit.rs:104-108) instead of a Gram; then scores with its own ``__call__``."""
    R = ml_small.coo().tocsr()

    def live():
        exp, training, items_mod = ref["lenskit.als._explicit"], ref["lenskit.training"], ref["lenskit.data._items"]
        m = exp.BiasedMFScorer(embedding_size=8, epochs=2, regularization=0.1, damping=5.0)
        trainer = m.create_trainer(ref_sandbox.FakeDataset(ml_small), training.TrainingOptions(rng=3))
        p0, q0 = m.user_embeddings.copy(), m.item_embeddings.copy()
        for _ in range(2):
            trainer.train_epoch()
        ui = accel.as_host_csr(trainer.ui_rates)
        assert ui.shape == (ml_small.n_users, ml_small.n_items)
        assert np.array_equal(ui.indptr, R.indptr) and np.array_equal(ui.indices, R.indices)  # the rating structure
        out = {"resid": np.asarray(ui.values, dtype=np.float32), "reg": np.array([trainer.u_ctx.reg, trainer.i_ctx.reg]),
               "p0": p0, "q0": q0, "p": m.user_embeddings[ROWS_U], "q": m.item_embeddings[ROWS_I]}  # fmt: skip
        trainer.finalize()
        scores = m(ml_small.user_ids[3], items_mod.ItemList(item_ids=ml_small.item_ids[[1, 50, 900]])).scores("numpy")
        assert np.all(np.isfinite(scores))
        return out

    theirs = _theirs("biased_mf_train", ref, live)
    ui = data.InteractionCSR.from_scipy(sps.csr_array((theirs["resid"], R.indices, R.indptr), shape=R.shape))
    iu = data.InteractionCSR.from_scipy(sps.csr_array((theirs["resid"], R.indices, R.indptr), shape=R.shape).T)
    p, q = theirs["p0"], theirs["q0"]
    for _ in range(2):
        p, _ = oracle.als_half("explicit", ui, p, q, reg=float(theirs["reg"][0]))
        q, _ = oracle.als_half("explicit", iu, q, p, reg=float(theirs["reg"][1]))
    assert np.linalg.norm(theirs["p"] - p[ROWS_U]) <= _tol() * np.linalg.norm(p[ROWS_U])
    assert np.linalg.norm(theirs["q"] - q[ROWS_I]) <= _tol() * np.linalg.norm(q[ROWS_I])


@pytest.mark.parametrize("feedback", ["explicit", "implicit"])
def test_reference_user_knn_scores_through_the_shim(ref, ml_small, feedback):
    """``UserKNNScorer.__call__`` (knn/user.py:157-255) -> ``knn.user_score_items_explicit / _implicit``
    (user_score.rs:21-98): the neighbour list (Int32 rows, Float32 similarities) and the reference's own
    ``user_ratings`` SparseRowArray go in, a nullable Float32 array comes out, the user mean is added by the
    reference; equal to the oracle's accumulator on the same neighbour list."""
    uidx = 42
    tgt = np.arange(0, ml_small.n_items, 11)

    def live():
        usr, training, items_mod = ref["lenskit.knn.user"], ref["lenskit.training"], ref["lenskit.data._items"]
        m = usr.UserKNNScorer(max_nbrs=15, min_nbrs=2, min_sim=1e-6, feedback=feedback)
        m.train(ref_sandbox.FakeDataset(ml_small), training.TrainingOptions())
        accel.clear_cache()
        out = m(ml_small.user_ids[uidx], items_mod.ItemList(item_ids=ml_small.item_ids[tgt]))
        # the neighbour list exactly as the reference builds it (user.py:183-200)
        _uidx, ratings, umean = m._get_user_data(ref["lenskit.data._query"].RecQuery.create(ml_small.user_ids[uidx]))
        sims = m.user_vectors @ ratings
        sims[uidx] = 0
        mask = sims >= m.config.min_sim
        rat = accel.as_host_csr(m.user_ratings)  # implicit feedback: a structure-only SparseRowArray
        return {"scores": out.scores("numpy").astype(np.float32), "nbrs": np.flatnonzero(mask).astype(np.int32),
                "sims": sims[mask].astype(np.float32), "umean": np.float32(umean), "rat_values": rat.values,
                "rat_indices": rat.indices, "rat_indptr": rat.indptr}  # fmt: skip

    theirs = _theirs(f"user_knn_score_{feedback}", ref, live)
    rat = sps.csr_array((theirs["rat_values"], theirs["rat_indices"], theirs["rat_indptr"]),
                        shape=(ml_small.n_users, ml_small.n_items))  # fmt: skip
    want, _ct = oracle.user_score(rat, theirs["nbrs"], theirs["sims"], tgt.astype(np.int32), 15, 2,
                                  explicit=feedback == "explicit")  # fmt: skip
    got = theirs["scores"]
    ok = ~np.isnan(want)
    assert ok.sum() > 50 and np.array_equal(np.isnan(got), ~ok)
    assert np.array_equal((want[ok] + theirs["umean"]).astype(np.float32).view(np.int32), got[ok].view(np.int32))


def test_reference_task_runner_drives_the_task_mirror(ref):
    """The reference's own ``run_accel_task`` (parallel/_task.py:25-57) over this package's ``AccelTask``:
    result hand-back, ``invoke(pool=...)`` on its worker thread, failures re-raised as its RuntimeError with the
    task's exception as the cause, progress tuples forwarded to the progress object.  Without the checkout:
    every task attribute the runner uses exists on ``AccelTask``."""
    import inspect

    def live():
        import sys
        import threading
        import time

        run = sys.modules["lenskit.parallel"].run_accel_task
        assert run.__module__ == "lenskit.parallel._task"
        seen = {}

        def body(task):
            seen["thread"] = threading.current_thread().name
            time.sleep(0.5)  # long enough for two polls of current_progress()
            return 42.0

        prog = ref_sandbox._Progress()
        assert run(accel.AccelTask(body, total=10), progress=prog) == 42.0
        assert seen["thread"].startswith("AccelTask-") and prog.updates >= 1

        def boom(_task):
            raise RuntimeError("ALS solve error: array minor of row 3 is not positive")

        with pytest.raises(RuntimeError, match="accelerator task failed") as ei:
            run(accel.AccelTask(boom, total=1))
        assert "ALS solve error" in str(ei.value.__cause__)
        t = accel.AccelTask(body, total=1)
        t.cancel()
        with pytest.raises(RuntimeError, match="accelerator task failed") as ei:
            run(t)
        assert "cancelled" in str(ei.value.__cause__)
        tree = ast.parse(inspect.getsource(run).lstrip())
        arg = tree.body[0].args.args[0].arg  # the task parameter
        used = {n.attr for n in ast.walk(tree) if isinstance(n, ast.Attribute) and isinstance(n.value, ast.Name) and n.value.id == arg}
        return {"task_attrs": np.array(sorted(used))}

    theirs = _theirs("task_runner", ref, live)
    task = accel.AccelTask(lambda _t: 1.0, total=1)
    assert len(theirs["task_attrs"]) >= 2
    for name in theirs["task_attrs"]:
        assert hasattr(task, str(name)), f"run_accel_task uses task.{name}, which AccelTask lacks"


def test_reference_item_list_top_n_through_the_argtopn_mirror(ref):
    """``ItemList.top_n`` (data/_items.py:942-998) -> ``_accel.data.argtopn(scores: pa.Array, n)``: Arrow nulls
    and NaNs are both unscored (sorting.rs:163-167), an Int32Array of positions comes back, best first."""
    import pyarrow as pa

    rng = np.random.default_rng(8)
    scores = rng.standard_normal(200).astype(np.float32)
    scores[::9] = np.nan

    def live():
        ItemList = ref["lenskit.data._items"].ItemList
        top = ItemList(item_ids=np.arange(1000, 1200), scores=scores).top_n(10)
        assert top.ordered
        return {"top_ids": np.asarray(top.ids())}

    theirs = _theirs("item_list_top_n", ref, live)
    got = accel.argtopn(pa.array(scores), 10)
    assert (1000 + got.to_numpy()).tolist() == theirs["top_ids"].tolist()
    # nullable Arrow scores, as the kNN entry points return them
    masked = np.zeros(200, dtype=bool)
    masked[::4] = True
    got = accel.argtopn(pa.array(scores, mask=masked), 25)
    assert isinstance(got, pa.Array) and got.type == pa.int32()
    assert got.to_numpy().tolist() == oracle.argtopn(np.where(masked, np.nan, scores).astype(np.float32), 25).tolist()


def test_integration_md_trainer_binding_matches_both_sides(ref):
    """The trainer-level binding printed in INTEGRATION.md §2: every ``engine.*`` / ``_lib.*`` name it uses exists
    in this package, and every ``context.*`` field it reads exists on the reference's ``TrainContext``.  With the
    checkout the code block is also compiled and its classes created on top of the reference's real
    ``ImplicitMFTrainer`` / ``ImplicitMFScorer``."""
    import re

    from lkpy_b200 import _lib, engine

    text = (Path(__file__).resolve().parent.parent / "INTEGRATION.md").read_text()
    blocks = re.findall(r"```python\n(.*?)```", text, flags=re.S)
    block = next(b for b in blocks if "class B200ImplicitMFTrainer" in b)
    tree = ast.parse(block)

    def live():
        ns: dict = {}
        exec(compile(tree, "INTEGRATION.md#trainer-binding", "exec"), ns)  # imports lenskit.als._implicit: the sandbox's
        imp = ref["lenskit.als._implicit"]
        assert issubclass(ns["B200ImplicitMFTrainer"], imp.ImplicitMFTrainer)
        assert issubclass(ns["B200ImplicitMFScorer"], imp.ImplicitMFScorer)
        assert not getattr(ns["B200ImplicitMFTrainer"], "__abstractmethods__", None)  # the hook is the only abstract piece it fills
        return {"context_fields": np.array(sorted(ref["lenskit.als._common"].TrainContext._fields))}

    theirs = _theirs("train_context", ref, live)
    used = {(n.value.id, n.attr) for n in ast.walk(tree) if isinstance(n, ast.Attribute) and isinstance(n.value, ast.Name)}
    for mod_name, mod in (("engine", engine), ("_lib", _lib)):
        for _m, attr in sorted(u for u in used if u[0] == mod_name):
            assert hasattr(mod, attr), f"INTEGRATION.md uses {mod_name}.{attr}, which does not exist"
    fields = {str(f) for f in theirs["context_fields"]}
    for _m, attr in sorted(u for u in used if u[0] in ("context", "ctx")):
        assert attr in fields, f"INTEGRATION.md reads context.{attr}; TrainContext has {sorted(fields)}"
