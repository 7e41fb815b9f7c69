"""
The roofline arithmetic of bench.py against the figures of SURVEY.md §8d (algorithmic bytes per
half-epoch / per build at ML-25M shape), and the host-side helpers that do not need a GPU.
"""

import importlib.util

import numpy as np
import pytest
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def _bench():
    spec = importlib.util.spec_from_file_location("lk_bench", ROOT / "bench.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["lk_bench"] = mod
    spec.loader.exec_module(mod)
    return mod


def test_als_algorithmic_bytes_match_survey():
    b = _bench()
    U, I, N, k = 162_541, 59_047, 25_000_095, 64
    # SURVEY.md §8d: N(k s + 8) + 4(R+1) + R k 4 2 + k^2 4 per half-epoch (OtOr pass counted separately)
    fp32 = b.als_half_bytes(U, I, N, k, 4, False) + b.als_half_bytes(I, U, N, k, 4, False)
    bf16 = b.als_half_bytes(U, I, N, k, 2, False) + b.als_half_bytes(I, U, N, k, 2, False)
    assert abs(fp32 / 1e9 - 13.3) < 0.1  # "≈ 13.4 GB/epoch" with the OtOr pass
    assert abs(bf16 / 1e9 - 6.9) < 0.1  # "bf16 gather ≈ 7.0 GB"
    with_otor = b.als_half_bytes(U, I, N, k, 4, True) + b.als_half_bytes(I, U, N, k, 4, True)
    assert abs(with_otor / 1e9 - 13.4) < 0.1
    # 4.0 ms / 2.1 ms at the H100 SXM data sheet's 3.35 TB/s (DESIGN.md §4)
    assert abs(fp32 / 3.35e12 * 1e3 - 3.98) < 0.1 and abs(bf16 / 3.35e12 * 1e3 - 2.06) < 0.1


def test_knn_algorithmic_bytes_match_survey():
    b = _bench()
    # P = 1.278e10 products => 102 GB streamed, 30.5 ms at the data sheet's 3.35 TB/s (SURVEY.md §8d)
    by = b.knn_build_bytes(12_764_118_364, 25_000_095, 162_541, 59_047, 1_180_940)
    assert abs(by / 1e9 - 102.3) < 0.5
    assert abs(by / 3.35e12 * 1e3 - 30.5) < 0.4


def test_host_threads_ignores_omp_env(monkeypatch):
    b = _bench()
    monkeypatch.setenv("OMP_NUM_THREADS", "1")  # what torchrun exports to every rank
    import os

    assert b.host_threads() == len(os.sched_getaffinity(0)) >= 1


def test_committed_bench_lines_have_the_contract_keys():
    """The bench lines kept under tests/golden/ (one H100, and the CPU reference arm) carry every key the
    benchmark's output contract names."""
    need = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks"}  # fmt: skip
    gold = ROOT / "tests" / "golden"
    for name in ("bench_h100_n1.json",):
        line = json.loads((gold / name).read_text().strip().splitlines()[-1])
        assert need <= set(line), (name, need - set(line))
        assert line["vs_baseline"] is None and line["higher_is_better"] is False
        assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(line["roofline"])
        assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(line["e2e"])
        assert "workload" in line["config"]
    ref = json.loads((gold / "bench_reference_arm.json").read_text().strip().splitlines()[-1])
    assert ref["impl"] == "reference" and ref["e2e"]["h2d_bytes_per_step"] == 0
    assert {"kind", "cores", "sample", "value"} <= set(ref["cpu_baseline"])


def test_solve_cholesky_property():
    """The reference's property test of `solve_cholesky` (tests/utils/test_math_solve.py:21-50) against the
    host fold-in solver that mirrors it (`lkpy_b200.als._solve_cholesky`)."""
    import numpy as np
    from pytest import approx

    from lkpy_b200.als import _solve_cholesky

    for seed in range(40):
        rng = np.random.RandomState(seed)
        size = int(rng.randint(2, 101))
        A = rng.randn(size, size) * 10
        b = rng.randn(size) * 10
        A = A * A
        xexp = np.linalg.lstsq(A, b, rcond=None)[0]
        F, y = A.T @ A, A.T @ b
        x = _solve_cholesky(F, y)
        assert x.shape == y.shape
        assert x == approx(xexp, rel=1.0e-3)
        assert F @ x == approx(y, rel=2.0e-6, abs=5.0e-9)


def test_biased_mf_fold_in_zeroes_an_infinite_user_bias():
    """BiasedMF's fold-in counts a user bias that is not finite as 0: NaN, as the reference's ``compute_for_items``
    does, and also an infinite one, which ``BiasModel.user_bias_for_items`` (the reference's rule) keeps."""
    from lkpy_b200.als import BiasedMFScorer, _solve_cholesky
    from lkpy_b200.basic import BiasModel
    from lkpy_b200.components import ItemList, Vocabulary

    rng = np.random.default_rng(7)
    m = BiasedMFScorer(embedding_size=8)
    m.items = Vocabulary(np.arange(20), "item")
    m.item_embeddings = rng.standard_normal((20, 8)).astype(np.float32)
    m.bias = BiasModel(3.5, (rng.standard_normal(20) * 0.1).astype(np.float32), np.zeros(4, np.float32), (5.0, 5.0))
    items = np.array([2, 7, 11])
    for ratings, rule in (([np.inf, 4.0, 3.0], np.inf), ([-np.inf, 4.0, 3.0], -np.inf), ([np.inf, -np.inf, 3.0], 0.0)):
        for dtype in (np.float32, np.float64):
            q = ItemList(item_ids=items, rating=np.array(ratings, dtype=dtype))
            assert m.bias.user_bias_for_items(items, q.field("rating")) == rule
            emb, u_bias = m.new_user_embedding(None, q)
            assert u_bias == 0.0
            rated = items[np.isfinite(ratings)]
            M = m.item_embeddings[rated]
            rv = (np.asarray(ratings)[np.isfinite(ratings)] - 3.5 - m.bias.item_biases[rated]).astype(np.float32)
            want = _solve_cholesky(M.T @ M + np.eye(8, dtype=np.float32) * 0.1 * len(rated), M.T @ rv)
            assert np.allclose(emb, want, rtol=1e-5, atol=1e-6)
            assert np.isfinite(m(q, ItemList(item_ids=[1, 2, 3])).scores()).all()


def test_accel_mirror_signatures_match_reference_stubs():
    """Every function the reference's typed stubs declare for the two hot paths (`_accel/als.pyi`,
    `_accel/knn.pyi`, recorded in tests/golden/accel_stub_signatures.json) exists in lkpy_b200.accel with
    the same parameter names in the same order — the call sites (als/_implicit.py:161-164,
    als/_explicit.py:115-118, knn/item.py:162-171, :273-287, knn/user.py:224-240) bind positionally."""
    import inspect
    import json

    from lkpy_b200 import accel

    stubs = json.loads((Path(__file__).parent / "golden" / "accel_stub_signatures.json").read_text())
    for mod, ns in (("als", accel.als), ("knn", accel.knn)):
        assert stubs[mod]
        for name, want in stubs[mod].items():
            ours = getattr(ns, name, None)
            assert ours is not None, f"_accel.{mod}.{name} missing from the mirror"
            got = list(inspect.signature(ours).parameters)
            assert got == want, (name, got, want)
    # user-kNN scoring lives in the Rust module without a stub entry: same argument order as user_score.rs:21-29
    got = list(inspect.signature(accel.knn.user_score_items_explicit).parameters)
    assert got == ["tgt_items", "nbr_rows", "nbr_sims", "ratings", "max_nbrs", "min_nbrs"]


def test_accel_task_protocol_without_device():
    """invoke-once, cancel-before-invoke and progress shape of the task mirror (tasks/mod.rs:62-106) — host only."""
    from lkpy_b200.accel import AccelTask, run_accel_task

    t = AccelTask(lambda task: 7, total=10)
    assert t.current_progress() == (0, 10)
    assert run_accel_task(t) == 7
    assert t.current_progress() == (10, 10)
    with pytest.raises(RuntimeError, match="already invoked"):
        t.invoke()
    t2 = AccelTask(lambda task: 1, total=None)
    assert t2.current_progress() is None
    t2.cancel()
    with pytest.raises(RuntimeError, match="cancelled"):
        t2.invoke()
    with pytest.raises(RuntimeError, match="accelerator task failed"):
        run_accel_task(AccelTask(lambda task: 1 / 0))


def test_arrow_csr_ingest_and_chunks():
    """Arrow List / LargeList<Struct{index,value}> -> host CSR views -> LargeList chunks (csr.rs:160-209,
    consumer.rs:96-142) round-trip without a device."""
    import pyarrow as pa

    from lkpy_b200 import accel
    from lkpy_b200.data import InteractionCSR

    rng = np.random.default_rng(1)
    lens = rng.integers(0, 7, 50)
    indptr = np.concatenate([[0], np.cumsum(lens)])
    cols = np.concatenate([np.sort(rng.choice(40, n, replace=False)) for n in lens]).astype(np.int32)
    vals = rng.standard_normal(len(cols)).astype(np.float32)
    csr = InteractionCSR(indptr.astype(np.int64), cols, vals, (50, 40))
    chunks = accel.csr_to_arrow_chunks(csr, 16)
    assert len(chunks) == 4 and all(pa.types.is_large_list(c.type) for c in chunks)
    back = accel.as_host_csr(pa.chunked_array(chunks), 40)
    assert np.array_equal(back.indptr, csr.indptr) and np.array_equal(back.indices, cols)
    assert np.array_equal(back.values.view(np.int32), vals.view(np.int32)) and back.shape == (50, 40)
    # a sliced List array (non-zero first offset) and a structure-only array
    small = pa.ListArray.from_arrays(
        pa.array(indptr.astype(np.int32)),
        pa.StructArray.from_arrays([pa.array(cols), pa.array(vals)], names=["index", "value"]),
    ).slice(10, 20)
    sl = accel.as_host_csr(small, 40)
    assert sl.shape == (20, 40) and sl.indptr[0] == 0 and sl.nnz == int(indptr[30] - indptr[10])
    assert np.array_equal(sl.indices, cols[indptr[10] : indptr[30]])
    only = accel.as_host_csr(pa.ListArray.from_arrays(pa.array(indptr.astype(np.int32)), pa.array(cols)), 40)
    assert np.all(only.values == 1.0) and np.array_equal(only.indices, cols)


def test_row_part_length_by_kernel_path():
    """ALSTrainerBase._chunk_nnz: which row-part length each kernel path is planned with (engine.TF32_CHUNK_NNZ*:
    the tf32 paths and k = 128 get shorter parts)."""
    from types import SimpleNamespace

    from lkpy_b200 import _lib, engine
    from lkpy_b200.als import ALSTrainerBase

    def chunk(k, gather, mode=_lib.LK_ALS_IMPLICIT, use_ratings=False):
        me = SimpleNamespace(MODE=mode, config=SimpleNamespace(gather_dtype=gather, use_ratings=use_ratings))
        return ALSTrainerBase._chunk_nnz(me, k)

    assert chunk(64, "bfloat16") == engine.DEFAULT_CHUNK_NNZ  # als_tc_kernel: one accumulation per 16 rows
    assert chunk(64, "float32") == engine.TF32_CHUNK_NNZ  # als_tc_kernel, tf32 x3
    assert chunk(64, "bfloat16", use_ratings=True) == engine.TF32_CHUNK_NNZ  # weighted: tf32 path as well
    assert chunk(64, "float32", mode=_lib.LK_ALS_EXPLICIT) == engine.TF32_CHUNK_NNZ
    assert chunk(128, "bfloat16") == engine.TF32_CHUNK_NNZ  # als_tc_kernel, bf16 MMA
    assert chunk(128, "float32") == engine.TF32_CHUNK_NNZ_K128  # als_tc_kernel, tf32 x3
    assert chunk(128, "bfloat16", use_ratings=True) == engine.TF32_CHUNK_NNZ_K128
    assert chunk(32, "float32") == engine.DEFAULT_CHUNK_NNZ  # SIMT kernel
    assert engine.TF32_CHUNK_NNZ_K128 < engine.TF32_CHUNK_NNZ < engine.DEFAULT_CHUNK_NNZ


def test_synthetic_matrix_cache_round_trip(tmp_path):
    """data.synth_interactions_cached: the cached arrays are the generator's own, and a cache of another shape is
    not reused."""
    from lkpy_b200 import data

    shape = dict(n_users=400, n_items=150, nnz=6000)
    f = str(tmp_path / "cache.npz")
    a = data.synth_interactions_cached(f, **shape)
    b = data.synth_interactions_cached(f, **shape)  # from the file
    c = data.synth_interactions(**shape)
    for x in (a, b):
        assert (x.n_users, x.n_items) == (c.n_users, c.n_items)
        assert np.array_equal(x.users, c.users) and np.array_equal(x.items, c.items)
        assert np.array_equal(x.ratings.view(np.int32), c.ratings.view(np.int32))
    other = data.synth_interactions_cached(f, n_users=300, n_items=150, nnz=5000)
    assert other.n_users == 300 and other.nnz == 5000
    assert data.synth_interactions_cached(None, **shape).nnz == c.nnz


def test_own_index_type_matches_the_reference_wire_format():
    """Without lenskit in the process the index field of a result carries this package's own class of the
    ``lenskit.sparse_index`` extension type: same name, same JSON metadata (data/matrix.py:104-146), unregistered."""
    import json
    import sys

    import pyarrow as pa

    from lkpy_b200 import accel

    if "lenskit.data.matrix" in sys.modules:
        pytest.skip("lenskit is loaded: its own class is used")
    t = accel.sparse_index_type(9066)
    assert t.extension_name == "lenskit.sparse_index" and t.storage_type == pa.int32() and t.dimension == 9066
    assert json.loads(t.__arrow_ext_serialize__().decode()) == {"dimension": 9066}
    assert type(t).__arrow_ext_deserialize__(pa.int32(), t.__arrow_ext_serialize__()).dimension == 9066
