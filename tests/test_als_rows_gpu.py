"""
The ALS row solve (lk_als_half_epoch) on every kernel route.  The routes are the entries of ROUTES below, and
every test here takes its routes from that table.

Row by row, at the row lengths where the kernels change behaviour.  A matrix-level check compares a whole
half-step with one relative Frobenius error: one row in a thousand off by 1e-3 moves that number by ~3e-5 and
passes.  So test_route_rows and the boundary, failing-row and replica tests hold every row r with nonzeros to

    e(r) = |x_gpu - x64| / |x64|  <=  max(A, B * f(r)),      f(r) = |x32 - x64| / |x64|

where x64 is the f64 oracle and x32 the f32 oracle on the same inputs (gathered rows rounded to bf16 when the
route gathers bf16, the same f32 OtOr the device is given).  A and B are per kernel family (TOL below).  The
sum of squared row changes must match the f64 oracle's, empty rows must come out exactly 0, and a rerun must
give the same bits.

The rows are built by hand: lengths 1 .. 129 around the SIMT kernel's 32-row stages and the MMA paths' 16 / 8-row
steps, lengths around 1, 2 and 3 part lengths, a row of over 40 parts, and empty rows.  The plan is checked
to really contain each of them.  A larger variant adds ~16k short rows so that every CTA of the persistent grid
works through many chunks in sequence (mbarrier phases, pad-column re-zeroing, claim-ahead).

Whole matrices, on the tensor-core kernel (als_tc.cu) with small synthetic data, and with OtOr and the bf16
copy of `other` built on the device by lk_als_otor as the trainers build them: the relative Frobenius error
against the f64 oracle, agreement with the SIMT kernel on the same inputs, split rows (bit-identical reruns,
close to the one-part solve), badly conditioned systems, and the LK_ALS_TF32 switch.

Failures: a system that is not positive definite, or that meets an exact zero pivot on any one-warp solver,
must be reported in the status word and leave its row untouched.
"""

from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import pytest
import torch

import oracle
from lkpy_b200 import _lib, data, engine
from lkpy_b200.als import ALSTrainerBase

from helpers import implicit_init, rel_fro, small_synth

pytestmark = pytest.mark.gpu

N_OTHER = 3000
REG = 0.1
UNIFORM_CONF = 40.0
DEFAULT_CHUNK = engine.DEFAULT_CHUNK_NNZ
BASE_LENGTHS = (1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129)
COPIES = 3
N_EMPTY = 4
MANY_PARTS = 40
#: short rows of the large boundary matrix: ~10x the persistent grid at k <= 64 (132 SMs x 12 CTAs)
N_SHORT = 16000

# Per-row bounds by kernel family: e(r) <= max(A, B * f(r)) with A = max(A0, A1 * part length), entries
# (A0, A1, B).  Set from the worst rows of every route and boundary case below over three seeds on an H100 80GB
# HBM3 (700 W power limit), with a margin of 2-3x over the A each needed at B = 4:
#   simt     worst e 9.9e-6, A needed 5.3e-6 (bf16 rows, k = 8; e / f <= 5.1 elsewhere)
#   simt-k1  k = 1: x = y / a, and y's cancellation makes f(r) small by chance; A needed 3.3e-5
#   bf16mma  A needed 1.3e-5 (parts of 4096; 4.2e-6 at parts <= 1024)
#   tf32     grows with the rows one part sums on the tensor cores: worst e 4.8e-6 / 7.4e-6 / 2.35e-5 /
#            8.2e-5 at parts of 32 / 256 / 1024 / 4096, i.e. ~2e-8 per row of the part
TOL = {
    "simt": (1.5e-5, 0.0, 4.0),
    "simt-k1": (1e-4, 0.0, 4.0),
    "bf16mma": (4e-5, 0.0, 4.0),
    "tf32": (1.5e-5, 6e-8, 4.0),
}


def chunk_lengths(c: int) -> tuple[int, ...]:
    return (c - 1, c, c + 1, 2 * c, 2 * c + 1, 3 * c - 1)


def many_parts_length(c: int) -> int:
    return MANY_PARTS * c + 7


# ---------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------


def boundary_lengths(c: int, *, n_short: int, many_parts: bool, rng) -> np.ndarray:
    lens = list(BASE_LENGTHS) * COPIES + list(chunk_lengths(c)) * COPIES + [0] * N_EMPTY
    if many_parts:
        lens.append(many_parts_length(c))
    lens += rng.choice(BASE_LENGTHS, n_short).tolist()
    return rng.permutation(np.array(lens, dtype=np.int64))


def boundary_csr(c: int, kind: str, *, n_short: int = 0, many_parts: bool = True, seed: int = 0,
                 n_other: int = N_OTHER) -> data.InteractionCSR:  # fmt: skip
    """CSR with the boundary lengths for part length c.  Columns are distinct within a row where the row fits in
    `other`, and the first and last rows of `other` are always gathered.  kind: "uniform" (one implicit
    confidence), "weighted" (per-nonzero confidences), "negative" (weighted, one confidence below zero) or
    "explicit" (centred ratings)."""
    rng = np.random.default_rng([seed, c, n_short])
    lens = boundary_lengths(c, n_short=n_short, many_parts=many_parts, rng=rng)
    cols = []
    for n in lens:
        if n <= n_other:
            cols.append(np.sort(rng.choice(n_other, n, replace=False)))
        else:  # the many-part row: every row of `other`, then repeats
            cols.append(np.sort(np.concatenate([np.arange(n_other), rng.integers(0, n_other, n - n_other)])))
    long_rows = np.flatnonzero(lens >= 2)
    for r in long_rows[:3]:  # sorted and distinct stays true: 0 and n_other - 1 replace the extremes
        cols[r][0], cols[r][-1] = 0, n_other - 1
    indices = np.concatenate(cols).astype(np.int32)
    nnz = len(indices)
    if kind == "uniform":
        vals = np.full(nnz, UNIFORM_CONF, dtype=np.float32)
    elif kind in ("weighted", "negative"):
        vals = rng.uniform(0.5, 40.0, nnz).astype(np.float32)
        if kind == "negative":
            vals[rng.integers(nnz)] = -0.5
    else:
        vals = rng.standard_normal(nnz).astype(np.float32)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    csr = data.InteractionCSR(indptr, indices, vals, (len(lens), n_other))
    assert 0 in indices and n_other - 1 in indices
    return csr


def factors(n_rows: int, n_other: int, k: int, seed: int) -> tuple[np.ndarray, np.ndarray]:
    rng = np.random.default_rng([seed, k, 77])
    this = (rng.standard_normal((n_rows, k)) * 0.1).astype(np.float32)
    other = (rng.standard_normal((n_other, k)) * 0.1).astype(np.float32)
    return this, other


def trainer_chunk(k: int, bf16: bool, kind: str) -> int:
    """The part length ALSTrainerBase plans this configuration with."""
    mode = _lib.LK_ALS_EXPLICIT if kind == "explicit" else _lib.LK_ALS_IMPLICIT
    cfg = SimpleNamespace(gather_dtype="bfloat16" if bf16 else "float32", use_ratings=kind in ("weighted", "negative"))
    return ALSTrainerBase._chunk_nnz(SimpleNamespace(MODE=mode, config=cfg), k)


def synth_matrices(inter, kind: str, rng) -> tuple[data.InteractionCSR, data.InteractionCSR]:
    """(ui, iu) of `small_synth` interactions.  kind: "uniform" (one implicit confidence), "weighted"
    (confidences scaled by the ratings) or "explicit" (ratings drawn from rng)."""
    if kind == "explicit":
        coo = inter.coo(rng.standard_normal(inter.nnz).astype(np.float32))
        return data.InteractionCSR.from_scipy(coo), data.InteractionCSR.from_scipy(coo.T)
    return data.als_implicit_matrices(inter, UNIFORM_CONF, use_ratings=kind == "weighted")


def synth_factors(rng, n_users: int, n_items: int, k: int) -> tuple[np.ndarray, np.ndarray]:
    """User factors, then item factors, N(0, 0.1^2)."""
    p = (rng.standard_normal((n_users, k)) * 0.1).astype(np.float32)
    q = (rng.standard_normal((n_items, k)) * 0.1).astype(np.float32)
    return p, q


# ---------------------------------------------------------------------------
# device run, oracles, checker
# ---------------------------------------------------------------------------


def run_device(kind, csr, this, other, *, k, bf16, chunk=DEFAULT_CHUNK, otor32=None, device_otor=False, reg=REG,
               misaligned=False, replicas=None, replica_row0=0):  # fmt: skip
    """One half-step through lk_als_half_epoch; returns (x, sqrt(sqdelta), status, plan).  OtOr is otor32, or
    with device_otor it and the bf16 copy of `other` are built on the device by lk_als_otor, as the trainers
    build them."""
    dev = _lib.require_device()
    plan = engine.ALSHalfPlan.create(engine.DeviceCSR.from_host(csr, dev), k, chunk)
    d_this = torch.from_numpy(this.copy()).to(dev)
    src = torch.from_numpy(other).to(dev)
    implicit = kind != "explicit"
    if device_otor:
        ws = engine.OtorWorkspace.create(k, dev)
        obf = torch.empty_like(src, dtype=torch.bfloat16) if bf16 else None
        otor = engine.als_otor(src, reg, ws, obf)
        src = obf if bf16 else src
    else:
        otor = torch.from_numpy(otor32).to(dev) if implicit else None
        if bf16:
            src = src.to(torch.bfloat16)
    if misaligned:  # a contiguous view whose storage starts one element past a 16-byte boundary
        buf = torch.empty(src.numel() + 1, dtype=src.dtype, device=dev)
        buf[1:] = src.reshape(-1)
        src = buf[1:].view(other.shape)
        assert src.is_contiguous() and src.data_ptr() % 16 != 0
    engine.als_half_epoch(
        plan, _lib.LK_ALS_IMPLICIT if implicit else _lib.LK_ALS_EXPLICIT, d_this, src,
        otor=otor if implicit else None, reg=reg, replicas=replicas, replica_row0=replica_row0,
    )  # fmt: skip
    torch.cuda.synchronize()
    return d_this.cpu().numpy(), float(np.sqrt(plan.sqdelta.item())), int(plan.status.item()), plan


def oracle64(kind, csr, this, other, *, bf16, reg=REG):
    """(x64, delta64, otor32): the f64 oracle on the inputs the device sees, and the f32 OtOr (None in explicit
    mode)."""
    mode = "explicit" if kind == "explicit" else "implicit"
    o32 = o64 = None
    if mode == "implicit":
        o32, o64 = oracle.otor(oracle.bf16_round(other) if bf16 else other, reg)
    x64, d64 = oracle.als_half_f64(mode, csr, this, other, otor_mat=o64, reg=reg, bf16_other=bf16)
    return x64, d64, o32


def oracles(kind, csr, this, other, *, bf16, reg=REG):
    """(x64, delta64, x32, otor32): the f64 and f32 oracles on the inputs the device sees."""
    x64, d64, o32 = oracle64(kind, csr, this, other, bf16=bf16, reg=reg)
    mode = "explicit" if kind == "explicit" else "implicit"
    x32, _ = oracle.als_half(mode, csr, this, other, otor_mat=o32, reg=reg, bf16_other=bf16)
    return x64, d64, x32, o32


def row_parts(csr, chunk: int) -> np.ndarray:
    n = np.diff(csr.indptr).astype(np.int64)
    return np.where(n > chunk, -(-n // chunk), 1)


def row_errors(got, x64, x32, rows):
    den = np.linalg.norm(x64[rows], axis=1)
    e = np.linalg.norm(got[rows].astype(np.float64) - x64[rows], axis=1) / den
    f = np.linalg.norm(x32[rows].astype(np.float64) - x64[rows], axis=1) / den
    return e, f


def row_failures(got, x64, x32, csr, chunk, tol, rows=None) -> tuple[list[str], dict]:
    """Rows (with nonzeros, or the given subset) outside max(A, B f(r)); a description of the worst ones and the
    worst e(r), e(r) / f(r) seen."""
    a0, a1, b_tol = tol
    n = np.diff(csr.indptr)
    if rows is None:
        rows = np.flatnonzero(n > 0)
    e, f = row_errors(got, x64, x32, rows)
    bound = np.maximum(np.maximum(a0, a1 * np.minimum(n[rows], chunk)), b_tol * f)
    ratio = e / np.maximum(f, 1e-30)
    bad = ~(e <= bound)  # NaN fails
    parts = row_parts(csr, chunk)
    worst = np.argsort(-np.where(bad, np.inf, e / bound), kind="stable")[: min(5, len(rows))]
    msgs = [
        f"row {rows[i]}: len {n[rows[i]]}, parts {parts[rows[i]]}, e {e[i]:.3g}, f {f[i]:.3g}, bound {bound[i]:.3g}"
        for i in worst
        if bad[i]
    ]
    stats = {"max_e": float(np.nanmax(e)), "max_ratio": float(np.nanmax(ratio)), "rows": int(len(rows)),
             "n_bad": int(bad.sum()), "worst": msgs}  # fmt: skip
    return msgs, stats


def check_rows(got, x64, x32, csr, chunk, tol, label="", rows=None) -> dict:
    msgs, stats = row_failures(got, x64, x32, csr, chunk, tol, rows)
    assert not msgs, f"{label}: {stats['n_bad']} of {stats['rows']} rows out of tolerance; worst:\n" + "\n".join(msgs)
    return stats


def plan_rows(plan, csr) -> dict[int, tuple[int, list[int]]]:
    """row -> (n_parts, part lengths) from the plan the device ran."""
    ch = plan.chunks.cpu().numpy()[: plan.n_chunks]
    out: dict[int, tuple[int, list[int]]] = {}
    for row, _begin, ln, parts, _s, part, _sp, _z in ch:
        nparts, lens = out.setdefault(int(row), (int(parts), [0] * int(parts)))
        assert nparts == parts
        lens[int(part)] = int(ln)
    return out


def check_plan(plan, csr, chunk: int, *, many_parts: bool) -> dict:
    """The plan holds every intended length with the intended split, every part 1 .. chunk long; returns the
    histogram {length: (rows, parts)} of the boundary lengths."""
    n = np.diff(csr.indptr)
    pr = plan_rows(plan, csr)
    assert set(pr) == set(range(len(n)))
    hist = {}
    want = set(BASE_LENGTHS) | set(chunk_lengths(chunk)) | {0}
    if many_parts:
        want.add(many_parts_length(chunk))
    for r, (nparts, lens) in pr.items():
        assert sum(lens) == n[r]
        assert nparts == max(1, -(-int(n[r]) // chunk))
        if nparts > 1:
            assert min(lens) >= 1 and max(lens) <= chunk, (r, lens)
        if n[r] in want:
            cnt, _ = hist.get(int(n[r]), (0, nparts))
            hist[int(n[r])] = (cnt + 1, nparts)
    for length in want:
        copies = N_EMPTY if length == 0 else 1 if length == many_parts_length(chunk) else COPIES
        assert hist.get(length, (0, 0))[0] >= copies, (length, hist)
    if many_parts:
        assert hist[many_parts_length(chunk)][1] >= MANY_PARTS
    assert plan.n_split_rows == int(np.sum(n > chunk))
    return hist


_ORACLE_CACHE: dict = {}


def case(route, kind, chunk, *, seed=0, n_short=0, many_parts=None, check=True) -> dict:
    """Run one route on the boundary matrix for `chunk` and hold every row to the route's bound.  The oracles
    are shared between routes that see the same inputs."""
    k, bf16, family = route["k"], route["bf16"], route["family"]
    if many_parts is None:
        # the 40-part row at chunk 1024 / 4096 (41k / 164k nonzeros) only in the large matrix: its oracle solve is serial
        many_parts = many_parts_length(chunk) <= 12_000
    key = (k, bf16, kind, chunk, seed, n_short, many_parts)
    if key not in _ORACLE_CACHE:
        csr = boundary_csr(chunk, kind, n_short=n_short, many_parts=many_parts, seed=seed)
        this, other = factors(csr.shape[0], N_OTHER, k, seed)
        while len(_ORACLE_CACHE) >= 8 or (n_short and _ORACLE_CACHE):
            _ORACLE_CACHE.pop(next(iter(_ORACLE_CACHE)))
        _ORACLE_CACHE[key] = (csr, this, other, oracles(kind, csr, this, other, bf16=bf16))
    csr, this, other, (x64, d64, x32, o32) = _ORACLE_CACHE[key]
    misaligned = route.get("misaligned", False)
    got, delta, status, plan = run_device(kind, csr, this, other, k=k, bf16=bf16, chunk=chunk, otor32=o32,
                                          misaligned=misaligned)  # fmt: skip
    again, _, _, _ = run_device(kind, csr, this, other, k=k, bf16=bf16, chunk=chunk, otor32=o32, misaligned=misaligned)
    assert status == 0
    assert plan.vals_uniform == (kind == "uniform")
    hist = check_plan(plan, csr, chunk, many_parts=many_parts)
    label = f"{route['id']} k={k} {kind} chunk={chunk} seed={seed}"
    stats = {"label": label, "family": family, "hist": hist}
    if check:
        stats.update(check_rows(got, x64, x32, csr, chunk, TOL[family], label))
        assert np.array_equal(got.view(np.int32), again.view(np.int32)), f"{label}: rerun differs"
        assert np.all(got[np.diff(csr.indptr) == 0] == 0.0)
        assert delta == pytest.approx(d64, rel=1e-3)
    else:
        stats.update(row_failures(got, x64, x32, csr, chunk, TOL[family])[1])
        stats["rerun_equal"] = bool(np.array_equal(got.view(np.int32), again.view(np.int32)))
        stats["delta_rel"] = abs(delta - d64) / d64
    stats.update(got=got, x64=x64, x32=x32, csr=csr, this=this, other=other, o32=o32)
    return stats


# ---------------------------------------------------------------------------
# routes
# ---------------------------------------------------------------------------

ALL = ("uniform", "weighted", "explicit")
SIMT_ONLY = {"LK_ALS_TC": 0}


def _r(id_, k, bf16, family, kinds=ALL, **kw):
    return dict(id=id_, k=k, bf16=bf16, family=family, kinds=kinds, **kw)


ROUTES = [
    # SIMT kernel (als_kernels.cu), KP = 32 / 64 / 128, bulk copy (k * sizeof(row element) % 16 == 0) or element copy
    *[_r("simt32-f32-bulk", k, False, "simt") for k in (8, 32)],
    _r("simt32-f32-elem", 1, False, "simt-k1"),
    _r("simt32-f32-elem", 31, False, "simt"),
    *[_r("simt32-bf16-bulk", k, True, "simt") for k in (8, 32)],
    _r("simt32-bf16-elem", 20, True, "simt"),
    _r("simt64-f32-bulk", 48, False, "simt"),
    _r("simt64-f32-bulk", 64, False, "simt", opts={"LK_ALS_TF32": 0}),
    *[_r("simt64-f32-elem", k, False, "simt") for k in (33, 50)],
    _r("simt64-bf16-bulk", 48, True, "simt"),
    _r("simt64-bf16-bulk", 64, True, "simt", opts=SIMT_ONLY),
    _r("simt64-bf16-elem", 50, True, "simt"),
    *[_r("simt128-f32-bulk", k, False, "simt") for k in (96, 100)],
    *[_r("simt128-f32-elem", k, False, "simt") for k in (65, 127)],
    _r("simt128-bf16-bulk", 96, True, "simt"),
    _r("simt128-bf16-elem", 100, True, "simt"),
    # tensor-core kernel (als_tc.cu)
    *[_r("tc-bf16mma", k, True, "bf16mma", kinds=("uniform", "explicit")) for k in (64, 128)],
    *[_r("tc-tf32", k, False, "tf32") for k in (64, 128)],
    *[_r("tc-tf32-bf16rows", k, True, "tf32", kinds=("weighted",)) for k in (64, 128)],
    # launch_als_tc hands these back to the SIMT kernel
    *[_r("fallback-misaligned", k, False, "simt", misaligned=True) for k in (64, 128)],
    _r("fallback-negative-conf", 64, False, "simt", kinds=("negative",)),
]
_DEFAULT_OPTS = {"LK_ALS_TC": 1, "LK_ALS_TF32": 1}
_ROUTE_BY_ID = {(r["id"], r["k"]): r for r in ROUTES}
assert len(_ROUTE_BY_ID) == len(ROUTES), "a route id appears twice at one k"


def route(id_: str, k: int) -> dict:
    """The ROUTES entry `id_` at k (a KeyError, at collection, if there is none)."""
    return _ROUTE_BY_ID[id_, k]


def route_params(*cases) -> list:
    """pytest params of (route, value, ...) tuples, named after the route and the values."""
    return [pytest.param(*c, id="-".join([f"{c[0]['id']}-k{c[0]['k']}", *map(str, c[1:])])) for c in cases]


def use_route(lk_options, r: dict) -> None:
    """Set the kernel switches to their defaults, then to the route's own."""
    for name, value in {**_DEFAULT_OPTS, **r.get("opts", {})}.items():
        lk_options(name, value)


def route_cases():
    for r in ROUTES:
        for kind in r["kinds"]:
            for which in ("trainer", "32"):
                yield pytest.param(r, kind, which, id=f"{r['id']}-k{r['k']}-{kind}-{which}")


@pytest.mark.parametrize("route,kind,which", list(route_cases()))
def test_route_rows(cuda_lib, lk_options, route, kind, which):
    """Every route, every mode it serves, at the trainers' part length for it and at 32: each row within bound."""
    use_route(lk_options, route)
    chunk = 32 if which == "32" else trainer_chunk(route["k"], route["bf16"], kind)
    st = case(route, kind, chunk)
    if route["id"].startswith("fallback"):
        # the fallback is the SIMT kernel: same bits as that kernel pinned on aligned rows (bulk and element copy
        # do the same arithmetic)
        lk_options("LK_ALS_TC", 0)
        simt, _, status, _ = run_device(kind, st["csr"], st["this"], st["other"], k=route["k"], bf16=False,
                                        chunk=chunk, otor32=st["o32"])  # fmt: skip
        assert status == 0
        assert np.array_equal(st["got"].view(np.int32), simt.view(np.int32))


BOUNDARY_ROUTES = [
    (route("simt64-f32-bulk", 48), "explicit"),  # pad columns 48..63 re-zeroed every chunk
    (route("simt128-f32-bulk", 100), "uniform"),
    (route("tc-bf16mma", 64), "uniform"),  # three stages, claim-ahead
    (route("tc-tf32", 64), "weighted"),
]


@pytest.mark.parametrize("chunk", [32, 64, 256, 1024, 4096])
@pytest.mark.parametrize("route,kind", [pytest.param(r, kd, id=f"{r['id']}-k{r['k']}-{kd}") for r, kd in BOUNDARY_ROUTES])
def test_boundary_rows_many_chunks_per_cta(cuda_lib, lk_options, route, kind, chunk):
    """The boundary lengths among ~16k short rows and a row of over 40 parts, so that each CTA of the persistent
    grid solves many chunks in sequence."""
    use_route(lk_options, route)
    st = case(route, kind, chunk, n_short=N_SHORT, many_parts=True)
    assert st["rows"] > N_SHORT


def test_checker_rejects_one_perturbed_row(cuda_lib, lk_options):
    """Self-test: one row of a passing result moved by 1e-3 relative fails the per-row check, while the
    matrix-level bar (relative Frobenius error < 1e-4) still accepts it."""
    r = route("simt64-f32-bulk", 64)
    use_route(lk_options, r)
    st = case(r, "uniform", 4096, n_short=N_SHORT, many_parts=True)
    got, x64, x32, csr = st["got"], st["x64"], st["x32"], st["csr"]
    assert rel_fro(got, x64) < 1e-4
    n = np.diff(csr.indptr)
    for r in (int(np.argmax(n)), int(np.flatnonzero(n == 17)[0])):
        bent = got.copy()
        u = np.random.default_rng(r).standard_normal(got.shape[1])
        bent[r] = (got[r] + 1e-3 * np.linalg.norm(x64[r]) * u / np.linalg.norm(u)).astype(np.float32)
        msgs, _ = row_failures(bent, x64, x32, csr, 4096, TOL["simt"])
        assert len(msgs) == 1 and msgs[0].startswith(f"row {r}:"), msgs
        assert rel_fro(bent, x64) < 1e-4


# ---------------------------------------------------------------------------
# one failing row among good ones
# ---------------------------------------------------------------------------

FAIL_ROUTES = [
    pytest.param(route("simt32-f32-bulk", 32), id="simt-k32"),
    pytest.param(route("tc-bf16mma", 64), id="bf16mma-k64"),
    pytest.param(route("tc-tf32", 64), id="tf32-k64"),
]


@pytest.mark.parametrize("route", FAIL_ROUTES)
def test_one_failing_row_among_good_ones(cuda_lib, lk_options, route):
    """A NaN row of `other` gathered by one whole row and one split row: status names one of them, both keep
    their old values, and every other row is solved, within bound, and counted in the delta."""
    use_route(lk_options, route)
    k, bf16, chunk = route["k"], route["bf16"], 32
    good = boundary_csr(chunk, "explicit", many_parts=True, seed=5)
    n = np.diff(good.indptr)
    whole, split = int(np.flatnonzero(n == 9)[0]), int(np.flatnonzero(n == 65)[0])
    nan_col = N_OTHER  # one extra row of `other`, all NaN, gathered only by these two rows
    cols, vals, indptr = [], [], [0]
    for r in range(len(n)):
        c = good.indices[good.indptr[r] : good.indptr[r + 1]]
        v = good.values[good.indptr[r] : good.indptr[r + 1]]
        if r in (whole, split):
            c, v = np.append(c, nan_col), np.append(v, np.float32(1.0))
        cols.append(c)
        vals.append(v)
        indptr.append(indptr[-1] + len(c))
    csr = data.InteractionCSR(np.array(indptr, np.int32), np.concatenate(cols).astype(np.int32),
                              np.concatenate(vals).astype(np.float32), (len(n), N_OTHER + 1))  # fmt: skip
    this, other = factors(len(n), N_OTHER + 1, k, 5)
    other[nan_col] = np.nan
    # oracle: the same matrix with the two failing rows emptied (an empty row adds nothing to the delta)
    keep = np.ones(len(n), bool)
    keep[[whole, split]] = False
    rows_ok = np.flatnonzero(keep & (n > 0))
    lens_ok = np.where(keep, np.diff(csr.indptr), 0)
    sel = np.concatenate([np.arange(csr.indptr[r], csr.indptr[r + 1]) for r in range(len(n)) if keep[r]])
    ref_csr = data.InteractionCSR(np.concatenate([[0], np.cumsum(lens_ok)]).astype(np.int32), csr.indices[sel],
                                  csr.values[sel], csr.shape)  # fmt: skip
    x64, d64, x32, _ = oracles("explicit", ref_csr, this, other, bf16=bf16)

    got, delta, status, plan = run_device("explicit", csr, this, other, k=k, bf16=bf16, chunk=chunk)
    assert row_parts(csr, chunk)[split] > 1 and row_parts(csr, chunk)[whole] == 1
    assert status - 1 in (whole, split), status
    for r in (whole, split):
        assert np.array_equal(got[r].view(np.int32), this[r].view(np.int32)), r
    check_rows(got, x64, x32, csr, chunk, TOL[route["family"]], route["id"], rows=rows_ok)
    assert np.all(got[n == 0] == 0.0)
    assert delta == pytest.approx(d64, rel=1e-3)


# ---------------------------------------------------------------------------
# replica writes (the path parallel.py uses for peer rows), on one device
# ---------------------------------------------------------------------------


@pytest.mark.parametrize(
    "route,kind",
    [
        pytest.param(route("simt32-f32-bulk", 32), "uniform", id="simt-k32"),
        pytest.param(route("tc-bf16mma", 64), "uniform", id="bf16mma-k64"),
        pytest.param(route("tc-tf32", 128), "explicit", id="tf32-k128"),
    ],
)
def test_replica_rows_match_this(cuda_lib, lk_options, route, kind):
    """replicas=[r], replica_row0=row0: r[row0 + row] holds exactly the bits of this[row] (zeros for empty rows),
    and nothing outside that window is written."""
    use_route(lk_options, route)
    k, bf16, chunk = route["k"], route["bf16"], 32
    csr = boundary_csr(chunk, kind, many_parts=True, seed=9)
    n_rows = csr.shape[0]
    this, other = factors(n_rows, N_OTHER, k, 9)
    o32 = oracle.otor(oracle.bf16_round(other) if bf16 else other, REG)[0] if kind != "explicit" else None
    row0, margin = 37, 11
    dev = _lib.require_device()
    sentinel = -123.25
    rep = torch.full((row0 + n_rows + margin, k), sentinel, dtype=torch.float32, device=dev)
    got, _, status, _ = run_device(kind, csr, this, other, k=k, bf16=bf16, chunk=chunk, otor32=o32,
                                   replicas=[rep], replica_row0=row0)  # fmt: skip
    assert status == 0
    r = rep.cpu().numpy()
    assert np.array_equal(r[row0 : row0 + n_rows].view(np.int32), got.view(np.int32))
    assert np.all(r[row0 : row0 + n_rows][np.diff(csr.indptr) == 0] == 0.0)
    assert np.all(r[:row0] == sentinel) and np.all(r[row0 + n_rows :] == sentinel)


# ---------------------------------------------------------------------------
# whole matrices on the tensor-core kernel, OtOr and the bf16 copy of `other` built on the device
# ---------------------------------------------------------------------------

#: relative Frobenius distance to the SIMT kernel (LK_ALS_TC=0) on the same inputs, by (family, k).  The bounds
#: are the ones each path was first tested with: bf16mma agrees with the SIMT kernel to rounding; the tf32 x3 Gram
#: drops the lo.lo term and truncates lo, so it sits a few 1e-5 from f32 arithmetic, inside the 1e-4 bound against
#: the f64 oracle.  The worst distances over test_parity's cases on an H100 80GB HBM3 (700 W power limit) were
#: 5.6e-7 / 1.5e-6 for bf16mma and 6.6e-6 / 2.2e-5 for tf32 at k = 64 / 128.
SIMT_AGREEMENT = {("bf16mma", 64): 2e-5, ("bf16mma", 128): 3e-5, ("tf32", 64): 6e-5, ("tf32", 128): 6e-5}


@pytest.mark.parametrize(
    "route,kind,chunk,seed",
    route_params(
        *[(route("tc-bf16mma", 64), kind, chunk, 21)
          for kind in ("uniform", "explicit") for chunk in (DEFAULT_CHUNK, 256, 64, 32)],
        *[(route("tc-tf32", k), kind, DEFAULT_CHUNK, 21) for k in (64, 128) for kind in ALL],
        *[(route("tc-tf32-bf16rows", k), "weighted", DEFAULT_CHUNK, 21) for k in (64, 128)],
        (route("tc-bf16mma", 128), "explicit", DEFAULT_CHUNK, 21),
        *[(route("tc-bf16mma", 128), kind, DEFAULT_CHUNK, 31) for kind in ("uniform", "explicit")],
    ),
)
def test_parity(cuda_lib, lk_options, route, kind, chunk, seed):
    """Both half-steps against the f64 oracle and against the SIMT kernel, for row parts from whole rows down to
    32 nonzeros (split rows are summed from their partial systems in slot order)."""
    use_route(lk_options, route)
    k, bf16 = route["k"], route["bf16"]
    inter = small_synth(900, 500, 40000, seed=seed)
    rng = np.random.default_rng(seed)
    p, q = synth_factors(rng, inter.n_users, inter.n_items, k)
    ui, iu = synth_matrices(inter, kind, rng)
    for csr, this, other in ((ui, p, q), (iu, q, p)):
        got, delta, status, plan = run_device(kind, csr, this, other, k=k, bf16=bf16, chunk=chunk, device_otor=True)
        assert status == 0
        assert plan.vals_uniform == (kind == "uniform")
        if chunk < 64:
            assert plan.n_split_rows > 0
        x64, d64, _ = oracle64(kind, csr, this, other, bf16=bf16)
        assert rel_fro(got, x64) < 1e-4, rel_fro(got, x64)
        assert delta == pytest.approx(d64, rel=1e-3)
        assert np.all(got[np.diff(csr.indptr) == 0] == 0.0)
        lk_options("LK_ALS_TC", 0)
        simt, _, status, _ = run_device(kind, csr, this, other, k=k, bf16=bf16, chunk=chunk, device_otor=True)
        lk_options("LK_ALS_TC", 1)
        assert status == 0
        assert rel_fro(got, simt) < SIMT_AGREEMENT[route["family"], k], rel_fro(got, simt)


@pytest.mark.parametrize(
    "route,kind,chunk",
    route_params(
        *[(route("tc-bf16mma", 64), kind, chunk) for kind in ("uniform", "explicit") for chunk in (32, 64, 96)],
        *[(route("tc-tf32", k), kind, 32) for k in (64, 128) for kind in ALL],
        *[(route("tc-bf16mma", 128), kind, 32) for kind in ("uniform", "explicit")],
    ),
)
def test_split_rows_deterministic(cuda_lib, lk_options, route, kind, chunk):
    """Rows cut into parts of `chunk` nonzeros (96: not a power of two) give the same bits on a rerun, stay within
    the oracle's bound and close to the one-part solve."""
    use_route(lk_options, route)
    k, bf16 = route["k"], route["bf16"]
    inter = small_synth(300, 200, 20000, seed=5)
    rng = np.random.default_rng(5)
    _ui, iu = synth_matrices(inter, kind, rng)
    p, q = synth_factors(rng, 300, 200, k)
    a, _, status, plan = run_device(kind, iu, q, p, k=k, bf16=bf16, chunk=chunk, device_otor=True)
    assert status == 0
    assert plan.n_split_rows > 0
    b, _, status, _ = run_device(kind, iu, q, p, k=k, bf16=bf16, chunk=chunk, device_otor=True)
    assert status == 0
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    x64, _, _ = oracle64(kind, iu, q, p, bf16=bf16)
    assert rel_fro(a, x64) < 1e-4
    c, _, status, _ = run_device(kind, iu, q, p, k=k, bf16=bf16, chunk=1 << 20, device_otor=True)
    assert status == 0
    # split (parts added with round-to-nearest) vs unsplit (one tensor-core accumulation chain per row): the
    # accumulation orders differ, and on the tf32 path the 128x128 solve amplifies that more than the 64x64 one
    assert rel_fro(a, c) < (1e-4 if (route["family"], k) == ("tf32", 128) else 1e-5)


@pytest.mark.parametrize(
    "route,reg",
    route_params(
        (route("tc-bf16mma", 64), 1e-2),
        (route("tc-bf16mma", 64), 1e-3),
        (route("tc-tf32", 64), 1e-2),
        (route("tc-bf16mma", 128), 1e-2),
    ),
)
def test_badly_conditioned(cuda_lib, lk_options, route, reg):
    """Large Gram, small ridge (cond ~1e4 at reg 1e-2, ~1e5 at 1e-3): the tensor-core kernel stays within a small
    factor of what f32 arithmetic can deliver (the f32 oracle's own distance to the f64 oracle)."""
    use_route(lk_options, route)
    k, bf16 = route["k"], route["bf16"]
    inter = small_synth(400, 300, 60000, seed=9)
    rng = np.random.default_rng(9)
    ui, _ = synth_matrices(inter, "uniform", rng)
    p = (rng.standard_normal((400, k)) * 0.1).astype(np.float32)
    q = rng.standard_normal((300, k)).astype(np.float32)  # trained-scale-and-beyond item factors
    got, _, status, _ = run_device("uniform", ui, p, q, k=k, bf16=bf16, device_otor=True, reg=reg)
    assert status == 0
    x64, _, x32, _ = oracles("uniform", ui, p, q, bf16=bf16, reg=reg)
    e_gpu, e_cpu = rel_fro(got, x64), rel_fro(x32, x64)
    assert e_gpu < max(1e-4, 3.0 * e_cpu), (e_gpu, e_cpu)


@pytest.mark.parametrize(
    "route,kind",
    route_params(
        (route("tc-bf16mma", 64), "uniform"),
        (route("tc-tf32", 64), "uniform"),
        (route("tc-tf32", 64), "weighted"),
        (route("tc-bf16mma", 128), "uniform"),
    ),
)
def test_not_positive_definite_is_reported(cuda_lib, lk_options, route, kind):
    """A system that is not positive definite (the reference's `ALS solve error`, implicit.rs:79) sets the status
    word and leaves the row untouched, on each Gram path of the tensor-core kernel: bf16 MMAs, tf32 x3 on fp32
    rows, tf32 x3 on sqrt(v)-scaled rows (per-nonzero confidences)."""
    use_route(lk_options, route)
    k, bf16 = route["k"], route["bf16"]
    ui, _ = synth_matrices(small_synth(60, 40, 600, seed=2), kind, None)
    this, other = np.full((60, k), 0.5, np.float32), np.zeros((40, k), np.float32)
    got, _, status, plan = run_device(kind, ui, this, other, k=k, bf16=bf16, otor32=-np.eye(k, dtype=np.float32),
                                      reg=0.0)  # fmt: skip
    assert plan.vals_uniform == (kind == "uniform")
    assert status > 0
    assert np.all(got[np.diff(ui.indptr) > 0] == 0.5)  # failed solves do not write


def test_zero_weight(cuda_lib, lk_options):
    """weight = 0 makes every confidence 0: A = OtOr, the Gram scaled by zero."""
    r = route("tc-bf16mma", 64)
    use_route(lk_options, r)
    ui, _ = data.als_implicit_matrices(small_synth(200, 150, 5000, seed=3), 0.0)
    p, q = synth_factors(np.random.default_rng(3), 200, 150, 64)
    got, _, status, _ = run_device("uniform", ui, p, q, k=64, bf16=r["bf16"], device_otor=True)
    assert status == 0
    x64, _, _ = oracle64("uniform", ui, p, q, bf16=r["bf16"])
    assert np.isfinite(got).all()
    assert rel_fro(got, x64) < 1e-4


@pytest.mark.parametrize("route", route_params(*[(route("tc-tf32", k),) for k in (64, 128)]))
def test_tf32_switch_off(cuda_lib, lk_options, route):
    """LK_ALS_TF32=0 sends fp32 rows back to the SIMT kernel (same bits as LK_ALS_TC=0)."""
    use_route(lk_options, route)
    k = route["k"]
    ui, _ = synth_matrices(small_synth(300, 200, 9000, seed=6), "uniform", None)
    p, q = synth_factors(np.random.default_rng(6), 300, 200, k)
    lk_options("LK_ALS_TF32", 0)
    a, _, status_a, _ = run_device("uniform", ui, p, q, k=k, bf16=False, device_otor=True)
    lk_options("LK_ALS_TF32", 1)
    lk_options("LK_ALS_TC", 0)
    b, _, status_b, _ = run_device("uniform", ui, p, q, k=k, bf16=False, device_otor=True)
    assert status_a == status_b == 0
    assert np.array_equal(a.view(np.int32), b.view(np.int32))


def test_ml_small_half_steps(cuda_lib, lk_options, ml_small):
    """Config 1 (ml-latest-small, reference init): both half-steps from the init on the fp32 tensor-core path
    track the f64 oracle as closely as the f32 oracle does (the init makes the first systems ill-conditioned)."""
    use_route(lk_options, route("tc-tf32", 64))
    ui, iu = synth_matrices(ml_small, "uniform", None)
    p, q = implicit_init(np.random.default_rng(42), ml_small.n_items, ml_small.n_users, 64)
    for csr, this, other in ((ui, p, q), (iu, q, p)):
        got, _, status, _ = run_device("uniform", csr, this, other, k=64, bf16=False, device_otor=True)
        assert status == 0
        x64, _, x32, _ = oracles("uniform", csr, this, other, bf16=False)
        assert rel_fro(got, x64) < max(1e-4, 1.5 * rel_fro(x32, x64)), (rel_fro(got, x64), rel_fro(x32, x64))


def test_short_and_odd_rows(cuda_lib, lk_options):
    """k = 128 rows of 1..40 nonzeros (not multiples of the 16-row stage), an odd number of chunks, empty rows."""
    r = route("tc-bf16mma", 128)
    use_route(lk_options, r)
    rng = np.random.default_rng(3)
    n_rows, n_other = 77, 150
    lens = rng.integers(0, 41, n_rows)
    lens[[0, 5]] = 0
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = np.concatenate([np.sort(rng.choice(n_other, n, replace=False)) for n in lens]).astype(np.int32)
    csr = data.InteractionCSR(indptr, cols, np.full(len(cols), UNIFORM_CONF, np.float32), (n_rows, n_other))
    p, q = synth_factors(rng, n_rows, n_other, 128)
    got, _, status, _ = run_device("uniform", csr, p, q, k=128, bf16=r["bf16"], device_otor=True)
    assert status == 0
    x64, _, _ = oracle64("uniform", csr, p, q, bf16=r["bf16"])
    assert rel_fro(got, x64) < 1e-4
    assert np.all(got[lens == 0] == 0.0)


# ---------------------------------------------------------------------------
# an exact zero pivot
# ---------------------------------------------------------------------------


@pytest.mark.parametrize(
    "route",
    route_params(
        (route("simt32-f32-bulk", 32),),
        (route("simt64-f32-bulk", 64),),  # LK_ALS_TF32=0
        (route("tc-bf16mma", 64),),
        (route("tc-tf32", 64),),
    ),
)
@pytest.mark.parametrize("where", ["first", "mid", "last"])
def test_zero_pivot_row_is_reported_and_untouched(cuda_lib, lk_options, route, where):
    """A row solve whose pivot is exactly zero (not NaN) is reported and leaves its row untouched.

    Explicit mode with reg = 0 makes the system the bare Gram.  Gathered rows of `other` that are zero from feature
    f0 on give a Gram whose rows and columns from f0 on are exactly zero, so the factorisation meets a zero pivot at
    column f0 (column 0, the middle of a panel and the last column are tried).  Every other row gathers enough
    random rows to be well conditioned and must still be solved."""
    use_route(lk_options, route)
    k, bf16 = route["k"], route["bf16"]
    f0 = {"first": 0, "mid": k // 2 + 3, "last": k - 1}[where]
    rng = np.random.default_rng([k, f0, 11])
    n_good, n_other, per_row = 40, 400, 3 * k
    other = (rng.standard_normal((n_other + 8, k)) * 0.5).astype(np.float32)
    other[n_other:, f0:] = 0.0  # the last 8 rows of `other` span only features 0 .. f0-1
    bad_row = 17
    cols, vals, indptr = [], [], [0]
    for r in range(n_good + 1):
        if r == bad_row:
            c = np.arange(n_other, n_other + 8)
        else:
            c = np.sort(rng.choice(n_other, per_row, replace=False))
        cols.append(c)
        vals.append(rng.uniform(1.0, 5.0, len(c)).astype(np.float32))
        indptr.append(indptr[-1] + len(c))
    csr = data.InteractionCSR(np.array(indptr, np.int32), np.concatenate(cols).astype(np.int32),
                              np.concatenate(vals), (n_good + 1, n_other + 8))  # fmt: skip
    this = (rng.standard_normal((n_good + 1, k)) * 0.1).astype(np.float32)
    got, _, status, _ = run_device("explicit", csr, this, other, k=k, bf16=bf16, chunk=1024, reg=0.0)

    assert status == bad_row + 1
    assert np.array_equal(got[bad_row].view(np.int32), this[bad_row].view(np.int32))
    # the other rows: A x = O^T v with the (bf16-rounded) gathered rows, in f64
    o = (oracle.bf16_round(other) if bf16 else other).astype(np.float64)
    for r in range(n_good + 1):
        if r == bad_row:
            continue
        c, v = csr.indices[csr.indptr[r] : csr.indptr[r + 1]], csr.values[csr.indptr[r] : csr.indptr[r + 1]]
        x = np.linalg.solve(o[c].T @ o[c], o[c].T @ v.astype(np.float64))
        assert np.linalg.norm(got[r] - x) <= 1e-3 * np.linalg.norm(x), r
