#!/usr/bin/env python
"""
FlexMF training at the synthetic ML-25M shape (162,541 x 59,047, 25,000,095 interactions), k = 64, on one GPU:
``--model implicit`` (default) with negative_count 1, or ``--model explicit``, the squared error on the generator's
ratings less their mean, no negatives and no bias terms (the reference's explicit model).  Per configuration and
batch size:

* epoch time (host clock around a synchronise; median of ``--epochs`` epochs after one warm-up epoch), split into the
  part before the first step (``plan_batches``: sampling, sorting, grouping) and the steps (``run_batches``);
* the same ``--steps`` steps on the device step and on the plain-torch step of ``tests/flexmf_oracle.py`` (explicit:
  ``tests/flexmf_explicit_oracle.py``) run on the same device (autograd + ``torch.optim``), alternated, both fed the
  device sampler's negatives and neither charged for the grouping; their parameters are compared first (update error ‖new − want‖ / ‖want − old‖ after ``--steps`` steps, bound 1e-3: f32 rounding
  through that many Adam steps);
* kernel time per step by kernel name from ``torch.profiler`` in a separate pass over the steps alone, the launch gaps
  (wall time per step with the profiler off minus that sum), and the bytes each kernel must move, from shapes, against 3.35 TB/s;
* implicit only: a NumPy rejection sampler on the host for one batch, the stand-in for what a host-side sampler
  costs per step.

Prints one JSON line per measurement; needs a CUDA device.
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
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import flexmf_explicit_oracle as feo  # noqa: E402
import flexmf_oracle as fo  # noqa: E402
from lkpy_b200 import _lib, engine, flexmf, prep  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
CONFIGS = [("logistic", "AdamW", True), ("logistic", "L2", True), ("pairwise", None, False)]
EXPLICIT_CONFIGS = [("mse", "L2", False), ("mse", "AdamW", False), ("mse", None, False)]


def step_bytes(n_users, n_items, k, B, n, reg_method, ub, ib, uniq_u, uniq_i, targets=False) -> dict[str, float]:
    """Bytes each kernel of a step has to move, from shapes (row gathers counted once per occurrence)."""
    row = 4 * k
    fwd = B * (row + (n + 1) * row) + 4 * B * (n + 3) + 4 * B * (n + 2)  # rows, indices and biases, coef + loss out
    fwd += 4 * B if targets else 0
    grad = B * (n + 1) * row * 2 + 4 * B * (n + 1) * 2 + (uniq_u + uniq_i) * (row + 4)  # both sides' gathers, partials
    cols = k + (1 if ub else 0), k + (1 if ib else 0)
    if reg_method == "AdamW":
        upd = (n_users * cols[0] + n_items * cols[1]) * 4 * 6 + 8 * (n_users + n_items)
    else:
        upd = (uniq_u * cols[0] + uniq_i * cols[1]) * 4 * 7
    return {"flexmf_forward_kernel": fwd, "flexmf_grad_kernel": grad, "flexmf_update_kernel": upd,
            "flexmf_loss_kernel": 4 * B}  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=162_541)
    ap.add_argument("--items", type=int, default=59_047)
    ap.add_argument("--nnz", type=int, default=25_000_095)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--batch-sizes", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--model", choices=["implicit", "explicit"], default="implicit")
    a = ap.parse_args()
    explicit = a.model == "explicit"
    dev = _lib.require_device()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()  # fmt: skip
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi}), flush=True)
    users, items, ratings = prep.synth_interactions_device(a.users, a.items, a.nnz, device=dev)
    k, n = 64, 0 if explicit else 1
    targets = None
    if explicit:  # the explicit trainer's targets: ratings less their f32 mean, formed on the host
        host_r = ratings.cpu()
        targets = (host_r - host_r.mean()).to(dev)
    else:
        # host rejection sampler, one batch of 8,192
        hu, hi = users.cpu().numpy(), items.cpu().numpy()
        indptr = np.concatenate([[0], np.cumsum(np.bincount(hu, minlength=a.users))])
        rows = hu[np.random.default_rng(0).integers(0, a.nnz, 8192)]
        t0 = time.perf_counter()
        fo.sample_negatives(indptr, hi, rows, a.items, n, seed=1)
        print(json.dumps({"host_numpy_sampler_ms_per_8192_batch": (time.perf_counter() - t0) * 1e3}), flush=True)

    for loss, reg_method, biases in EXPLICIT_CONFIGS if explicit else CONFIGS:
        for B in a.batch_sizes:
            tag = ({"model": "explicit"} if explicit else {}) | {"loss": loss, "reg_method": reg_method, "batch_size": B}
            params = flexmf.initial_parameters(a.users, a.items, k, biases, biases, torch.Generator().manual_seed(1))
            mk = lambda: engine.FlexMFState(params, users, items, loss=loss, reg_method=reg_method, batch_size=B,  # noqa: E731
                                            negative_count=n, ratings=targets, seed=5, device=dev)  # fmt: skip
            # --- the same steps on both paths: first compared, then timed alternately
            st = mk()
            at = torch.randperm(a.nnz, device=dev, generator=torch.Generator(dev).manual_seed(3))[: a.steps * B]
            su, sp = users[at], items[at]
            sneg = None if explicit else st.sample(su)
            sr = targets[at] if explicit else None
            model = fo.Model(params, sparse=reg_method != "AdamW", device=dev)
            opt = fo.make_optimizer(model, reg_method, st.lr, st.reg)
            kw = dict(loss=loss, reg_method=reg_method, regularization=st.reg, positive_weight=1.0)

            def torch_steps():
                for s in range(a.steps):
                    sl = slice(s * B, (s + 1) * B)
                    if explicit:
                        out, _ = feo.mse_terms(model, su[sl], sp[sl], sr[sl], reg_method=reg_method, regularization=st.reg)
                    else:
                        out = fo.batch_loss(model, su[sl], sp[sl], sneg[sl], **kw)
                    out.backward()
                    opt.step()
                    opt.zero_grad()

            def timed(fn):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                return out, time.perf_counter() - t0

            plan, plan_s = timed(lambda: st.plan_batches(su, sp, sneg, ratings=sr))  # sorts and grouping: not part of a step
            st.run_batches(plan)
            torch_steps()
            errs = {}
            for name, want in model.state_dict().items():
                old = params[name].to(dev)
                errs[name] = float((st.params[name] - want).norm() / (want - old).norm())
            assert max(errs.values()) < 1e-3, errs
            times = {"device": [], "torch": []}
            for _rep in range(3):
                for which, fn in (("device", lambda: st.run_batches(plan)), ("torch", torch_steps)):
                    times[which].append(timed(fn)[1] / a.steps * 1e3)
            dev_ms = statistics.median(times["device"])
            print(json.dumps(tag | {"steps": a.steps, "update_error_vs_torch": max(errs.values()),
                                    "device_ms_per_step": dev_ms, "torch_ms_per_step": statistics.median(times["torch"]),
                                    "grouping_ms_for_these_steps": plan_s * 1e3}), flush=True)  # fmt: skip
            del model, opt

            # --- kernel times (separate pass, profiler on; the steps only)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA,
                                                    torch.profiler.ProfilerActivity.CPU]) as prof:  # fmt: skip
                timed(lambda: st.run_batches(plan))
            kern = {}
            for e in prof.key_averages():
                if "flexmf_" in e.key:
                    name = next(nm for nm in ("forward", "loss", "grad", "update", "sample") if f"flexmf_{nm}" in e.key)
                    kern[f"flexmf_{name}_kernel"] = kern.get(f"flexmf_{name}_kernel", 0.0) + e.device_time_total / a.steps
            uq_u = float(torch.unique(su[:B]).numel())
            uq_i = float(torch.unique(sp[:B] if explicit else torch.cat([sp[:B], sneg[:B, 0]])).numel())
            need = step_bytes(a.users, a.items, k, B, n, reg_method, biases, biases, uq_u, uq_i, targets=explicit)
            rows_out = {nm: {"us_per_step": us, "bytes": need.get(nm), "share_of_3.35TBps":
                             (need[nm] / HBM_BYTES_PER_S) / (us * 1e-6) if nm in need and us > 0 else None}
                        for nm, us in kern.items()}  # fmt: skip
            ksum = sum(kern.values())
            print(json.dumps(tag | {"profiled_steps": a.steps, "kernels": rows_out, "kernel_us_per_step": ksum,
                                    "launch_gap_us_per_step": dev_ms * 1e3 - ksum}), flush=True)  # fmt: skip
            del plan

            # --- whole epochs
            st = mk()
            rng = np.random.default_rng(2)
            ep = []
            for e in range(a.epochs + 1):
                perm = torch.from_numpy(rng.permutation(a.nnz)).to(dev)
                plan, plan_s = timed(lambda: st.plan_batches(users[perm], items[perm],
                                                             ratings=targets[perm] if explicit else None))  # fmt: skip
                losses, run_s = timed(lambda: st.run_batches(plan))
                del plan
                mean = float(losses.double().mean().item())
                ep.append((plan_s + run_s, plan_s, run_s))
            med = lambda j: statistics.median(x[j] for x in ep[1:])  # noqa: E731
            print(json.dumps(tag | {"epoch_s_median": med(0), "of_which_sampling_and_grouping_s": med(1),
                                    "of_which_steps_s": med(2), "steps_per_epoch": -(-a.nnz // B),
                                    "last_epoch_loss": mean}), flush=True)  # fmt: skip
            del st


if __name__ == "__main__":
    main()
