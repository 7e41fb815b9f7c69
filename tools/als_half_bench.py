"""
The two halves of the ALS-implicit epoch timed apart, at ``bench.py``'s shape (synthetic ML-25M, k = 64,
weight 40, reg 0.1): CUDA events around the user-half and the item-half row-solve launches, and around whole
epochs, for bf16 and fp32 gathered rows.  ``bench.py`` reports only the sum of the two launches.

Each variant runs ``--warmup`` epochs first (at least 3, so the timed epochs see trained-scale factors), then
``--steps`` epochs with events around the epoch, then ``--steps`` more with events around each launch.  Prints one
JSON object with the medians, and writes it to ``--out`` when given.
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from lkpy_b200 import _lib, data  # noqa: E402
from lkpy_b200.als import ImplicitMFScorer, ImplicitMFTrainer  # noqa: E402
from lkpy_b200.components import Dataset, TrainingOptions  # noqa: E402

K, WEIGHT, REG = 64, 40.0, 0.1  # bench.py's ALS configuration


def run(ds, gather_dtype: str, steps: int, warmup: int) -> dict:
    scorer = ImplicitMFScorer(features=K, epochs=1, regularization=REG, weight=WEIGHT, gather_dtype=gather_dtype)
    tr = ImplicitMFTrainer(scorer, ds, TrainingOptions(rng=42))
    for _ in range(max(warmup, 3)):
        tr.train_epoch_device()
    epoch = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        tr.train_epoch_device()
        e1.record()
        epoch.append((e0, e1))
    tr.kernel_events = []
    for _ in range(steps):
        tr.train_epoch_device()
    torch.cuda.synchronize()
    tr._raise_on_status()
    ms = [a.elapsed_time(b) for a, b in tr.kernel_events]
    assert len(ms) == 2 * steps, "one user-half and one item-half launch per epoch"
    return {
        "kernel": tr.solve_kernel_name(),
        "epoch_ms": statistics.median(a.elapsed_time(b) for a, b in epoch),
        "user_half_ms": statistics.median(ms[0::2]),
        "item_half_ms": statistics.median(ms[1::2]),
        "solve_ms": statistics.median(u + i for u, i in zip(ms[0::2], ms[1::2])),
    }


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--variants", default="bf16,fp32")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("als_half_bench.py needs a CUDA device")
    _lib.lib()
    torch.cuda.set_device(0)
    inter = data.synth_interactions_cached(os.environ.get("LK_BENCH_DATA_CACHE"), **data.ML25M_SHAPE)
    ds = Dataset(inter)
    out = {
        "device": torch.cuda.get_device_name(0),
        "shape": {"n_users": inter.n_users, "n_items": inter.n_items, "nnz": inter.nnz, "k": K},
        "steps": args.steps,
    }
    dtypes = {"bf16": "bfloat16", "fp32": "float32"}
    for tag in (v for v in args.variants.split(",") if v):
        out[tag] = run(ds, dtypes[tag], args.steps, args.warmup)
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
