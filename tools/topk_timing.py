"""Timing of the top-k similarity search against what a user had before it: row-blocked crossTanimotoSimilarity +
torch.topk. 2048-bit clustered fingerprints, a library of 1M, Q in {1, 1024, 16384}, k in {10, 100}, cosine at one of
them. CUDA-event times (3 warm-ups, median of 5, min-max printed), the two alternating in one process, results compared.
Needs a GPU; there is no CPU fallback.

    python tools/topk_timing.py [--library 1000000] [--out results.json]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nvmolkit_b200 import _lib, synthetic  # noqa: E402
from nvmolkit_b200.similarity import (crossCosineSimilarity, crossTanimotoSimilarity, topKCosineSimilarity,  # noqa: E402
                                      topKTanimotoSimilarity)

WARMUP, REPEATS = 3, 5
BLOCK_BYTES = 4 << 30  # the baseline's matrix block


def card() -> str:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()]


def timed(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop), out


def baseline(cross, q, lib, k):
    rows = max(1, BLOCK_BYTES // (8 * lib.shape[0]))
    vals, idx = [], []
    for r0 in range(0, q.shape[0], rows):
        v, i = torch.topk(cross(q[r0:r0 + rows], lib).torch(), k, dim=1)
        vals.append(v)
        idx.append(i)
    return torch.cat(vals), torch.cat(idx)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--library", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("topk_timing.py needs a CUDA device")
    name = card()
    print(f"card: {name}")
    n_q = 16384
    fps = synthetic.clustered_fingerprints((args.library + n_q + 24) // 25, 25, seed=7)
    lib = torch.from_numpy(fps[:args.library].view(np.int32)).cuda()
    queries = torch.from_numpy(fps[args.library:args.library + n_q].view(np.int32)).cuda()
    rows = []
    for metric, nq, k in (("tanimoto", 1, 10), ("tanimoto", 1, 100), ("tanimoto", 1024, 10), ("tanimoto", 1024, 100),
                          ("tanimoto", 16384, 10), ("tanimoto", 16384, 100), ("cosine", 1024, 100)):
        search = topKTanimotoSimilarity if metric == "tanimoto" else topKCosineSimilarity
        cross = crossTanimotoSimilarity if metric == "tanimoto" else crossCosineSimilarity
        q = queries[:nq]
        ours = lambda: tuple(r.torch() for r in search(q, lib, k=k))  # noqa: E731
        base = lambda: baseline(cross, q, lib, k)  # noqa: E731
        t_ours, t_base = [], []
        for it in range(WARMUP + REPEATS):
            ms_o, (v, i) = timed(ours)
            ms_b, (bv, bi) = timed(base)
            if it >= WARMUP:
                t_ours.append(ms_o)
                t_base.append(ms_b)
        same_values = bool(torch.equal(v, bv))
        same_at_indices = bool(torch.equal(torch.gather(cross(q[:256], lib).torch(), 1, i[:256].long()), v[:256]))
        pairs = nq * args.library
        row = {"metric": metric, "queries": nq, "library": args.library, "k": k,
               "topk_ms": statistics.median(t_ours), "topk_ms_min_max": [min(t_ours), max(t_ours)],
               "baseline_ms": statistics.median(t_base), "baseline_ms_min_max": [min(t_base), max(t_base)],
               "topk_pairs_per_s": pairs / (statistics.median(t_ours) * 1e-3),
               "values_equal_baseline": same_values, "values_are_matrix_entries_at_indices": same_at_indices,
               "slabs": _lib.get_option("topk_slabs_last"), "candidates_listed": _lib.get_option("topk_candidates_last"),
               "rows_redone": _lib.get_option("topk_rows_redone_last"), "tiles_skipped_by_popcount_bound": 0}
        row["candidates_per_slab"] = row["candidates_listed"] / max(1, row["slabs"])
        rows.append(row)
        print(json.dumps(row))
        if not (same_values and same_at_indices):
            sys.exit("top-k search and the baseline disagree")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
