"""Timing of the threshold similarity search against what a user had before it: row-blocked crossTanimotoSimilarity /
crossCosineSimilarity + (block >= t).nonzero() + concatenation into the same CSR. 2048-bit clustered fingerprints, a
library of 1M: Q in {1024, 16384} at Tanimoto 0.7 / 0.8 and cosine 0.8, self searches of 100k and 1M (the 1M baseline
would write ~8 TB of fp64 and is not run), and a dense case with about 1,000 hits per query. CUDA-event times (3 warm-ups,
median of 5, min-max printed), the two alternating in one process, results compared for equality; the search's time is
split into its pass, its re-count and its assembly by one further profiled call. Needs a GPU; there is no CPU fallback.

    python tools/threshold_timing.py [--library 1000000] [--out results.json]
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
from nvmolkit_b200.similarity import (crossCosineSimilarity, crossTanimotoSimilarity,  # noqa: E402
                                      thresholdCosineSimilarity, thresholdTanimotoSimilarity)

WARMUP, REPEATS = 3, 5
BLOCK_BYTES = 4 << 30  # the baseline's matrix block
PHASES = ("threshold_pass", "threshold_recount", "threshold_assembly")


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


def baseline(cross, q, lib, t):
    rows = max(1, BLOCK_BYTES // (8 * lib.shape[0]))
    counts, cols, vals = [], [], []
    for r0 in range(0, q.shape[0], rows):
        block = cross(q[r0:r0 + rows], lib).torch()
        r, c = (block >= t).nonzero(as_tuple=True)
        counts.append(torch.bincount(r, minlength=block.shape[0]))
        cols.append(c.to(torch.int32))
        vals.append(block[r, c])
    indptr = torch.zeros(q.shape[0] + 1, dtype=torch.int64, device=q.device)
    indptr[1:] = torch.cumsum(torch.cat(counts), 0)
    return indptr, torch.cat(cols), torch.cat(vals)


def phases(search, q, lib, t) -> dict:
    _lib.profile_enable(True)
    try:
        search(q, lib, threshold=t)
        torch.cuda.synchronize()
        return {p: _lib.profile_read(p) for p in PHASES}
    finally:
        _lib.profile_enable(False)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--library", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("threshold_timing.py needs a CUDA device")
    name = card()
    print(f"card: {name}")
    n_q = 16384
    fps = synthetic.clustered_fingerprints((args.library + n_q + 24) // 25, 25, seed=7)
    lib = torch.from_numpy(fps[:args.library].view(np.int32)).cuda()
    queries = torch.from_numpy(fps[args.library:args.library + n_q].view(np.int32)).cuda()
    # dense: 1,000 members per centre, so a query has about 1,000 hits
    dense = synthetic.clustered_fingerprints((args.library + 1024) // 1000 + 1, 1000, seed=8)
    dense_lib = torch.from_numpy(dense[:args.library].view(np.int32)).cuda()
    dense_q = torch.from_numpy(dense[args.library:args.library + 1024].view(np.int32)).cuda()
    del fps, dense
    cases = [("tanimoto", "cross", 16384, 0.7), ("tanimoto", "cross", 16384, 0.8), ("cosine", "cross", 16384, 0.8),
             ("tanimoto", "cross", 1024, 0.7), ("tanimoto", "cross", 1024, 0.8), ("cosine", "cross", 1024, 0.8),
             ("tanimoto", "dense", 1024, 0.7), ("cosine", "dense", 1024, 0.7),
             ("tanimoto", "self", 100_000, 0.7), ("cosine", "self", 100_000, 0.8), ("tanimoto", "self", args.library, 0.7)]
    rows = []
    for metric, kind, nq, t in cases:
        search = thresholdTanimotoSimilarity if metric == "tanimoto" else thresholdCosineSimilarity
        cross = crossTanimotoSimilarity if metric == "tanimoto" else crossCosineSimilarity
        if kind == "cross":
            q, y = queries[:nq], lib
        elif kind == "dense":
            q, y = dense_q[:nq], dense_lib
        else:
            q, y = lib[:nq], None
        ours = lambda: tuple(r.torch() for r in search(q, y, threshold=t))  # noqa: E731
        with_baseline = not (kind == "self" and nq > 100_000)  # (the 1M x 1M matrix: ~8 TB of fp64 writes)
        base = lambda: baseline(cross, q, q if y is None else y, t)  # noqa: E731
        t_ours, t_base = [], []
        for it in range(WARMUP + REPEATS):
            ms_o, got = timed(ours)
            if it >= WARMUP:
                t_ours.append(ms_o)
            if with_baseline:
                ms_b, want = timed(base)
                if it >= WARMUP:
                    t_base.append(ms_b)
        equal = all(torch.equal(a, b) for a, b in zip(got, want)) if with_baseline else None
        m = q.shape[0] if y is None else y.shape[0]
        row = {"metric": metric, "kind": kind, "queries": nq, "library": m, "threshold": t, "nnz": int(got[0][-1]),
               "threshold_ms": statistics.median(t_ours), "threshold_ms_min_max": [min(t_ours), max(t_ours)],
               "pairs_per_s": nq * m / (statistics.median(t_ours) * 1e-3),
               "superpose_last": _lib.get_option("similarity_superpose_last") if metric == "tanimoto" else None,
               "phase_ms": phases(search, q, y, t), "results_equal_baseline": equal}
        if with_baseline:
            row.update({"baseline_ms": statistics.median(t_base), "baseline_ms_min_max": [min(t_base), max(t_base)]})
        rows.append(row)
        print(json.dumps(row), flush=True)
        if with_baseline and not equal:
            sys.exit("threshold search and the baseline disagree")
        del got
        if with_baseline:
            del want
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
