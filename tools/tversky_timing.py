"""Timing of the Dice and Tversky calls against the matching Tanimoto / cosine call and against what a user had before
them: the Tanimoto matrix, row-blocked, then c recovered from it and the popcounts, then the measure in torch (then
torch.topk, or nonzero for a threshold). 2048-bit clustered fingerprints (seeded as tools/topk_timing.py); matrices
32k x 32k; top-k and threshold search with 16,384 queries against a library of 1M, k = 100, t = 0.8. CUDA-event times
(3 warm-ups, median of 5, min-max printed), the calls of a row alternating in one process, results compared. Needs a GPU;
there is no CPU fallback.

    python tools/tversky_timing.py [--library 1000000] [--out results.json]
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

from nvmolkit_b200 import synthetic  # noqa: E402
from nvmolkit_b200 import similarity as S  # noqa: E402

WARMUP, REPEATS = 3, 5
BLOCK_BYTES = 2 << 30  # the baseline's matrix block
TV = (0.9, 0.1)


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


def popcounts(fp):
    return torch.from_numpy(np.bitwise_count(fp.cpu().numpy().view(np.uint32)).sum(1).astype(np.float64)).cuda()


def measure_from_tanimoto(t, pa, pb, w):
    """What a user could do before: c = round(T (a + b) / (1 + T)) from the Tanimoto matrix, then the measure."""
    s = pa[:, None] + pb[None, :]
    c = torch.round(t * s / (1.0 + t))
    d = (w[0] * (pa[:, None] - c) + w[1] * (pb[None, :] - c)) + c
    return torch.where(c == 0, torch.zeros_like(t), c / d)


def blocks(q, lib, pa, pb, w, each):
    rows = max(1, BLOCK_BYTES // (8 * lib.shape[0]))
    return [each(r0, measure_from_tanimoto(S.crossTanimotoSimilarity(q[r0:r0 + rows], lib).torch(), pa[r0:r0 + rows], pb, w))
            for r0 in range(0, q.shape[0], rows)]


def run(label, calls, extra=None):
    times = {k: [] for k in calls}
    outs = {}
    for it in range(WARMUP + REPEATS):
        for k, fn in calls.items():
            ms, outs[k] = timed(fn)
            if it >= WARMUP:
                times[k].append(ms)
    row = {"case": label}
    for k, t in times.items():
        row[f"{k}_ms"] = statistics.median(t)
        row[f"{k}_ms_min_max"] = [min(t), max(t)]
    if extra:
        row.update(extra(outs))
    print(json.dumps(row), flush=True)
    return row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--library", type=int, default=1_000_000)
    ap.add_argument("--matrix", type=int, default=32768)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tversky_timing.py needs a CUDA device")
    name = card()
    print(f"card: {name}")
    n_q = 16384
    fps = synthetic.clustered_fingerprints((args.library + n_q + 24) // 25, 25, seed=7)
    lib = torch.from_numpy(fps[:args.library].view(np.int32)).cuda()
    queries = torch.from_numpy(fps[args.library:args.library + n_q].view(np.int32)).cuda()
    pl, pq = popcounts(lib), popcounts(queries)
    rows = []

    # ---- matrices
    m = lib[:args.matrix]
    pm = pl[:args.matrix]
    rows.append(run(f"cross {args.matrix} x {args.matrix}", {
        "dice": lambda: S.crossDiceSimilarity(m).torch(),
        "tversky_0.9_0.1": lambda: S.crossTverskySimilarity(m, alpha=TV[0], beta=TV[1]).torch(),
        "tanimoto": lambda: S.crossTanimotoSimilarity(m).torch(),
        "baseline_tversky": lambda: torch.cat(blocks(m, m, pm, pm, TV, lambda r0, v: v)),
    }, lambda o: {"baseline_equal": bool(torch.equal(o["baseline_tversky"], o["tversky_0.9_0.1"]))}))
    del m
    torch.cuda.empty_cache()

    # ---- top-k
    k = 100

    def base_topk(w):
        parts = blocks(queries, lib, pq, pl, w, lambda r0, v: torch.topk(v, k, dim=1))
        return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])

    rows.append(run(f"topk {n_q} x {args.library} k={k} dice", {
        "dice": lambda: tuple(r.torch() for r in S.topKDiceSimilarity(queries, lib, k=k)),
        "tanimoto": lambda: tuple(r.torch() for r in S.topKTanimotoSimilarity(queries, lib, k=k)),
        "baseline_dice": lambda: base_topk((0.5, 0.5)),
    }, lambda o: {"baseline_values_equal": bool(torch.equal(o["baseline_dice"][0], o["dice"][0])),
                  "indices_equal_tanimoto": bool(torch.equal(o["dice"][1], o["tanimoto"][1]))}))
    rows.append(run(f"topk {n_q} x {args.library} k={k} tversky 0.9 0.1", {
        "tversky_0.9_0.1": lambda: tuple(r.torch() for r in S.topKTverskySimilarity(queries, lib, k=k, alpha=TV[0],
                                                                                      beta=TV[1])),
        "cosine": lambda: tuple(r.torch() for r in S.topKCosineSimilarity(queries, lib, k=k)),
        "baseline_tversky": lambda: base_topk(TV),
    }, lambda o: {"baseline_values_equal": bool(torch.equal(o["baseline_tversky"][0], o["tversky_0.9_0.1"][0]))}))

    # ---- threshold
    t = 0.8

    def base_threshold(w):
        parts = blocks(queries, lib, pq, pl, w, lambda r0, v: (v >= t).nonzero())
        return sum(int(p.shape[0]) for p in parts)

    rows.append(run(f"threshold {n_q} x {args.library} t={t}", {
        "dice": lambda: [r.torch() for r in S.thresholdDiceSimilarity(queries, lib, threshold=t)],
        "tanimoto_2/3": lambda: [r.torch() for r in S.thresholdTanimotoSimilarity(queries, lib, threshold=t / (2 - t))],
        "tversky_0.9_0.1": lambda: [r.torch() for r in S.thresholdTverskySimilarity(queries, lib, alpha=TV[0], beta=TV[1],
                                                                                     threshold=t)],
        "baseline_dice": lambda: base_threshold((0.5, 0.5)),
        "baseline_tversky": lambda: base_threshold(TV),
    }, lambda o: {"nnz_dice": int(o["dice"][1].shape[0]), "nnz_tanimoto_2/3": int(o["tanimoto_2/3"][1].shape[0]),
                  "nnz_tversky": int(o["tversky_0.9_0.1"][1].shape[0]),
                  "baseline_nnz_equal": o["baseline_dice"] == int(o["dice"][1].shape[0]) and
                  o["baseline_tversky"] == int(o["tversky_0.9_0.1"][1].shape[0])}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
