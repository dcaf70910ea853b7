"""Timing of Butina on count fingerprints (clustering.fused_butina_counts_device) against what it replaces and what it
is built from: the full count threshold self search at t = 1 - cutoff (the same inner loop over all N^2 pairs, so the
ratio shows what the symmetric pass and the sum band save), the bit-vector fused_butina on the same molecules, and the
dense route butina(1 - crossTanimotoCountSimilarity(x)) at 32,768 rows, whose ids must equal the fused ones.

Data: Morgan count fingerprints (radius 2, 2048 bins) of the molecules tools/count_similarity_timing.py builds, and a
seeded clustered count set (centres from those fingerprints, each member a copy of one with --changes bins redrawn in
0 .. 3), so that the clusters are not all singletons. Sizes --sizes (100k and 1M); Tanimoto at cutoffs 0.3 and 0.2, Dice
at 0.2. CUDA-event times: a warm-up, then the median and min-max of --repeats calls; the full threshold search at the
largest size runs once per set, at the first case (it takes tens of seconds). Prints the pairs the pass compared
against n (n - 1) / 2, edges and clusters, and the card name, power limit and maximum SM clock. Needs a GPU; there is no CPU fallback.

    python tools/count_butina_timing.py [--sizes 100000 1000000] [--repeats 5] [--out results.json]
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from count_similarity_timing import card, molecules, timed  # noqa: E402

from nvmolkit_b200 import _lib  # noqa: E402
from nvmolkit_b200 import similarity as S  # noqa: E402
from nvmolkit_b200.clustering import butina, fused_butina_device, fused_butina_counts_device  # noqa: E402
from nvmolkit_b200.fingerprints import MorganFingerprintGenerator  # noqa: E402

CASES = [("tanimoto", 0.3), ("tanimoto", 0.2), ("dice", 0.2)]
WEIGHTS = {"tanimoto": (1.0, 1.0), "dice": (0.5, 0.5)}


def stats(fn, repeats: int) -> tuple[dict, object]:
    out = fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        t, out = timed(fn)
        times.append(t)
    return {"median_ms": statistics.median(times), "min_ms": min(times), "max_ms": max(times), "calls": repeats}, out


def clustered(fp: torch.Tensor, n: int, changes: int, seed: int = 11) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = fp[: max(1, n // 100)]
    x = centres[torch.randint(0, len(centres), (n,), device="cuda", generator=g)].clone()
    rows = torch.arange(n, device="cuda").repeat_interleave(changes)
    cols = torch.randint(0, fp.shape[1], (n * changes,), device="cuda", generator=g)
    x[rows, cols] = torch.randint(0, 4, (n * changes,), device="cuda", generator=g, dtype=x.dtype)
    return x


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--base", type=int, default=100_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--changes", type=int, default=3)
    ap.add_argument("--dense", type=int, default=32768, help="rows of the dense-route comparison (0: none)")
    ap.add_argument("--sets", nargs="+", default=["morgan", "clustered"], choices=["morgan", "clustered"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    gen = MorganFingerprintGenerator(2, 2048)
    graphs = molecules(max(args.sizes), args.base)
    counts, bits = gen.GetCountFingerprints(graphs).torch(), gen.GetFingerprints(graphs).torch()
    sets = {"morgan": counts, "clustered": clustered(counts, max(args.sizes), args.changes)}
    sets = {k: sets[k] for k in args.sets}
    res = {"card": card(), "rows": []}
    print("card:", res["card"], "| rows:", len(counts), flush=True)
    for name, full in sets.items():
        for n in args.sizes:
            x = full[:n].contiguous()
            allp = n * (n - 1) // 2
            for metric, cutoff in CASES:
                t, (ids, cen) = stats(lambda: fused_butina_counts_device(x, cutoff, metric=metric), args.repeats)
                pairs = _lib.get_option("count_neighbor_pairs_last")
                search = S.thresholdTanimotoCountSimilarity if metric == "tanimoto" else S.thresholdDiceCountSimilarity
                if n == max(args.sizes):  # once per set (warm from the smaller size): its time hardly depends on t
                    thr = None
                    if (metric, cutoff) == CASES[0]:
                        ms, _ = timed(lambda: search(x, threshold=1.0 - cutoff)[0].torch())
                        thr = {"median_ms": ms, "min_ms": ms, "max_ms": ms, "calls": 1}
                else:
                    thr, _ = stats(lambda: search(x, threshold=1.0 - cutoff)[0].torch(), args.repeats)
                row = {"set": name, "n": n, "metric": metric, "cutoff": cutoff, "fused_counts": t, "threshold_self": thr,
                       "pairs_compared": pairs, "all_pairs": allp, "pairs_fraction": pairs / allp,
                       "clusters": int(len(cen)), "edges": None}
                # the edge total of the same pass (the fused call does not return it)
                degrees = torch.zeros(n, dtype=torch.int32, device="cuda")
                ne = C.c_uint64(0)
                _lib.call("b200mol_count_neighbor_edges", x.data_ptr(), n, x.shape[1], *WEIGHTS[metric], float(cutoff),
                          degrees.data_ptr(), None, 0, C.byref(ne), None)
                row["edges"] = int(ne.value)
                if name == "morgan" and metric == "tanimoto":
                    b, _ = stats(lambda: fused_butina_device(bits[:n], cutoff), args.repeats)
                    row["fused_bits"] = b
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
            del x
    # the dense route where it still fits
    nd = args.dense
    for name, full in sets.items() if nd else ():
        x = full[:nd].contiguous()
        for metric, cutoff in CASES:
            cross = S.crossTanimotoCountSimilarity if metric == "tanimoto" else S.crossDiceCountSimilarity

            def dense():
                return butina(1.0 - cross(x).torch(), cutoff, return_centroids=True)[0].torch()

            td, ids_d = stats(dense, args.repeats)
            tf, (ids_f, _) = stats(lambda: fused_butina_counts_device(x, cutoff, metric=metric), args.repeats)
            row = {"set": name, "n": nd, "metric": metric, "cutoff": cutoff, "dense_route": td, "fused_counts": tf,
                   "ids_equal": bool(torch.equal(ids_d, ids_f))}
            assert row["ids_equal"], row
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
