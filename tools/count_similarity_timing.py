"""Timing of the count-fingerprint calls against their bit twins on the same molecules and against what a user had
before them: Morgan count fingerprints (radius 2, 2048 bins) of synthetic.random_molgraphs against GetFingerprints; the
count matrix, top-k and threshold search against the Tanimoto bit calls on the same molecules' bit fingerprints, and
against row blocks of torch.minimum(q[:, None], lib[None]).sum(-1) followed by the measure, torch.topk or >= t. Sizes:
1M molecules (--base distinct random molecules, repeated with a quarter of each copy's atom invariants replaced, so
that every copy has its own fingerprint at the base set's density: generating 1M molecules in Python takes minutes);
a 32k x 32k matrix; top-k of 16,384 queries against 1M, k = 100; threshold 0.7 for 16,384 x 1M and for the
1M self search. The torch route is timed on the first --torch-rows queries of each search and scaled to all of them
(it runs about 2 * bins operations per pair); its outputs are compared with the library's on those rows, and the count
matrix with it in full. CUDA-event times (warm-up, then median of --repeats, min-max printed; the torch route once). Prints the card name,
power limit and maximum SM clock. Needs a GPU; there is no CPU fallback.

    python tools/count_similarity_timing.py [--mols 1000000] [--matrix 32768] [--queries 16384] [--out results.json]
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

from nvmolkit_b200 import similarity as S  # noqa: E402
from nvmolkit_b200 import synthetic  # noqa: E402
from nvmolkit_b200.fingerprints import MorganFingerprintGenerator  # noqa: E402
from nvmolkit_b200.molgraph import MolGraphBatch  # noqa: E402


def molecules(n: int, base: int, seed: int = 7) -> MolGraphBatch:
    g = synthetic.random_molgraphs(min(n, base), seed=seed)
    reps = -(-n // len(g))
    na, nb = int(g.atom_starts[-1]), int(g.bond_starts[-1])
    rng = np.random.default_rng(seed)
    inv = np.tile(g.atom_inv, reps)
    relabel = rng.random(len(inv)) < 0.25
    relabel[:na] = False  # the first copy is the base set itself
    inv[relabel] = rng.integers(0, 1 << 32, size=int(relabel.sum()), dtype=np.uint64).astype(np.uint32)
    a_starts = np.concatenate([g.atom_starts[:-1] + r * na for r in range(reps)] + [[reps * na]])
    b_starts = np.concatenate([g.bond_starts[:-1] + r * nb for r in range(reps)] + [[reps * nb]])
    full = MolGraphBatch(a_starts, b_starts, inv, np.tile(g.bond_inv, reps), np.tile(g.bond_a, reps), np.tile(g.bond_b, reps))
    return full if len(full) == n else full.select(np.arange(n))


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


def bench(fns: dict, repeats: int) -> tuple[dict, dict]:
    """each function once to warm up, then `repeats` rounds alternating them; (ms stats, last outputs)"""
    outs = {k: f() for k, f in fns.items()}
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(repeats):
        for k, f in fns.items():
            t, outs[k] = timed(f)
            times[k].append(t)
    return {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in times.items()}, outs


def torch_tanimoto(q, lib, block_elems=1 << 31):
    """count Tanimoto in row blocks: c = sum of bin-wise minima, then c / (a + b - c) (0 when c = 0)"""
    a, b = q.sum(1, dtype=torch.int64), lib.sum(1, dtype=torch.int64)
    rows = max(1, block_elems // (lib.shape[0] * lib.shape[1]))
    out = torch.empty((q.shape[0], lib.shape[0]), dtype=torch.float64, device=q.device)
    for r0 in range(0, q.shape[0], rows):
        c = torch.minimum(q[r0:r0 + rows, None, :], lib[None]).sum(-1, dtype=torch.int64)
        d = (a[r0:r0 + rows, None] + b[None, :] - c).double()
        out[r0:r0 + rows] = torch.where(c == 0, 0.0, c.double() / d)
    return out


def torch_topk(q, lib, k, cols=1 << 16):
    """row blocks of the matrix, each column block merged into running (value desc, column asc) lists"""
    best_v = torch.full((q.shape[0], k), -1.0, dtype=torch.float64, device=q.device)
    best_i = torch.full((q.shape[0], k), 1 << 30, dtype=torch.int64, device=q.device)
    for c0 in range(0, lib.shape[0], cols):
        m = torch_tanimoto(q, lib[c0:c0 + cols])
        v = torch.cat([best_v, m], 1)
        i = torch.cat([best_i, torch.arange(c0, c0 + m.shape[1], device=q.device).expand(q.shape[0], -1)], 1)
        order = torch.argsort(i, 1)  # (stable sort by value after one by column: ties to the lowest column)
        v, i = v.gather(1, order), i.gather(1, order)
        order = torch.sort(v, dim=1, descending=True, stable=True).indices[:, :k]
        best_v, best_i = v.gather(1, order), i.gather(1, order)
    return best_v, best_i.int()


def torch_threshold(q, lib, t, cols=1 << 16):
    rows, cols_, vals = [], [], []
    for c0 in range(0, lib.shape[0], cols):
        m = torch_tanimoto(q, lib[c0:c0 + cols])
        r, c = torch.nonzero(m >= t, as_tuple=True)
        rows.append(r), cols_.append(c + c0), vals.append(m[r, c])
    r, c, v = torch.cat(rows), torch.cat(cols_), torch.cat(vals)
    order = torch.argsort(r * lib.shape[0] + c)
    return r[order], c[order].int(), v[order]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mols", type=int, default=1_000_000)
    ap.add_argument("--base", type=int, default=40000)
    ap.add_argument("--matrix", type=int, default=32768)
    ap.add_argument("--queries", type=int, default=16384)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--t", type=float, default=0.7)
    ap.add_argument("--torch-rows", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card()}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)

    graphs = molecules(args.mols, args.base)
    print(f"{len(graphs)} molecules", flush=True)
    gen = MorganFingerprintGenerator(2, 2048)
    res["fingerprints"], fps = bench({"counts": lambda: gen.GetCountFingerprints(graphs).torch(),
                                      "bits": lambda: gen.GetFingerprints(graphs).torch()}, args.repeats)
    counts, bits = fps["counts"], fps["bits"]
    nnz = (counts > 0).sum(1).double()
    res["nonzero_bins_per_row"] = {"mean": nnz.mean().item(), "max": nnz.max().item(), "max_count": counts.max().item()}
    print("fingerprints", json.dumps(res["fingerprints"]), json.dumps(res["nonzero_bins_per_row"]), flush=True)

    n = min(args.matrix, args.mols)
    cm, bm = counts[:n], bits[:n]
    res["matrix"], out = bench({"count": lambda: S.crossTanimotoCountSimilarity(cm).torch(),
                                "bits": lambda: S.crossTanimotoSimilarity(bm).torch()}, args.repeats)
    t_ms, want = timed(lambda: torch_tanimoto(cm.short(), cm.short(), 1 << 30))  # (once: it takes seconds)
    res["matrix"]["torch_ms"] = t_ms
    res["matrix"]["equal_to_torch"] = bool(torch.equal(out["count"], want))
    del out, want
    print("matrix", json.dumps(res["matrix"]), flush=True)

    nq, tr = min(args.queries, args.mols), args.torch_rows
    q, qb = counts[:nq], bits[:nq]
    res["topk"], out = bench({"count": lambda: [r.torch() for r in S.topKTanimotoCountSimilarity(q, counts, k=args.k)],
                              "bits": lambda: [r.torch() for r in S.topKTanimotoSimilarity(qb, bits, k=args.k)]},
                             args.repeats)
    t_ms, (tv, ti) = timed(lambda: torch_topk(q[:tr].short(), counts.short(), args.k))
    res["topk"]["torch_scaled_ms"] = t_ms * nq / tr
    res["topk"]["equal_to_torch_rows"] = bool(torch.equal(out["count"][0][:tr], tv) and torch.equal(out["count"][1][:tr], ti))
    print("topk", json.dumps(res["topk"]), flush=True)

    res["threshold"], out = bench({
        "count": lambda: [r.torch() for r in S.thresholdTanimotoCountSimilarity(q, counts, threshold=args.t)],
        "bits": lambda: [r.torch() for r in S.thresholdTanimotoSimilarity(qb, bits, threshold=args.t)]}, args.repeats)
    t_ms, (tr_r, tr_c, tr_v) = timed(lambda: torch_threshold(q[:tr].short(), counts.short(), args.t))
    indptr, idx, vals = out["count"]
    m = int(indptr[tr])
    res["threshold"]["torch_scaled_ms"] = t_ms * nq / tr
    res["threshold"]["nnz"] = int(indptr[-1])
    res["threshold"]["equal_to_torch_rows"] = bool(torch.equal(idx[:m], tr_c) and torch.equal(vals[:m], tr_v)
                                                   and torch.equal(torch.bincount(tr_r, minlength=tr).cumsum(0), indptr[1:tr + 1]))
    print("threshold", json.dumps(res["threshold"]), flush=True)

    res["threshold_self"], out = bench({
        "count": lambda: [r.torch() for r in S.thresholdTanimotoCountSimilarity(counts, threshold=args.t)],
        "bits": lambda: [r.torch() for r in S.thresholdTanimotoSimilarity(bits, threshold=args.t)]}, 1)
    t_ms, (tr_r, tr_c, tr_v) = timed(lambda: torch_threshold(counts[:tr].short(), counts.short(), args.t))
    indptr, idx, vals = out["count"]
    m = int(indptr[tr])
    res["threshold_self"]["torch_scaled_ms"] = t_ms * counts.shape[0] / tr
    res["threshold_self"]["nnz"] = int(indptr[-1])
    res["threshold_self"]["equal_to_torch_rows"] = bool(torch.equal(idx[:m], tr_c) and torch.equal(vals[:m], tr_v))
    print("threshold_self", json.dumps(res["threshold_self"]), flush=True)

    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
