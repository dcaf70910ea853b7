"""Times symmetry-aware alignment on the GPU (b200mol_best_align), one JSON line per workload:

  (i)   10,000 molecules x 100 probe conformers of A = 30 atoms against one reference conformer each, K = 2, 8 and 72
        mappings over all atoms: GetBestRMS (aligned and moved) and CalcRMS (in place), 1,000,000 jobs;
  (ii)  1,000 molecules x 10 probes of A = 60 atoms, K = 4,096 mappings, transforms only (GetBestAlignmentTransform);
  (iii) K = 1 beside b200mol_align on the same jobs as (i).

For each: the whole call by CUDA events (median of --reps after --warmup; host checks and plan, one upload, the
kernel), the kernel alone from a torch.profiler run of its own (median), and the algorithmic bytes -- every probe atom
read and, when moved, written (48 A B; 24 L B otherwise), each distinct reference's L atoms (24 L B), each mapping set
once (2 (K + 1) L B), 12 B of RMSD and index and 128 B per transform -- over kernel time, against the H100 SXM
data-sheet 3.35 TB/s. In the same run the expanded baseline is timed: b200mol_align over every (job, mapping) without
moving, torch argmin over the mappings, the winners copied to the host, and b200mol_align again on the winners (moving,
or writing transforms); with its largest RMSD difference from the fused call and whether it picked the same mappings.
The fp64 CPU oracle's jobs/s is taken on a sample. The card's name, power limit and SM clocks are read (not set) with
nvidia-smi in the same run.

    python tools/best_align_timing.py [--reps 5] [--warmup 1] [--out FILE.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from align_timing import HBM_TBS, card, events  # noqa: E402
from nvmolkit_b200 import molAlign as ma  # noqa: E402


def kernel_ms(call, reps: int, name: str) -> float | None:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    t = [e.device_time_total / 1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total / 1000.0
         for e in prof.events() if name in e.name and e.device_type.name == "CUDA"]
    return statistics.median(t) if t else None


def workload(rng, n_mol, per, A, K):
    """References [n_mol, A, 3], probes [n_mol * per, A, 3] (noisy rigid motions with their atoms shuffled), and one
    mapping set per molecule: P = all atoms, K reference lists of which the first is the true correspondence."""
    refs = rng.normal(size=(n_mol, A, 3)) * 2.0
    perm = np.argsort(rng.random((n_mol, A)), 1)
    probes = np.take_along_axis(refs, perm[:, :, None], 1)
    probes = np.repeat(probes, per, 0) + rng.normal(size=(n_mol * per, A, 3)) * 0.3 + rng.normal(size=(n_mol * per, 1, 3))
    base = np.argsort(rng.random((K, A)), 1).astype(np.int16)
    base[0] = np.arange(A)
    sets = [(np.arange(A), base[:, perm[m]], None) for m in range(n_mol)]  # per molecule: base composed with its perm
    return refs, probes, sets


class Expanded:
    """The pair lists of every (molecule, mapping), list m K + k, in the tables() form b200mol_align's wrapper reads."""

    def __init__(self, sets, K, A):
        self.start = np.arange(0, len(sets) * K * A + 1, A, dtype=np.int64)
        q = np.concatenate([s[1] for s in sets]).reshape(-1).astype(np.int32)
        self.pairs = np.ascontiguousarray(np.stack([np.tile(np.arange(A, dtype=np.int32), len(sets) * K), q], 1))

    def tables(self):
        return self.start, self.pairs, None


def run(args, rng, name, n_mol, per, A, K, mode, move, transform, baseline=True):
    refs, probes, sets = workload(rng, n_mol, per, A, K)
    n = n_mol * (per + 1)
    host = np.concatenate([refs.reshape(-1, 3), probes.reshape(-1, 3)])
    xyz0 = torch.from_numpy(host).cuda()
    cas = torch.arange(0, n * A + 1, A, dtype=torch.int32).cuda()
    atoms = np.full(n, A, np.int64)
    jp = np.arange(n_mol, n)
    jr = np.repeat(np.arange(n_mol), per)
    xyz = xyz0.clone()

    def call():
        if move:
            xyz.copy_(xyz0)
        return ma._run_best(jp, jr, jr, atoms, cas, xyz, sets, mode, False, 50, move, transform, None)

    call_ms = events(call, args.reps, args.warmup)
    from nvmolkit_b200.conformerRmsd import MapTables

    t0 = time.perf_counter()  # the part of the call that builds the mapping tables in Python
    for _ in range(args.reps):
        MapTables([(p, q) for p, q, _ in sets])
    tables_ms = (time.perf_counter() - t0) * 1e3 / args.reps
    if move:  # the copy that restores the inputs is not the call's
        call_ms -= events(lambda: xyz.copy_(xyz0), args.reps, args.warmup)
    k_ms = kernel_ms(call, args.reps, "bestAlignKernel")
    rmsd, best, T = call()
    torch.cuda.synchronize()
    jobs = len(jp)
    bytes_ = jobs * (48 * A if move else 24 * A) + n_mol * 24 * A + n_mol * 2 * (K + 1) * A + jobs * 12 + \
        (jobs * 128 if transform else 0)
    out = {"workload": name, "molecules": n_mol, "probes_per_molecule": per, "atoms": A, "K": K, "jobs": jobs,
           "mode": "in place" if mode else "aligned", "moved": move, "transforms": transform,
           "call_ms": round(call_ms, 3), "host_tables_ms": round(tables_ms, 3), "kernel_ms": None if k_ms is None else round(k_ms, 3),
           "algorithmic_bytes": bytes_,
           "hbm_fraction": None if not k_ms else round(bytes_ / (k_ms * 1e-3) / (HBM_TBS * 1e12), 4)}

    if baseline and mode == 0:  # the expanded baseline: every (job, mapping) through b200mol_align, argmin, the winners
        lists = Expanded(sets, K, A)
        ep, er = np.repeat(jp, K), np.repeat(jr, K)
        el = (er * K + np.tile(np.arange(K), jobs)).astype(np.int64)
        xb = xyz0.clone()

        def expanded():
            if move:
                xb.copy_(xyz0)
            r_all, _ = ma._run(ep, er, el, atoms, cas, xb, lists, False, 50, False, False, None)
            kk = r_all.view(jobs, K).argmin(1)
            kh = kk.cpu().numpy()
            r, t = ma._run(jp, jr, jr * K + kh, atoms, cas, xb, lists, False, 50, move, transform, None)
            return r, kk, t

        out["expanded_call_ms"] = round(events(expanded, args.reps, args.warmup), 3)
        if move:
            out["expanded_call_ms"] = round(out["expanded_call_ms"] - events(lambda: xb.copy_(xyz0), args.reps,
                                                                             args.warmup), 3)
        r2, k2, t2 = expanded()
        torch.cuda.synchronize()
        out["expanded_max_rmsd_diff"] = float((r2 - rmsd).abs().max())
        out["expanded_same_mapping"] = bool(torch.equal(k2.to(torch.int32), best))
        if move:
            out["expanded_max_coord_diff"] = float((xb - xyz).abs().max())
        out["speedup_vs_expanded"] = round(out["expanded_call_ms"] / call_ms, 2)
        if K == 1:  # b200mol_align alone on the same jobs
            xa = xyz0.clone()

            def align():
                if move:
                    xa.copy_(xyz0)
                return ma._run(jp, jr, jr, atoms, cas, xa, lists, False, 50, move, transform, None)

            out["align_call_ms"] = round(events(align, args.reps, args.warmup) - (
                events(lambda: xa.copy_(xyz0), args.reps, args.warmup) if move else 0.0), 3)
            ka = kernel_ms(align, args.reps, "alignKernel")
            out["align_kernel_ms"] = None if ka is None else round(ka, 3)
            r3, _ = align()
            out["align_bitwise_equal"] = bool(torch.equal(r3, rmsd)) and (not move or bool(torch.equal(xa, xyz)))

    from oracle import best_align as ob

    sample = rng.choice(jobs, 100, replace=False)
    t0 = time.perf_counter()
    for j in sample:
        ob.best_align(probes[j], refs[jr[j]], sets[jr[j]][0], sets[jr[j]][1], None, mode)
    out["oracle_jobs_per_s"] = round(len(sample) / (time.perf_counter() - t0), 1)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    info = card()
    lines = []
    # K = 1 first: it is the most common case, and its profiler run must not come after the largest ones
    lines.append(run(args, rng, "iii K = 1", 10000, 100, 30, 1, 0, True, False))
    for K in (2, 8, 72):
        lines.append(run(args, rng, "i GetBestRMS", 10000, 100, 30, K, 0, True, False))
        lines.append(run(args, rng, "i CalcRMS", 10000, 100, 30, K, 1, False, False, baseline=False))
    lines.append(run(args, rng, "ii GetBestAlignmentTransform", 1000, 10, 60, 4096, 0, False, True))
    for line in lines:
        line.update({"card": info})
        print(json.dumps(line), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
