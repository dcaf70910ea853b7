"""Times conformer alignment on the GPU (b200mol_align), one JSON line per workload:

  (i)   10,000 molecules x 100 conformers of A = 20, 50, 100 atoms: every conformer aligned onto its molecule's first
        over all atoms and moved (AlignMolConformers), 990,000 jobs;
  (ii)  the same over L = A / 2 atoms with weights;
  (iii) 100,000 probes of 30 atoms onto one reference through a 20-pair map, transforms only (GetAlignmentTransform).

For each: the whole call by CUDA events (median of --reps after --warmup; host plan, one upload, the kernel), the
kernel alone from a torch.profiler run of its own (median), and the algorithmic bytes -- read + write of every moved
probe atom (48 A B; 24 L B read when nothing moves), the listed reference atoms once per distinct reference (24 L B),
8 B of RMSD and 128 B per transform -- over kernel time, against the H100 SXM data-sheet 3.35 TB/s. In the same run a
torch batched Kabsch on the same data (weighted centring, bmm, torch.linalg.svd on (N, 3, 3), determinant fix, bmm)
is timed with its largest difference from the kernel, and the fp64 CPU oracle's jobs/s on a sample. The card's name,
power limit and SM clocks are read (not set) with nvidia-smi in the same run.

    python tools/align_timing.py [--reps 5] [--warmup 1] [--out FILE.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nvmolkit_b200 import molAlign as ma  # noqa: E402

HBM_TBS = 3.35


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, check=True).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in line.split(",")]))
    except (OSError, subprocess.CalledProcessError):
        return {"name": torch.cuda.get_device_name(0)}


def events(call, reps: int, warmup: int) -> float:
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        call()
        b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ev)


def kernel_ms(call, reps: int) -> float | None:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    t = [e.device_time_total / 1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total / 1000.0
         for e in prof.events() if "alignKernel" in e.name and e.device_type.name == "CUDA"]
    return statistics.median(t) if t else None


def torch_kabsch(P, Q, w, sel, move_atoms):
    """Batched weighted Kabsch of P[:, sel] onto Q[:, sel] ((N, A, 3) fp64): (RMSD [N], moved probes [N, A, 3])."""
    p, q = P[:, sel], Q[:, sel]
    W = w.sum()
    pb, qb = (w[None, :, None] * p).sum(1) / W, (w[None, :, None] * q).sum(1) / W
    pc, qc = p - pb[:, None], q - qb[:, None]
    H = torch.bmm((w[None, :, None] * pc).transpose(1, 2), qc)
    U, _, Vt = torch.linalg.svd(H)
    d = torch.sign(torch.linalg.det(torch.bmm(Vt.transpose(1, 2), U.transpose(1, 2))))
    D = torch.ones_like(pb)
    D[:, 2] = d
    R = torch.bmm(Vt.transpose(1, 2) * D[:, None, :], U.transpose(1, 2))
    res = torch.bmm(pc, R.transpose(1, 2)) - qc
    rmsd = torch.sqrt((w[None, :] * (res * res).sum(2)).sum(1) / len(sel))
    moved = torch.bmm(move_atoms - pb[:, None], R.transpose(1, 2)) + qb[:, None]
    return rmsd, moved


def conformers_workload(name, A, L, weighted, reps, warmup):
    n_mols, n_conf = 10000, 100
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(7)
    base = torch.randn(n_mols, 1, A, 3, dtype=torch.float64, device=dev, generator=gen) * 1.5
    xyz0 = (base + 0.5 * torch.randn(n_mols, n_conf, A, 3, dtype=torch.float64, device=dev, generator=gen)).contiguous()
    del base
    rng = np.random.default_rng(3)
    sel = np.sort(rng.choice(A, L, replace=False)) if L < A else np.arange(A)
    w = rng.uniform(0.5, 2.0, L) if weighted else None
    lists = ma.PairLists()
    for _ in range(n_mols):  # one list per molecule, as AlignMolConformers builds them
        lists.add(np.stack([sel, sel], 1), w)
    n = n_mols * n_conf
    atoms = np.full(n, A, np.int64)
    cas = torch.arange(0, n * A + 1, A, dtype=torch.int32, device=dev)
    conf = np.arange(n).reshape(n_mols, n_conf)
    jp, jr = conf[:, 1:].reshape(-1), np.repeat(conf[:, 0], n_conf - 1)
    jl = np.repeat(np.arange(n_mols), n_conf - 1)
    xyz = xyz0.clone().reshape(-1, 3)
    call = lambda: ma._run(jp, jr, jl, atoms, cas, xyz, lists, False, 50, True, False, None)  # noqa: E731
    rmsd, _ = call()
    torch.cuda.synchronize()
    first = rmsd.clone()
    moved_once = None
    x1 = xyz0.clone().reshape(-1, 3)
    r1, _ = ma._run(jp, jr, jl, atoms, cas, x1, lists, False, 50, True, False, None)
    torch.cuda.synchronize()
    moved_once = x1.reshape(n_mols, n_conf, A, 3)
    call_ms = events(call, reps, warmup)
    k_ms = kernel_ms(call, reps)
    jobs = len(jp)
    bytes_ = jobs * (48 * A + 8) + n_mols * 24 * L
    # torch baseline on the same data
    P = xyz0[:, 1:].reshape(-1, A, 3)
    Q = xyz0[:, :1].expand(-1, n_conf - 1, -1, -1).reshape(-1, A, 3)
    wt = torch.as_tensor(np.ones(L) if w is None else w, dtype=torch.float64, device=dev)
    st = torch.as_tensor(sel, device=dev)
    base_call = lambda: torch_kabsch(P, Q, wt, st, P)  # noqa: E731
    base_ms = events(base_call, reps, warmup)
    br, bm = base_call()
    diff_rmsd = float((br - r1).abs().max())
    diff_xyz = float((bm - moved_once[:, 1:].reshape(-1, A, 3)).abs().max())
    oracle_rate = oracle_jobs_per_s(xyz0, sel, w, A)
    res = {"workload": name, "mols": n_mols, "confs": n_conf, "atoms": A, "pairs": L, "weighted": weighted, "jobs": jobs,
           "call_ms": call_ms, "kernel_ms": k_ms, "algorithmic_GB": bytes_ / 1e9,
           "GBps": bytes_ / (k_ms / 1e3) / 1e9 if k_ms else None,
           "frac_of_3.35TBps": bytes_ / (k_ms / 1e3) / (HBM_TBS * 1e12) if k_ms else None,
           "torch_kabsch_ms": base_ms, "torch_max_diff_rmsd": diff_rmsd, "torch_max_diff_xyz": diff_xyz,
           "repeat_rmsd_bitwise": bool(torch.equal(first, r1)), "oracle_jobs_per_s": oracle_rate}
    del xyz0, xyz, x1, P, Q, bm, moved_once
    torch.cuda.empty_cache()
    return res


def oracle_jobs_per_s(xyz0, sel, w, A) -> float:
    from oracle import align as oracle_align

    sample = xyz0[:20].cpu().numpy()
    pairs = np.stack([sel, sel], 1)
    t0 = time.perf_counter()
    k = 0
    for m in range(len(sample)):
        for c in range(1, sample.shape[1]):
            oracle_align.align(sample[m, c], sample[m, 0], pairs, w)
            k += 1
    return k / (time.perf_counter() - t0)


def template_workload(reps, warmup):
    n, A, L = 100000, 30, 20
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(9)
    xyz0 = torch.randn(n + 1, A, 3, dtype=torch.float64, device=dev, generator=gen) * 1.5
    rng = np.random.default_rng(4)
    pairs = np.stack([rng.choice(A, L, replace=False), rng.choice(A, L, replace=False)], 1)
    lists = ma.PairLists()
    lists.add(pairs, None)
    atoms = np.full(n + 1, A, np.int64)
    cas = torch.arange(0, (n + 1) * A + 1, A, dtype=torch.int32, device=dev)
    jp, jr, jl = np.arange(1, n + 1), np.zeros(n, np.int64), np.zeros(n, np.int64)
    xyz = xyz0.reshape(-1, 3)
    call = lambda: ma._run(jp, jr, jl, atoms, cas, xyz, lists, False, 50, False, True, None)  # noqa: E731
    call_ms = events(call, reps, warmup)
    k_ms = kernel_ms(call, reps)
    rmsd, _ = call()
    bytes_ = n * (24 * L + 8 + 128) + 24 * L
    P = xyz0[1:][:, torch.as_tensor(pairs[:, 0], device=dev)]
    Q = xyz0[:1][:, torch.as_tensor(pairs[:, 1], device=dev)].expand(n, -1, -1)
    wt = torch.ones(L, dtype=torch.float64, device=dev)
    st = torch.arange(L, device=dev)
    base_call = lambda: torch_kabsch(P, Q, wt, st, P)  # noqa: E731
    base_ms = events(base_call, reps, warmup)
    br, _ = base_call()
    return {"workload": "iii", "jobs": n, "atoms": A, "pairs": L, "call_ms": call_ms, "kernel_ms": k_ms,
            "algorithmic_GB": bytes_ / 1e9, "GBps": bytes_ / (k_ms / 1e3) / 1e9 if k_ms else None,
            "frac_of_3.35TBps": bytes_ / (k_ms / 1e3) / (HBM_TBS * 1e12) if k_ms else None,
            "torch_kabsch_ms": base_ms, "torch_max_diff_rmsd": float((br - rmsd).abs().max())}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("align_timing.py needs a CUDA device; there is nothing to time on the CPU")
    info = card()
    lines = []
    runs = [lambda A=A: conformers_workload("i", A, A, False, args.reps, args.warmup) for A in (20, 50, 100)]
    runs += [lambda A=A: conformers_workload("ii", A, A // 2, True, args.reps, args.warmup) for A in (20, 50, 100)]
    runs += [lambda: template_workload(args.reps, args.warmup)]
    for run in runs:
        r = run()
        r["card"] = info
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    tail = json.dumps({"card_after": card()})
    print(tail)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines + [tail]) + "\n")


if __name__ == "__main__":
    main()
