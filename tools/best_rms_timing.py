"""Times symmetry-aware conformer RMSD matrices on the GPU (b200mol_conformer_rmsd_mapped, the engine of
conformerRmsd.GetAllConformerBestRMS), one JSON line per workload, against the best a user can do without it:

  (a) 2,000 molecules x 300 conformers, n = 30 atoms, K = 2, 8 and 48 mappings;
  (b) 20 molecules x 3,000 conformers, n = 30, K = 8;
  (c) 200 molecules x 100 conformers, n = 60, K = 1,296 (four methyls: every permutation of each one's hydrogens).

Every molecule of a workload shares one mapping table: the probe list is every atom in order and the mappings permute
groups of atoms (K = 2, 8: swaps of atom pairs; K = 48: 3! x 2^3; K = 1,296: (3!)^4).

The workaround, alternated with the mapped call in the same process: per mapping, one plain b200mol_conformer_rmsd over
the C originals (probe order) followed by their C permuted copies, the off-diagonal block kept and folded in with
torch.minimum. It evaluates every pair with probe and reference swapped (Jacobi on H H^T instead of H^T H), so the two
agree to 1e-10 A rather than bitwise; the largest difference is reported. Both are timed by CUDA events around the
whole call (median of --reps after --warmup), and rates are (pair, mapping) evaluations per second. The fp64 CPU
oracle's rate on a sample (one molecule, 40 conformers, the workload's mappings) is reported as the oracle's; RDKit is
not present. The card's name, power limit and SM clocks are read (not set) with nvidia-smi in the same run.

    python tools/best_rms_timing.py [--reps 5] [--warmup 1] [--out FILE.jsonl]
"""
from __future__ import annotations

import argparse
import itertools
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

from nvmolkit_b200 import _lib  # noqa: E402
from nvmolkit_b200 import conformerRmsd as cr  # noqa: E402


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, check=True).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in line.split(",")]))
    except (OSError, subprocess.CalledProcessError):
        return {"name": torch.cuda.get_device_name(0)}


def group_mappings(n: int, groups) -> np.ndarray:
    """Every combination of a permutation within each group of atoms (the rest fixed): [K, n] reference lists."""
    out = []
    for choice in itertools.product(*[list(itertools.permutations(g)) for g in groups]):
        q = list(range(n))
        for g, p in zip(groups, choice):
            for a, b in zip(g, p):
                q[a] = b
        out.append(q)
    return np.array(out, np.int64)


def mappings(n: int, K: int) -> np.ndarray:
    if K == 2:
        return group_mappings(n, [(0, 1)])
    if K == 8:
        return group_mappings(n, [(0, 1), (2, 3), (4, 5)])
    if K == 48:
        return group_mappings(n, [(0, 1, 2), (3, 4), (5, 6), (7, 8)])
    if K == 1296:
        return group_mappings(n, [(4 * i + 1, 4 * i + 2, 4 * i + 3) for i in range(4)])
    raise ValueError(K)


def timed(call, reps: int, warmup: int):
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    ms, out = [], None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = call()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return ms, out


def run(name: str, n_mols: int, n_conf: int, n_atoms: int, K: int, reps: int, warmup: int) -> dict:
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(11)
    base = torch.randn(n_mols, 1, n_atoms, 3, dtype=torch.float64, device=dev, generator=gen) * 1.5
    X = base + 0.5 * torch.randn(n_mols, n_conf, n_atoms, 3, dtype=torch.float64, device=dev, generator=gen)
    del base
    q = mappings(n_atoms, K)
    assert len(q) == K
    p = np.arange(n_atoms)
    counts = np.full(n_mols, n_conf, np.int64)
    atoms = np.full(n_mols, n_atoms, np.int64)
    xyz = X.reshape(-1, 3).contiguous()
    cas = torch.arange(0, n_mols * n_conf * n_atoms + 1, n_atoms, dtype=torch.int32, device=dev)
    tables = cr.MapTables([(p, q)] * n_mols)
    mapped = lambda: cr._run(counts, atoms, None, cas, xyz, False, None, tables)  # noqa: E731

    # the workaround: per mapping, originals then permuted copies through the plain call
    C = n_conf
    pairs = C * (C - 1) // 2
    big = 2 * C * (2 * C - 1) // 2
    ii, jj = np.tril_indices(C, -1)  # pair (I, J), I > J, in output order
    pick = torch.from_numpy((C + jj) * (C + jj - 1) // 2 + ii).to(dev)  # entry (copy J, original I) of the 2C matrix
    counts2 = np.full(n_mols, 2 * C, np.int64)
    mcs2 = np.arange(0, 2 * C * n_mols + 1, 2 * C).astype(np.int32)
    atoms32 = atoms.astype(np.int32)
    cas2 = torch.arange(0, n_mols * 2 * C * n_atoms + 1, n_atoms, dtype=torch.int32, device=dev)
    big_out = torch.empty(n_mols * big, dtype=torch.float64, device=dev)
    qd = torch.from_numpy(q).to(dev)

    def workaround():
        best = None
        for k in range(K):
            y = torch.cat([X, X[:, :, qd[k]]], dim=1).reshape(-1, 3).contiguous()
            _lib.call("b200mol_conformer_rmsd", n_mols, mcs2.ctypes.data, atoms32.ctypes.data, None, cas2.data_ptr(),
                      y.data_ptr(), 0, big_out.data_ptr(), None)
            v = big_out.view(n_mols, big)[:, pick]
            best = v if best is None else torch.minimum(best, v)
        return best

    m_ms, w_ms = [], []
    for _ in range(warmup):
        mapped(), workaround()
    torch.cuda.synchronize()
    for _ in range(reps):  # alternate the two in the same process
        a, out_m = timed(mapped, 1, 0)
        b, out_w = timed(workaround, 1, 0)
        m_ms.append(a[0])
        w_ms.append(b[0])
    got = torch.stack([r.torch() for r in out_m])
    again = torch.stack([r.torch() for r in mapped()])
    diff = float((got - out_w).abs().max())
    mm, wm = statistics.median(m_ms), statistics.median(w_ms)
    evals = n_mols * pairs * K
    res = {"workload": name, "mols": n_mols, "confs": n_conf, "atoms": n_atoms, "K": K, "pairs": n_mols * pairs,
           "mapped_ms": mm, "workaround_ms": wm, "mapped_ms_all": m_ms, "workaround_ms_all": w_ms,
           "speedup_vs_workaround": wm / mm,
           "mapped_evals_per_s": evals / (mm / 1e3), "workaround_evals_per_s": evals / (wm / 1e3),
           "chunks": _lib.get_option("rmsd_match_chunks_last"),
           "max_abs_diff_vs_workaround": diff, "agree_1e-10": diff <= 1e-10,
           "bitwise_repeat": bool(torch.equal(got, torch.stack([x for x in again])))}
    del X, xyz, cas, big_out, out_m, out_w, got, again
    torch.cuda.empty_cache()
    return res


def oracle_evals_per_s(n_atoms: int, K: int) -> float:
    from oracle import best_rms as oracle_best

    rng = np.random.default_rng(3)
    confs = [rng.normal(size=(n_atoms, 3)) * 1.5 for _ in range(40)]
    t0 = time.perf_counter()
    oracle_best.molecules([confs], [(np.arange(n_atoms), mappings(n_atoms, K))])
    return 40 * 39 / 2 * K / (time.perf_counter() - t0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("best_rms_timing.py needs a CUDA device; there is nothing to time on the CPU")
    info = card()
    lines = []
    for name, m, c, n, K in (("a", 2000, 300, 30, 2), ("a", 2000, 300, 30, 8), ("a", 2000, 300, 30, 48),
                             ("b", 20, 3000, 30, 8), ("c", 200, 100, 60, 1296)):
        r = run(name, m, c, n, K, args.reps, args.warmup)
        r["card"] = info
        r["oracle_evals_per_s"] = oracle_evals_per_s(n, K)
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    info_after = card()
    print(json.dumps({"card_after": info_after}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines + [json.dumps({"card_after": info_after})]) + "\n")


if __name__ == "__main__":
    main()
