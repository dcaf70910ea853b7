"""Times the conformer RMSD matrices on the GPU (b200mol_conformer_rmsd), one JSON line per (shape, atoms, mode):

  (a) 2,000 molecules x 300 conformers, (b) 20 molecules x 3,000 conformers: about 9e7 pairs and 720 MB of fp64 output
  each, at n = 16, 30, 64 and 100 atoms, with and without the superposition (prealigned).

For each: the whole call by CUDA events (median of --reps after --warmup), then the operand pass and the pair pass
separately from a torch.profiler run of their own (median kernel durations). Rates: pairs/s of the pair pass, the
covariance product's fp64 rate (18 n FLOP per pair) against the H100 SXM data-sheet 67 TFLOP/s FP64 tensor figure, and
the output-write GB/s against the data-sheet 3.35 TB/s. The n sweep separates the epilogue's fixed cost per pair from
the product. The fp64 CPU oracle's pairs/s is measured on a 300-conformer sample. The card's name, power limit and SM
clocks are read (not set) with nvidia-smi in the same run.

    python tools/conformer_rmsd_timing.py [--reps 7] [--warmup 2] [--out FILE.jsonl]
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

from nvmolkit_b200 import conformerRmsd as cr  # noqa: E402

HBM_TBS = 3.35
FP64_TC_TFLOPS = 67.0


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, check=True).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in line.split(",")]))
    except (OSError, subprocess.CalledProcessError):
        return {"name": torch.cuda.get_device_name(0)}


def oracle_pairs_per_s(n_atoms: int, prealigned: bool) -> float:
    from oracle import rmsd as oracle_rmsd

    rng = np.random.default_rng(3)
    confs = [rng.normal(size=(n_atoms, 3)) * 1.5 for _ in range(300)]
    t0 = time.perf_counter()
    oracle_rmsd.molecules([confs], prealigned)
    return 300 * 299 / 2 / (time.perf_counter() - t0)


def run(name: str, n_mols: int, n_conf: int, n_atoms: int, prealigned: bool, reps: int, warmup: int) -> dict:
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(7)
    base = torch.randn(n_mols, 1, n_atoms, 3, dtype=torch.float64, device=dev, generator=gen) * 1.5
    xyz = (base + 0.5 * torch.randn(n_mols, n_conf, n_atoms, 3, dtype=torch.float64, device=dev, generator=gen))
    xyz = xyz.reshape(-1, 3).contiguous()
    del base
    cas = torch.arange(0, n_mols * n_conf * n_atoms + 1, n_atoms, dtype=torch.int32, device=dev)
    counts = np.full(n_mols, n_conf, np.int64)
    atoms = np.full(n_mols, n_atoms, np.int64)
    call = lambda: cr._run(counts, atoms, None, cas, xyz, prealigned, None)  # noqa: E731
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        out = call()
        b.record()
    torch.cuda.synchronize()
    call_ms = statistics.median(a.elapsed_time(b) for a, b in ev)
    ref = out[0].torch().clone()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            out = call()
        torch.cuda.synchronize()
    per = {"rmsdOperandKernel": [], "rmsdPairKernel": []}
    for e in prof.events():
        for k in per:
            if k in e.name and e.device_type.name == "CUDA":
                per[k].append(e.device_time_total / 1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total / 1000.0)
    op_ms = statistics.median(per["rmsdOperandKernel"]) if per["rmsdOperandKernel"] else None
    pair_ms = statistics.median(per["rmsdPairKernel"]) if per["rmsdPairKernel"] else None
    pairs = n_mols * n_conf * (n_conf - 1) // 2
    sec = pair_ms / 1e3 if pair_ms else None
    res = {"shape": name, "mols": n_mols, "confs": n_conf, "atoms": n_atoms, "prealigned": prealigned, "pairs": pairs,
           "out_MB": pairs * 8 / 1e6, "call_ms": call_ms, "operand_ms": op_ms, "pair_ms": pair_ms,
           "pairs_per_s": pairs / sec if sec else None,
           "product_TFLOPs": 18.0 * n_atoms * pairs / sec / 1e12 if sec else None,
           "product_frac_of_67TFLOPs": 18.0 * n_atoms * pairs / sec / (FP64_TC_TFLOPS * 1e12) if sec else None,
           "write_GBps": pairs * 8 / sec / 1e9 if sec else None,
           "write_frac_of_3.35TBps": pairs * 8 / sec / (HBM_TBS * 1e12) if sec else None,
           "bitwise_repeat": bool(torch.equal(out[0].torch(), ref))}
    del out, xyz, cas
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("conformer_rmsd_timing.py needs a CUDA device; there is nothing to time on the CPU")
    info = card()
    lines = []
    for prealigned in (False, True):
        for n in (16, 30, 64, 100):
            for name, m, c in (("a", 2000, 300), ("b", 20, 3000)):
                r = run(name, m, c, n, prealigned, args.reps, args.warmup)
                r["card"] = info
                if name == "a":
                    r["oracle_pairs_per_s"] = oracle_pairs_per_s(n, prealigned)
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
