"""Times the TFD matrix computation on the GPU (b200mol_tfd_matrices), one JSON line per shape:

  (a) 2,000 molecules x 300 conformers, (b) 20 molecules x 3,000 conformers: about 9e7 pairs and 360 MB of fp32 output
  each. Molecules have 30 atoms and one of two torsion mixes: "typical" (8 single torsions, symmetric ones of 2 and 3
  quartets, one 6-ring: 14 features per row, 22 comparisons per pair) and "symmetric" (6 single, symmetric ones of 3,
  9, 9 and 9 quartets, one 6-ring: 37 features, 259 comparisons per pair).

For each shape: the whole call by CUDA events (median of --reps after --warmup), then the feature pass and the pair pass
separately from a torch.profiler run of their own (median kernel durations), and the host build of the torsion tables
(tfd_torsions through the RDKit accessors; where RDKit is absent, through the stand-in of tests/fake_rdkit on synthetic
molecules of the same size, which times this package's Python, not RDKit's). Rates: pairs/s and output-write GB/s of
the pair pass (4 B per pair, against the H100 SXM data-sheet 3.35 TB/s), comparisons/s. The card's name, power limit
and SM clocks are read (not set) with nvidia-smi in the same run.

    python tools/tfd_timing.py [--reps 7] [--warmup 2] [--out FILE.jsonl]
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

from nvmolkit_b200 import synthetic, tfd  # noqa: E402

HBM_TBS = 3.35


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, check=True).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in line.split(",")]))
    except (OSError, subprocess.CalledProcessError):
        return {"name": torch.cuda.get_device_name(0)}


MIXES = {  # (single torsions, Q of each symmetric torsion); every molecule also has one 6-ring
    "typical": (8, (2, 3)),
    "symmetric": (6, (3, 9, 9, 9)),
}


def tables(n_mols: int, n_atoms: int, rng, mix: str) -> tfd.TFDTorsions:
    n_single, sym_q = MIXES[mix]
    per_mol = []
    for _ in range(n_mols):
        pick = lambda k: [int(x) for x in rng.choice(n_atoms, size=k, replace=False)]  # noqa: E731
        tors = [([tuple(pick(4))], tfd.SINGLE, float(rng.uniform(0.1, 1.0)), 180.0) for _ in range(n_single)]
        for q in sym_q:
            a, b = pick(2)
            tors.append(([(int(rng.integers(n_atoms)), a, b, int(rng.integers(n_atoms))) for _ in range(q)], tfd.SYMMETRIC,
                         float(rng.uniform(0.1, 1.0)), 180.0))
        ring = pick(6)
        tors.append(([tuple(ring[(i + k) % 6] for k in range(4)) for i in range(6)], tfd.RING, 1.5, tfd._ring_maxdev(6)))
        per_mol.append(tors)
    return tfd.TFDTorsions.from_lists(per_mol)


def host_build_seconds(n_mols: int) -> dict:
    """tfd_torsions over n_mols synthetic molecules of 10-14 heavy atoms with hydrogens (median of 3)."""
    try:
        from rdkit import Chem  # noqa: F401

        source = "rdkit"
    except ImportError:
        sys.path.insert(0, os.path.join(ROOT, "tests", "fake_rdkit"))
        source = "tests/fake_rdkit stand-in"
    if source == "rdkit":  # (the synthetic molecules are dicts for the stand-in; real RDKit needs SMILES input)
        return {"host_build_s": None, "host_build_source": "not measured: RDKit present, no SMILES set here"}
    from tfd_molecules import Mol

    _flat, raw = synthetic.random_embed_molecules(n_mols, 10, 14, seed=5)
    mols = [Mol(d) for d in raw]
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        tfd.tfd_torsions(mols)
        times.append(time.perf_counter() - t0)
    return {"host_build_s": statistics.median(times), "host_build_source": source, "host_build_mols": n_mols,
            "host_build_atoms_mean": float(np.mean([len(d["z"]) for d in raw]))}


def run(name: str, n_mols: int, n_conf: int, mix: str, reps: int, warmup: int) -> dict:
    rng = np.random.default_rng(7)
    n_atoms = 30
    tors = tables(n_mols, n_atoms, rng, mix)
    dev = torch.device("cuda", 0)
    xyz = torch.randn(n_mols * n_conf * n_atoms, 3, dtype=torch.float64, device=dev) * 1.5
    cas = torch.arange(0, n_mols * n_conf * n_atoms + 1, n_atoms, dtype=torch.int32, device=dev)
    counts = np.full(n_mols, n_conf, np.int64)
    call = lambda: tfd._run(tors, counts, None, cas, xyz, None)  # noqa: E731
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
    ref = out.clone()
    # kernels on their own, in a separate profiled run
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            out = call()
        torch.cuda.synchronize()
    per = {"tfdFeatureKernel": [], "tfdPairKernel": []}
    for e in prof.events():
        for k in per:
            if k in e.name and e.device_type.name == "CUDA":
                per[k].append(e.device_time_total / 1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total / 1000.0)
    feat_ms = statistics.median(per["tfdFeatureKernel"]) if per["tfdFeatureKernel"] else None
    pair_ms = statistics.median(per["tfdPairKernel"]) if per["tfdPairKernel"] else None
    pairs = n_mols * n_conf * (n_conf - 1) // 2
    q = np.diff(tors.quartet_start)
    comps_per_pair = float(np.where(tors.type == tfd.SYMMETRIC, q * q, 1).sum()) / n_mols
    features = int(np.where(tors.type == tfd.SYMMETRIC, q, 1).sum()) // n_mols
    res = {"shape": name, "torsions": mix, "features_per_row": features, "mols": n_mols, "confs": n_conf, "pairs": pairs,
           "out_MB": pairs * 4 / 1e6, "call_ms": call_ms, "feature_ms": feat_ms, "pair_ms": pair_ms,
           "pairs_per_s": pairs / (pair_ms / 1e3) if pair_ms else None,
           "write_GBps": pairs * 4 / (pair_ms / 1e3) / 1e9 if pair_ms else None,
           "write_frac_of_3.35TBps": pairs * 4 / (pair_ms / 1e3) / (HBM_TBS * 1e12) if pair_ms else None,
           "comparisons_per_pair": comps_per_pair,
           "comparisons_per_s": comps_per_pair * pairs / (pair_ms / 1e3) if pair_ms else None,
           "bitwise_repeat": bool(torch.equal(out, ref))}
    if mix == "typical":
        res.update(host_build_seconds(n_mols))
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tfd_timing.py needs a CUDA device; there is nothing to time on the CPU")
    info = card()
    lines = []
    for (name, m, c), mix in [(shape, mix) for mix in MIXES for shape in (("a", 2000, 300), ("b", 20, 3000))]:
        r = run(name, m, c, mix, args.reps, args.warmup)
        r["card"] = info
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
