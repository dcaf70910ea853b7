"""Timing of Leader diversity picking (nvmolkit_b200.diversity.LeaderPicker) against what a user could build before it:
a host-driven loop over windows of the pool with crossTanimotoSimilarity(window, picks) and a torch "any covered" test,
then a greedy pass over crossTanimotoSimilarity(survivors, survivors) inside the window. 2048-bit clustered
fingerprints (synthetic.clustered_fingerprints: 2,000 / 20,000 centres x 50 members): pools of 100k and 1M at thresholds 0.65 and
0.35, pickSize 0 (no limit) and 1,000; and the all-picks worst case, 100k random fingerprints at threshold 0.2.
CUDA-event times (one warm-up, median of 3, min-max printed); picks compared with the loop's and, where it runs in about
a minute, the CPU oracle's (its OpenMP thread count printed). Also reported: windows, pairs through the bulk count pass
and through the resolver, and pairs per second. Needs a GPU; there is no CPU fallback.

    python tools/leader_timing.py [--out results.json]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import oracle  # noqa: E402
from nvmolkit_b200 import _lib, synthetic  # noqa: E402
from nvmolkit_b200.diversity import LeaderPicker  # noqa: E402
from nvmolkit_b200.similarity import crossTanimotoSimilarity  # noqa: E402
from oracle import leader as oracle_leader  # noqa: E402

REPEATS = 3
WINDOW = 16384  # rows per window of the torch loop
PICK_CHUNK = 65536  # picks per similarity block of the torch loop (16384 x 65536 x 8 B = 8.6 GB)


def card() -> str:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()]


def timed(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop), out


def torch_loop(d, pool, threshold, pick):
    """Windows in index order: drop the items an earlier pick covers, then a greedy walk over the survivors' own matrix."""
    cap = pool if pick == 0 else pick
    picks = torch.empty(0, dtype=torch.int64, device=d.device)
    for lo in range(0, pool, WINDOW):
        if len(picks) >= cap:
            break
        hi = min(pool, lo + WINDOW)
        covered = torch.zeros(hi - lo, dtype=torch.bool, device=d.device)
        for p0 in range(0, len(picks), PICK_CHUNK):
            s = crossTanimotoSimilarity(d[lo:hi], d[picks[p0:p0 + PICK_CHUNK]]).torch()
            covered |= (1.0 - s <= threshold).any(dim=1)
        surv = torch.nonzero(~covered).flatten() + lo
        if len(surv) == 0:
            continue
        near = (1.0 - crossTanimotoSimilarity(d[surv]).torch() <= threshold).cpu().numpy()
        gone = np.zeros(len(surv), dtype=bool)
        new = []
        for k in range(len(surv)):
            if gone[k]:
                continue
            new.append(k)
            if len(picks) + len(new) >= cap:
                break
            gone |= near[k]
        picks = torch.cat([picks, surv[torch.tensor(new, device=d.device)]])
    return picks[:cap].to(torch.int32).cpu()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--oracle-max-s", type=float, default=90.0, help="skip the CPU oracle where it would take longer")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("leader_timing.py needs a CUDA device")
    name = card()
    threads = oracle.set_threads(0)
    print(f"card: {name}; CPU oracle on {threads} OpenMP threads", flush=True)
    clustered = {100_000: synthetic.clustered_fingerprints(2_000, 50, seed=40),
                 1_000_000: synthetic.clustered_fingerprints(20_000, 50, seed=41)}
    rng = np.random.default_rng(42)
    random100k = np.packbits(rng.random((100_000, 2048)) < 0.025, axis=1, bitorder="little").view(np.uint32)
    workloads = [(pool, thr, pick, "clustered") for pool in (100_000, 1_000_000) for thr in (0.65, 0.35) for pick in (0, 1000)]
    workloads.append((100_000, 0.2, 0, "random"))
    picker = LeaderPicker()
    rows = []
    oracle_rate = None  # seconds per (pick x pool item) of the oracle, from its first run
    for pool, thr, pick, kind in workloads:
        fps = clustered[pool] if kind == "clustered" else random100k
        d = torch.from_numpy(fps[:pool].view(np.int32)).cuda()
        row = {"pool": pool, "threshold": thr, "pick": pick, "data": kind, "bits": 2048}
        times = []
        for it in range(1 + REPEATS):
            ms, p = timed(lambda: picker.LazyBitVectorPick(d, pool, thr, pick).torch())
            if it:
                times.append(ms)
        got = p.cpu()
        bulk = _lib.get_option("leader_bulk_pairs_last")
        win, blk = _lib.get_option("leader_window_pairs_last"), _lib.get_option("leader_block_pairs_last")
        row.update({"picks": len(got), "gpu_ms": statistics.median(times), "gpu_ms_min_max": [min(times), max(times)],
                    "windows": _lib.get_option("leader_windows_last"), "bulk_pairs": bulk,
                    "resolver_pairs_window": win, "resolver_pairs_block": blk})
        row["pairs_per_s"] = (bulk + win + blk) / (row["gpu_ms"] * 1e-3)
        ms_loop, want = timed(lambda: torch_loop(d, pool, thr, pick))
        row["torch_loop_ms"] = ms_loop
        assert torch.equal(got, want), f"picks differ from the torch loop ({row})"
        row["picks_equal_torch_loop"] = True
        est = None if oracle_rate is None else oracle_rate * len(got) * pool
        if est is None or est <= args.oracle_max_s:
            t0 = time.perf_counter()
            cpu = oracle_leader.leader_pick(fps, pool, thr, pick)
            row["oracle_s"] = time.perf_counter() - t0
            oracle_rate = oracle_rate or row["oracle_s"] / max(1, len(cpu) * pool)
            assert (cpu == got.numpy()).all(), f"picks differ from the CPU oracle ({row})"
            row["picks_equal_oracle"] = True
        else:
            row["oracle_s"] = None  # (estimated over the limit: not run)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "omp_threads": threads, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
