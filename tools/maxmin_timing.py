"""Timing of MaxMin diversity picking (nvmolkit_b200.diversity) against what a user could build before it: a host-driven
loop of a one-row crossTanimotoSimilarity, torch.minimum and torch.argmax per pick. 2048-bit clustered fingerprints,
pools of 100k (fingerprints resident in shared memory) and 1M (streamed), pickSize 1,000 and 10,000, both modes.
CUDA-event times (one warm-up, median of 3, min-max printed); picks compared with the loop's. Also reported: the pair
distances each mode evaluated, as a fraction of the pairs the dense mode visits, and the popcount bound's skip rate; on
one sample, the CPU oracles and their thread count. Needs a GPU; there is no CPU fallback.

    python tools/maxmin_timing.py [--out results.json]
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
from nvmolkit_b200.diversity import MaxMinPicker  # noqa: E402
from nvmolkit_b200.similarity import crossTanimotoSimilarity  # noqa: E402
from oracle import pick as oracle_pick  # noqa: E402

REPEATS = 3


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


def torch_loop(d, pool, pick, first):
    picks = [first]
    mn = 1.0 - crossTanimotoSimilarity(d[first:first + 1], d[:pool]).torch()[0]
    taken = torch.zeros(pool, dtype=torch.bool, device=d.device)
    taken[first] = True
    while len(picks) < pick:
        w = int(torch.argmax(torch.where(taken, -1.0, mn)))
        picks.append(w)
        taken[w] = True
        mn = torch.minimum(mn, 1.0 - crossTanimotoSimilarity(d[w:w + 1], d[:pool]).torch()[0])
    return torch.tensor(picks, dtype=torch.int32)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--pools", default="100000,1000000")
    ap.add_argument("--picks", default="1000,10000")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("maxmin_timing.py needs a CUDA device")
    name = card()
    print(f"card: {name}", flush=True)
    pools = [int(x) for x in args.pools.split(",")]
    fps = synthetic.clustered_fingerprints((max(pools) + 24) // 25, 25, seed=15)
    d = torch.from_numpy(fps.view(np.int32)).cuda()
    picker = MaxMinPicker()
    rows = []
    for pool in pools:
        for pick in (int(x) for x in args.picks.split(",")):
            row = {"pool": pool, "pick": pick, "bits": 2048}
            ms_loop, want = timed(lambda: torch_loop(d, pool, pick, 0))
            row["torch_loop_ms"] = ms_loop
            row["torch_loop_us_per_pick"] = 1e3 * ms_loop / (pick - 1)
            for mode, label in ((0, "dense"), (1, "deferred")):
                with _lib.options(maxmin_mode=mode):
                    times = []
                    for it in range(1 + REPEATS):
                        ms, p = timed(lambda: picker.LazyBitVectorPick(d, pool, pick, [0]).torch())
                        if it:
                            times.append(ms)
                assert torch.equal(p.cpu(), want), f"{label} picks differ from the torch loop ({pool}, {pick})"
                ev, sk = _lib.get_option("maxmin_distances_last"), _lib.get_option("maxmin_popcount_skips_last")
                row[f"{label}_ms"] = statistics.median(times)
                row[f"{label}_ms_min_max"] = [min(times), max(times)]
                row[f"{label}_us_per_pick"] = 1e3 * statistics.median(times) / (pick - 1)
                row[f"{label}_distances"] = ev
                row[f"{label}_popcount_skip_rate"] = sk / max(1, ev + sk)
                row[f"{label}_resident"] = _lib.get_option("maxmin_resident_last")
            visited = row["dense_distances"] / max(1e-9, 1.0 - row["dense_popcount_skip_rate"])  # pairs dense visits
            row["dense_pairs_visited"] = visited
            row["deferred_fraction_evaluated"] = row["deferred_distances"] / visited
            row["dense_fraction_evaluated"] = row["dense_distances"] / visited
            row["picks_equal_torch_loop"] = True
            rows.append(row)
            print(json.dumps(row), flush=True)
    # the CPU oracles on one sample
    pool, pick = pools[0], 1000
    threads = oracle.set_threads(0)
    t0 = time.perf_counter()
    dense, _ = oracle_pick.maxmin_dense(fps, pool, pick, [0])
    t1 = time.perf_counter()
    lazy, _ = oracle_pick.maxmin_lazy(fps, pool, pick, [0])
    t2 = time.perf_counter()
    cpu = {"pool": pool, "pick": pick, "omp_threads": threads, "dense_oracle_s": t1 - t0, "lazy_oracle_serial_s": t2 - t1,
           "equal": bool((dense == lazy).all())}
    print(json.dumps(cpu), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "rows": rows, "cpu_oracle": cpu}, f, indent=1)


if __name__ == "__main__":
    main()
