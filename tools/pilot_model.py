"""CPU model of the superposition pilot of the Butina neighbour pass (launchSimilarityTensor, tanimoto_tc.cu).

The pilot runs the superposed pass over a prefix sample of the fingerprints at 4 x C for C = 4, 2, 1 and counts the
candidates the pre-filter lets through. This script computes the same counts without a GPU: the same sample, the same
float32 alpha and fixed-point pre-filter terms, the same symmetric-group mask, and the same cost model

    time(S, C) = pairs / (S C) * tPair + candidates * pairs / pilot pairs * S C * tVerify,

with tPair and tVerify read from the library's source. It prints the candidates per factor with the sample in the
caller's order and in popcount order (what the pass uses), and the factor the pilot picks.

    python tools/pilot_model.py                      # the bench data (1M points, 2048 bits, cutoff 0.3)
    python tools/pilot_model.py --n-centres 2000     # the bench generator at a smaller size
    python tools/pilot_model.py --seed 7             # the bench generator with another seed
    python tools/pilot_model.py --fingerprints fp.npy --cutoff 0.35
"""
import argparse
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GROUP_ROWS = 8192  # kGroupRows
SUPER_ROWS = 4  # the pilot's row factor (similarity_superpose)
SUPER_COLS = 4  # its widest column factor (similarity_superpose_cols)


def cost_constants() -> tuple[float, float]:
    """(tPair, tVerify) as launchSimilarityTensor defines them."""
    src = open(os.path.join(ROOT, "nvmolkit_b200", "csrc", "tanimoto_tc.cu")).read()
    m = re.search(r"constexpr double tPair = ([0-9.eE+-]+), tVerify = ([0-9.eE+-]+);", src)
    if not m:
        raise RuntimeError("tPair / tVerify not found in tanimoto_tc.cu")
    return float(m.group(1)), float(m.group(2))


def prefilter_alpha(cutoff: float) -> np.float32:
    """The float32 alpha launchTensorImpl hands the tile: (1 - cutoff) / (2 - cutoff) rounded down, one ulp further."""
    a = (1.0 - cutoff) / (2.0 - cutoff) if cutoff < 2.0 else 0.0
    af = np.float32(a)
    if float(af) > a:
        af = np.nextafter(af, np.float32(-1))
    return max(np.nextafter(af, np.float32(-1)), np.float32(0))


def prefilter_term(m, alpha: np.float32) -> np.ndarray:
    """tileMetaKernel's floor(__fmul_rd(256 alpha, m))."""
    exact = float(np.float32(256.0) * alpha) * np.asarray(m, dtype=np.float64)
    f = exact.astype(np.float32)
    f = np.where(f.astype(np.float64) > exact, np.nextafter(f, np.float32(-np.inf)), f)
    return np.floor(f).astype(np.int64)


def popcounts(fp: np.ndarray) -> np.ndarray:
    return np.unpackbits(np.ascontiguousarray(fp).view(np.uint8), axis=1).sum(1).astype(np.int64)


def popcount_order(fp: np.ndarray) -> np.ndarray:
    """The pass's order: ascending popcount, ties by index."""
    return np.argsort(popcounts(fp), kind="stable")


def _superposed(e: torch.Tensor, pop: np.ndarray, k: int):
    """Sums of k consecutive rows of the 0/1 expansion and each sum's smallest member popcount."""
    n = e.shape[0]
    rows = (n + k - 1) // k
    pad = rows * k - n
    sums = torch.cat([e, e.new_zeros(pad, e.shape[1])]).view(rows, k, -1).sum(1)
    mins = np.concatenate([pop, np.full(pad, 1 << 30)]).reshape(rows, k).min(1)
    return sums, mins


def candidates(fp: np.ndarray, cutoff: float, S: int, C: int) -> int:
    """Candidates the symmetric superposed pass over `fp` (in the given order) lists at S x C."""
    pop = popcounts(fp)
    e = torch.from_numpy(np.unpackbits(np.ascontiguousarray(fp).view(np.uint8), axis=1).astype(np.float32))
    xs, xmin = _superposed(e, pop, S)
    ys, ymin = _superposed(e, pop, C)
    alpha = prefilter_alpha(cutoff)
    row_t, col_t = torch.from_numpy(prefilter_term(xmin, alpha)), torch.from_numpy(prefilter_term(ymin, alpha))
    cols = torch.arange(ys.shape[0])
    total = 0
    for r0 in range(0, xs.shape[0], 1024):
        acc = (xs[r0:r0 + 1024] @ ys.T).to(torch.int64)  # exact: sums <= 16 x 4096 < 2^24
        r = torch.arange(r0, r0 + acc.shape[0])[:, None]
        live = r * S + 1 < (cols[None, :] + 1) * C  # the group holds a pair i < j
        passed = 256 * acc - col_t[None, :] >= row_t[r0:r0 + acc.shape[0], None]
        total += int((live & passed).sum())
    return total


def pilot(fp: np.ndarray, cutoff: float, ordered: bool = True) -> dict:
    """What the pilot of a symmetric pass over all of `fp` measures and picks (None if it does not run)."""
    n = len(fp)
    if n < 8 * GROUP_ROWS:
        return None
    ns = min(32768, max(2 * GROUP_ROWS, n // 8))
    sample = fp[:ns]
    if ordered:
        sample = sample[popcount_order(sample)]
    t_pair, t_verify = cost_constants()
    total_pairs, pilot_pairs = n * (n - 1) / 2.0, ns * (ns - 1) / 2.0
    best_t, best = total_pairs * t_pair, (1, 1)
    got, cost = {}, {}
    c = SUPER_COLS
    while c >= 1:
        got[c] = candidates(sample, cutoff, SUPER_ROWS, c)
        t_pass = total_pairs / (SUPER_ROWS * c) * t_pair
        t_ver = got[c] * total_pairs / pilot_pairs * SUPER_ROWS * c * t_verify
        cost[c] = t_pass + t_ver
        if t_pass + t_ver < best_t:
            best_t, best = t_pass + t_ver, (SUPER_ROWS, c)
        if t_ver <= t_pass:
            break
        c //= 2
    return {"sample": ns, "candidates": got, "cost_s": cost, "chosen": best, "chosen_cost_s": best_t}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--fingerprints", help=".npy of uint32 [n][words] (default: the bench generator)")
    ap.add_argument("--n-centres", type=int, default=20000, help="bench generator: centres x 50 members")
    ap.add_argument("--seed", type=int, default=None, help="bench generator seed (default: the bench's own)")
    ap.add_argument("--cutoff", type=float, default=0.3)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    if args.fingerprints:
        fp = np.load(args.fingerprints)
    else:
        from nvmolkit_b200 import synthetic

        seed = synthetic.SEED if args.seed is None else args.seed
        fp = synthetic.clustered_fingerprints(args.n_centres, 50, seed=seed)
    print(f"{len(fp)} fingerprints of {32 * fp.shape[1]} bits, cutoff {args.cutoff}; tPair, tVerify = {cost_constants()}")
    for ordered in (False, True):
        r = pilot(fp, args.cutoff, ordered)
        if r is None:
            print("fewer than 65,536 fingerprints: the pilot does not run")
            return
        name = "popcount order" if ordered else "caller's order"
        per = ", ".join(f"4 x {c}: {r['candidates'][c]:,} candidates, {r['cost_s'][c]:.3f} s" for c in r["candidates"])
        print(f"{name:>15} (sample {r['sample']:,}): {per}; picks {r['chosen'][0]} x {r['chosen'][1]} "
              f"({r['chosen_cost_s']:.3f} s)")


if __name__ == "__main__":
    main()
