"""CPU model of the superposition pilot of the Butina neighbour pass (launchSimilarityTensor, tanimoto_tc.cu).

The pilot runs the superposed pass over a prefix sample of the fingerprints at 4 x C for C = 4, 2, 1 and counts the
candidates the pre-filter lets through. This script computes the same counts without a GPU: the same sample, the same
float32 alpha and fixed-point pre-filter terms, the same symmetric-group mask, and the same cost model

    time(S, C) = pairs / (S C) * tPair + candidates * pairs / pilot pairs * S C * tVerify,

with tPair and tVerify read from the library's source. In popcount order the pass skips, per row group, the tile
columns past the group's popcount band (popcountBandKernel): `pairs` are then the pairs the band leaves, counted in the
sample at each column factor, and the whole pass is costed at the sample's share of them. It prints the candidates per
factor with the sample in the caller's order and in popcount order (what the pass uses), and the factor the pilot picks;
then, for the whole set in popcount order at 4 x 4, the pairs and CTA-pair units the band leaves and the largest rank's
share of the units at 2, 4 and 8 ranks.

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
TILE_M, TILE_N = 128, 256  # kTM, kTN
NEVER = 0xFFFF  # thresh entry of a popcount sum no pair reaches
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
    """The float32 alpha passParams hands the tile: (1 - cutoff) / (2 - cutoff) rounded down, one ulp further."""
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


def is_neighbour(c, a, b, cutoff):
    """The fp64 predicate, elementwise."""
    c, u = np.asarray(c, dtype=np.int64), np.asarray(a, dtype=np.int64) + np.asarray(b, dtype=np.int64) - c
    sim = np.where(c == 0, 0.0, c / np.where(u == 0, 1, u))
    return 1.0 - sim <= cutoff


def thresh_table(bits: int, cutoff: float) -> np.ndarray:
    """threshTableKernel: thresh[s] = the smallest c in [0, s / 2] with is_neighbour(c, s - c, 0), NEVER if none."""
    s = np.arange(2 * bits + 1, dtype=np.int64)
    lo, hi = np.zeros_like(s), s // 2
    ok = is_neighbour(hi, s, 0, cutoff)
    while (lo < hi).any():
        mid = (lo + hi) // 2
        p = is_neighbour(mid, s, 0, cutoff)
        open_ = lo < hi
        hi = np.where(open_ & p, mid, hi)
        lo = np.where(open_ & ~p, mid + 1, lo)
    return np.where(ok, lo, NEVER)


def band_table(thresh: np.ndarray) -> np.ndarray:
    """popcountBandKernel's suffix minimum of thresh: tmin[s] = min over s' >= s of thresh[s']."""
    return np.minimum.accumulate(thresh[::-1])[::-1]


def band_cuts(tmin: np.ndarray, a, b) -> np.ndarray:
    """bandCuts: no pair of a row group whose largest popcount is a with a column of popcount b can be a neighbour."""
    a, b = np.asarray(a, dtype=np.int64), np.asarray(b, dtype=np.int64)
    return tmin[a + b] > a


def band_ends(pop_x: np.ndarray, pop_y: np.ndarray, thresh: np.ndarray, col_span: int) -> np.ndarray:
    """popcountBandKernel: per row group of GROUP_ROWS rows of the ascending popcounts pop_x, the end tile column (of
    col_span fingerprints each) of the columns of pop_y (ascending) that can hold a neighbour."""
    tiles_n = -(-((len(pop_y) + col_span // TILE_N - 1) // (col_span // TILE_N)) // TILE_N)
    a_max = pop_x[np.minimum(len(pop_x), np.arange(1, -(-len(pop_x) // GROUP_ROWS) + 1) * GROUP_ROWS) - 1]
    # first column the band cuts (bandCuts is monotone along ascending b); searchsorted over a boolean per distinct b
    tmin = band_table(thresh)
    j_cut = np.array([np.searchsorted(band_cuts(tmin, a, pop_y), True) for a in a_max], dtype=np.int64)
    return np.minimum(tiles_n, -(-j_cut // col_span))


def band_pairs(n: int, ends: np.ndarray | None, col_span: int) -> float:
    """bandPairs (symmetric): pairs i < j with j below the end of i's row group (all pairs when ends is None)."""
    total = 0.0
    for g, r0 in enumerate(range(0, n, GROUP_ROWS)):
        r1 = min(n, r0 + GROUP_ROWS)
        e = n if ends is None else min(n, int(ends[g]) * col_span)
        i_end = min(r1, e - 1 if e > 0 else 0)
        if i_end <= r0:
            continue
        m = float(i_end - r0)
        total += m * float(e - 1) - (float(r0) + float(i_end) - 1.0) * m / 2.0
    return total


def group_units(n: int, S: int, C: int, ends: np.ndarray | None, pair: bool = True, run: int = 1) -> np.ndarray:
    """countUnits of a symmetric pass, per row group: CTA-pair units (pair) or tiles, run tile columns per unit."""
    tiles_m = -(-(-(-n // S)) // TILE_M)
    tiles_n = -(-(-(-n // C)) // TILE_N)
    group_tiles = GROUP_ROWS // (TILE_M * S)
    G = group_tiles // 2 if pair else group_tiles
    unit_rows = (tiles_m + 1) // 2 if pair else tiles_m
    out = []
    for g in range(-(-unit_rows // G)):
        g_rows = min(G, unit_rows - g * G)
        tn0 = (g * group_tiles * TILE_M * S + 1) // (TILE_N * C)
        lim = tiles_n if ends is None else min(tiles_n, int(ends[g]))
        out.append(g_rows * -(-(lim - tn0) // run) if tn0 < lim else 0)
    return np.array(out, dtype=np.int64)


def owner(groups: int, world: int) -> np.ndarray:
    """The rank that owns each row group: serpentine over cycles of `world` groups (UnitWalk)."""
    g = np.arange(groups)
    cycle, at = g // world, g % world
    return np.where(cycle % 2 == 1, world - 1 - at, at)


def candidates(fp: np.ndarray, cutoff: float, S: int, C: int, band: bool = False) -> int:
    """Candidates the symmetric superposed pass over `fp` (in the given order) lists at S x C; band: fp is in popcount
    order and the pass skips the tile columns past each row group's popcount band, as the pass in that order does."""
    pop = popcounts(fp)
    e = torch.from_numpy(np.unpackbits(np.ascontiguousarray(fp).view(np.uint8), axis=1).astype(np.float32))
    xs, xmin = _superposed(e, pop, S)
    ys, ymin = _superposed(e, pop, C)
    alpha = prefilter_alpha(cutoff)
    row_t, col_t = torch.from_numpy(prefilter_term(xmin, alpha)), torch.from_numpy(prefilter_term(ymin, alpha))
    cols = torch.arange(ys.shape[0])
    ends = band_ends(pop, pop, thresh_table(32 * fp.shape[1], cutoff), TILE_N * C) if band else None
    total = 0
    for r0 in range(0, xs.shape[0], 1024):
        acc = (xs[r0:r0 + 1024] @ ys.T).to(torch.int64)  # exact: sums <= 16 x 4096 < 2^24
        r = torch.arange(r0, r0 + acc.shape[0])[:, None]
        live = r * S + 1 < (cols[None, :] + 1) * C  # the group holds a pair i < j
        if ends is not None:
            live = live & (cols[None, :] // TILE_N < torch.from_numpy(ends)[(r * S) // GROUP_ROWS])
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
    thresh = thresh_table(32 * fp.shape[1], cutoff)
    best_t, best = None, (1, 1)
    got, cost, left = {}, {}, {}
    c = SUPER_COLS
    while c >= 1:
        got[c] = candidates(sample, cutoff, SUPER_ROWS, c, band=ordered)
        pop = popcounts(sample)
        left[c] = band_pairs(ns, band_ends(pop, pop, thresh, TILE_N * c), TILE_N * c) if ordered else pilot_pairs
        pass_pairs = total_pairs * (left[c] / pilot_pairs)
        if best_t is None:
            best_t = pass_pairs * t_pair
        t_pass = pass_pairs / (SUPER_ROWS * c) * t_pair
        t_ver = got[c] * pass_pairs / left[c] * SUPER_ROWS * c * t_verify if left[c] > 0 else 0.0
        cost[c] = t_pass + t_ver
        if t_pass + t_ver < best_t:
            best_t, best = t_pass + t_ver, (SUPER_ROWS, c)
        if t_ver <= t_pass:
            break
        c //= 2
    return {"sample": ns, "candidates": got, "banded_pairs": left, "cost_s": cost, "chosen": best, "chosen_cost_s": best_t}


def band_report(fp: np.ndarray, cutoff: float, S: int = 4, C: int = 4) -> dict:
    """The whole symmetric pass in popcount order at S x C (CTA pairs): pairs and units with and without the band, and
    the largest rank's share of the units at 2, 4 and 8 ranks."""
    n = len(fp)
    pop = np.sort(popcounts(fp))
    ends = band_ends(pop, pop, thresh_table(32 * fp.shape[1], cutoff), TILE_N * C)
    full, banded = group_units(n, S, C, None), group_units(n, S, C, ends)
    shares = {}
    for world in (2, 4, 8):
        per = np.bincount(owner(len(banded), world), weights=banded, minlength=world)
        shares[world] = float(per.max() / per.sum() * world)  # 1.0 = perfectly balanced
    return {"pairs": band_pairs(n, None, TILE_N * C), "banded_pairs": band_pairs(n, ends, TILE_N * C),
            "units": int(full.sum()), "banded_units": int(banded.sum()), "largest_rank_vs_mean": shares}


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
        if ordered:
            print(" " * 16 + "pairs the band leaves in the sample: " +
                  ", ".join(f"4 x {c}: {v:,.0f}" for c, v in r["banded_pairs"].items()))
    b = band_report(fp, args.cutoff)
    print(f"whole pass at 4 x 4: band leaves {b['banded_pairs']:.4g} of {b['pairs']:.4g} pairs "
          f"({100 * (1 - b['banded_pairs'] / b['pairs']):.2f} % skipped), {b['banded_units']:,} of {b['units']:,} CTA-pair units "
          f"({100 * (1 - b['banded_units'] / b['units']):.2f} % skipped); largest rank / mean: " +
          ", ".join(f"{w} ranks {v:.4f}" for w, v in b["largest_rank_vs_mean"].items()))


if __name__ == "__main__":
    main()
