"""Pairs on the neighbour boundary, through every path of the thresholded pair pass.

A pair (A, B) with c = |A & B| is a neighbour iff the fp64 predicate 1 - c / (|A| + |B| - c) <= cutoff holds (the
similarity is 0 when c = 0). The count passes test it as c >= thresh[|A| + |B|], the smallest passing c. Before that
test the tensor-core tile applies a fixed-point pre-filter to each accumulator acc (the pair's c when unsuperposed, the
sum of a group's S x C counts when superposed):

    256 acc - T(|B|) >= T(|A|),   T(m) = floor(RD(256 alpha m)),

with alpha = (1 - cutoff) / (2 - cutoff) rounded down to float32 and then one ulp further (passParams), RD a
float32 product rounded down, and |A|, |B| the smallest popcounts of the group (tileMetaKernel). It must never reject a
neighbour: the margin 256 thresh[|A| + |B|] - T(|A|) - T(|B|) must be >= 0 for every pair that can exist.

The CPU test below checks that margin for every feasible pair of popcounts. The GPU tests build the pairs with the
smallest margin, at c = thresh (a neighbour) and at c = thresh - 1 (not one), and run them through the SIMT tile and
every tensor-core variant, unsuperposed and superposed in groups whose accumulator is exactly the pair's c. Expected
results come from a float64 matmul of the 0/1 expansions and the fp64 predicate, with the C oracle as a cross-check.
"""

import ctypes as C
import functools

import numpy as np
import pytest
import torch

import oracle
from nvmolkit_b200 import synthetic as S

CUTOFFS = [0.0, 0.1, 0.2, 0.3, 0.30000000000000004, 0.29999999999999993, 1 / 3, 0.35, 0.5, 0.65, 0.7, 0.9, 0.999, 1.0]
NEVER = 0xFFFF  # thresh entry of a popcount sum no pair reaches
FILL = 2  # superposed blocks: fillers have this many more bits than the boundary pair member they sit next to
SEVEN_TENTHS = [(7, 10, 7), (8, 9, 7), (10, 7, 7), (14, 20, 14), (70, 100, 70)]  # (|A|, |B|, c) with sim exactly 7/10


# ------------------------------------------------------------------ CPU model of the predicate and the pre-filter
def prefilter_alpha(cutoff: float) -> np.float32:
    """The float32 alpha passParams hands the tile: (1 - cutoff) / (2 - cutoff) in fp64, rounded down to float32,
    one ulp further down, clamped at 0."""
    a = (1.0 - cutoff) / (2.0 - cutoff) if cutoff < 2.0 else 0.0
    af = np.float32(a)
    if float(af) > a:
        af = np.nextafter(af, np.float32(-1))
    af = np.nextafter(af, np.float32(-1))
    return max(af, np.float32(0))


def prefilter_term(m, alpha: np.float32) -> np.ndarray:
    """tileMetaKernel's floor(__fmul_rd(256 alpha, m)) for popcounts m."""
    exact = float(np.float32(256.0) * alpha) * np.asarray(m, dtype=np.float64)  # exact: 24-bit x 14-bit significands
    f = exact.astype(np.float32)
    f = np.where(f.astype(np.float64) > exact, np.nextafter(f, np.float32(-np.inf)), f)  # round toward -inf
    return np.floor(f).astype(np.int64)


def is_neighbour(c, a, b, cutoff):
    """The fp64 predicate, elementwise."""
    c, u = np.asarray(c, dtype=np.int64), np.asarray(a, dtype=np.int64) + np.asarray(b, dtype=np.int64) - c
    sim = np.where(c == 0, 0.0, c / np.where(u == 0, 1, u))
    return 1.0 - sim <= cutoff


@functools.lru_cache(maxsize=None)
def thresh_table(bits: int, cutoff: float) -> np.ndarray:
    """thresh[s] = the smallest c in [0, s / 2] with is_neighbour(c, s - c, 0) (sum of popcounts s), NEVER if none.
    The predicate is monotone in c, so a bisection over all s at once finds it."""
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


def block_bits(a, b, c):
    """Bits a superposed block of 16 fingerprints needs: A | B, three row fillers of |A| + FILL bits and three column
    fillers of |B| + FILL bits, all disjoint."""
    return (a + b - c) + 3 * (a + FILL) + 3 * (b + FILL)


@functools.lru_cache(maxsize=None)
def boundary(bits: int, cutoff: float):
    """Pre-filter margins (1/256 units) at c = thresh[a + b] over every feasible pair of popcounts a <= b.

    Returns (smallest margin, its triples (a, b, c), smallest margin of the triples whose superposed block fits the
    width, those triples). Of tied triples, the four with the smallest a + b and the two with the largest are kept."""
    t = thresh_table(bits, cutoff)
    T = prefilter_term(np.arange(bits + 1), prefilter_alpha(cutoff))
    best = [[np.iinfo(np.int64).max, []], [np.iinfo(np.int64).max, []]]  # all | fitting the block

    def keep(trip):
        trip = sorted(set(trip), key=lambda x: (x[0] + x[1], x))
        return trip[:4] + [x for x in trip[-2:] if x not in trip[:4]]

    b = np.arange(bits + 1, dtype=np.int64)[None, :]
    for a0 in range(0, bits + 1, 256):
        a = np.arange(a0, min(a0 + 256, bits + 1), dtype=np.int64)[:, None]
        c = t[a + b]
        feasible = (b >= a) & (c != NEVER) & (c <= a) & (a + b - c <= bits)
        margin = 256 * c - T[a] - T[b]
        for k, mask in enumerate((feasible, feasible & (block_bits(a, b, c) <= bits))):
            if not mask.any():
                continue
            m = margin[mask].min()
            if m > best[k][0]:
                continue
            ia, ib = np.nonzero(mask & (margin == m))
            s = ia + a0 + ib
            order = np.argsort(s, kind="stable")
            pick = np.concatenate([order[:4], order[-2:]])
            trip = [(int(ia[i] + a0), int(ib[i]), int(c[ia[i], ib[i]])) for i in pick]
            best[k] = [m, keep(trip if m < best[k][0] else best[k][1] + trip)]
    return int(best[0][0]), best[0][1], int(best[1][0]), best[1][1]


@pytest.mark.parametrize("bits", [128, 2048, 4096])
def test_prefilter_never_rejects_a_neighbour(bits):
    """For every cutoff and every pair of popcounts a pair can have at this width, the pre-filter passes the pair at
    c = thresh: the margin is >= 0. And thresh is what its name says: c = thresh passes the fp64 predicate, c - 1 not."""
    for cutoff in CUTOFFS:
        t = thresh_table(bits, cutoff)
        s = np.arange(len(t))
        has = t != NEVER
        assert is_neighbour(t[has], s[has], 0, cutoff).all(), cutoff
        pos = has & (t > 0)
        assert not is_neighbour(t[pos] - 1, s[pos], 0, cutoff).any(), cutoff
        margin, trip, _, _ = boundary(bits, cutoff)
        assert margin >= 0, (cutoff, margin, trip)
    # the tightest cases the model finds (at the bench cutoff 0.3 the slack is 16/256, elsewhere down to 1/256)
    if bits >= 2048:
        assert boundary(bits, 0.3)[0] == 16
        assert boundary(bits, 0.5)[0] == 1 and (1, 2, 1) in boundary(bits, 0.5)[1]
        assert boundary(bits, 0.30000000000000004)[0] == 1
        assert boundary(bits, 1.0)[0] == 0 and (0, 0, 0) in boundary(bits, 1.0)[1]


def test_prefilter_model_examples():
    """Hand-checked values of the model: alpha and T at cutoff 0.5, where alpha = 1/3."""
    alpha = prefilter_alpha(0.5)
    assert alpha < np.float32(1 / 3) and np.nextafter(np.nextafter(alpha, np.float32(1)), np.float32(1)) >= np.float32(1 / 3)
    assert prefilter_term([0, 1, 2, 3], alpha).tolist() == [0, 85, 170, 255]  # 256 / 3 = 85.33; 3 x 85.33 just below 256
    assert thresh_table(2048, 0.5)[3] == 1  # (1, 2, 1): sim 1/2, distance 0.5 <= 0.5
    assert 256 * 1 - 85 - 170 == 1


# ------------------------------------------------------------------ GPU: the boundary pairs through the passes
def _expand(fp: np.ndarray) -> np.ndarray:
    return np.unpackbits(np.ascontiguousarray(fp).view(np.uint8), axis=1, bitorder="little").astype(np.float64)


def _reference(x: np.ndarray, y: np.ndarray, cutoff: float) -> np.ndarray:
    """[nx][ny] neighbour flags from exact counts (float64 matmul of the 0/1 expansions) and the fp64 predicate."""
    ex, ey = _expand(x), _expand(y)
    c = ex @ ey.T
    return is_neighbour(c, ex.sum(1)[:, None], ey.sum(1)[None, :], cutoff)


def _pair_bits(rng, bits, a, b, c):
    """Two bool rows with popcounts a, b and intersection c at random positions."""
    perm = rng.permutation(bits)
    ra, rb = np.zeros(bits, dtype=bool), np.zeros(bits, dtype=bool)
    ra[perm[:a]] = True
    rb[perm[a - c:a - c + b]] = True
    return ra, rb


def _cases(bits, cutoff, fit_block):
    """(a, b, c) triples to build: the smallest-margin ones at c = thresh and c = thresh - 1, and the sim = 7/10 pairs."""
    _, trip, _, trip_fit = boundary(bits, cutoff)
    fits = (lambda a, b, c: block_bits(a, b, c) <= bits) if fit_block else (lambda a, b, c: a + b - c <= bits)
    out = []
    for a, b, c in trip_fit if fit_block else trip:
        out.append((a, b, c))
        if c > 0 and fits(a, b, c - 1):
            out.append((a, b, c - 1))
    out += [t for t in SEVEN_TENTHS if fits(*t)]
    for a, b, c in out:  # the construction puts them on the intended sides of the boundary
        assert a + b - c <= bits and c <= min(a, b)
        if (a, b, c + 1) in out:
            assert not is_neighbour(c, a, b, cutoff)
    return out


@pytest.fixture(params=[(-1, 1), (0, 0), (0, 1), (0, 3)], ids=["simt_tile", "single_cta", "multicast_pair", "row_stationary"])
def pair_tile(cuda, request):
    """The tile a small X-vs-Y count runs on: SIMT, or tensor variant 0, 1 or 3 (unsuperposed: acc = c)."""
    from nvmolkit_b200 import _lib

    with _lib.options(similarity_tensor_min_pairs=request.param[0], similarity_tensor_cluster=request.param[1]):
        yield request.param


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [128, 2048, 4096])
def test_count_ge_on_the_boundary(cuda, pair_tile, bits):
    """b200mol_tanimoto_count_ge over X = [A..., B..., empty, empty] and Y = [B..., A..., empty, empty]: each boundary
    pair in both orientations, plus two empty rows (neighbours of everything at cutoff 1.0, of each other included)."""
    from nvmolkit_b200 import _lib

    rng = np.random.default_rng(bits)
    for cutoff in CUTOFFS:
        cases = _cases(bits, cutoff, fit_block=False)
        rows = [_pair_bits(rng, bits, *t) for t in cases]
        ra, rb = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
        empty = np.zeros((2, bits), dtype=bool)
        x = S.pack_bits(np.concatenate([ra, rb, empty]))
        y = S.pack_bits(np.concatenate([rb, ra, empty]))
        want_pair = is_neighbour([t[2] for t in cases], [t[0] for t in cases], [t[1] for t in cases], cutoff)
        ref = _reference(x, y, cutoff)
        k = len(cases)
        assert (np.diag(ref)[:k] == want_pair).all() and (np.diag(ref)[k:2 * k] == want_pair).all()
        want = ref.sum(1).astype(np.int32)
        assert (oracle.count_ge(x, y, cutoff) == want).all(), cutoff
        dx, dy = torch.from_numpy(x.view(np.int32)).to(cuda), torch.from_numpy(y.view(np.int32)).to(cuda)
        counts = torch.zeros(len(x), dtype=torch.int32, device=cuda)
        _lib.call("b200mol_tanimoto_count_ge", dx.data_ptr(), len(x), dy.data_ptr(), len(y), bits // 32, 0, cutoff, 1,
                  counts.data_ptr(), torch.cuda.current_stream().cuda_stream)
        got = counts.cpu().numpy()
        assert (got == want).all(), (cutoff, [(cases[i % k], got[i], want[i]) for i in np.nonzero(got != want)[0]])


def _blocks(rng, bits, cases):
    """One block of 16 fingerprints per boundary pair: A at 16 k + ra, B at 16 k + 12 + rb, the other members of rows
    16 k .. 16 k + 3 are row fillers (|A| + FILL bits), those of rows 16 k + 12 .. 16 k + 15 column fillers (|B| + FILL
    bits), rows 16 k + 4 .. 16 k + 11 are empty; all supports disjoint except A & B. For every superposition S x C
    (S, C in 1, 2, 4) the group holding the pair then sums exactly its c, and its smallest popcounts are |A| and |B|
    wherever in the group A and B sit. Blocks reuse bit positions: no group holding a boundary pair reaches outside its
    block."""
    out = np.zeros((16 * len(cases), bits), dtype=bool)
    where = []
    for k, (a, b, c) in enumerate(cases):
        ra, rb = k % 4, (k + k // 4 + 1) % 4
        perm = rng.permutation(bits)
        blk = out[16 * k:16 * k + 16]
        blk[ra, perm[:a]] = True
        blk[12 + rb, perm[a - c:a - c + b]] = True
        at = a + b - c
        for r in [r for r in range(4) if r != ra]:
            blk[r, perm[at:at + a + FILL]] = True
            at += a + FILL
        for r in [12 + r for r in range(4) if r != rb]:
            blk[r, perm[at:at + b + FILL]] = True
            at += b + FILL
        assert at <= bits
        where.append((16 * k + ra, 16 * k + 12 + rb))
    return S.pack_bits(out), where


@pytest.fixture(params=[None, (4, 4), (4, 2), (4, 1), (2, 1), (1, 1)],
                ids=["simt_tile", "super4x4", "super4x2", "super4x1", "super2x1", "plain"])
def superposition(cuda, request):
    """The neighbour pass on the SIMT tile, or on the tensor tile with rows x columns superposition (no pilot)."""
    from nvmolkit_b200 import _lib

    if request.param is None:
        tile = _lib.options(similarity_tensor_min_pairs=-1)
    else:
        tile = _lib.options(similarity_tensor_min_pairs=0, similarity_superpose=request.param[0],
                            similarity_superpose_cols=request.param[1])
    with tile:
        yield request.param


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2048, 4096])
def test_neighbor_edges_on_the_boundary(cuda, superposition, bits):
    """b200mol_neighbor_edges over blocks that each hold one boundary pair in a tight group: the degrees and the edge
    set must equal the fp64 definition's (a clustering could hide a missing edge)."""
    from nvmolkit_b200 import _lib

    rng = np.random.default_rng(bits + 1)
    sptr = torch.cuda.current_stream().cuda_stream
    for cutoff in CUTOFFS:
        cases = _cases(bits, cutoff, fit_block=True)
        fp, where = _blocks(rng, bits, cases)
        n = len(fp)
        ref = _reference(fp, fp, cutoff)
        want_pair = is_neighbour([t[2] for t in cases], [t[0] for t in cases], [t[1] for t in cases], cutoff)
        assert all(ref[i, j] == w for (i, j), w in zip(where, want_pair))
        assert (oracle.count_ge(fp, fp, cutoff) == ref.sum(1)).all(), cutoff
        np.fill_diagonal(ref, False)  # (an empty row is its own neighbour only at cutoff 1.0; no pass lists self pairs)
        want_deg = ref.sum(1).astype(np.int32)
        wi, wj = np.nonzero(np.triu(ref))
        d = torch.from_numpy(fp.view(np.int32)).to(cuda)
        cap = max(1, n * (n - 1) // 2)
        counts = torch.zeros(n, dtype=torch.int32, device=cuda)
        edges = torch.empty((cap, 2), dtype=torch.int32, device=cuda)
        found = C.c_uint64(0)
        _lib.call("b200mol_neighbor_edges", d.data_ptr(), n, bits // 32, 0, float(cutoff), 0, 1, counts.data_ptr(),
                  edges.data_ptr(), cap, C.byref(found), sptr)
        if superposition is not None:
            assert _lib.get_option("similarity_superpose_last") == superposition[0] * superposition[1]
        deg = counts.cpu().numpy()
        e = edges[: found.value].cpu().numpy().astype(np.int64)
        missing = sorted(set(zip(wi.tolist(), wj.tolist())) - set(zip(e[:, 0].tolist(), e[:, 1].tolist())))
        assert (deg == want_deg).all() and not missing, (cutoff, [(cases[k], p) for k, p in enumerate(where) if p in missing])
        assert (e[:, 0] < e[:, 1]).all()
        key = np.sort(e[:, 0] * n + e[:, 1])
        assert len(key) == len(wi) and (key == np.sort(wi * n + wj)).all(), cutoff
