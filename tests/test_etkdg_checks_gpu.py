"""Every ETKDG acceptance check of csrc/etkdg.cu at each branch and on both sides of its threshold, and every stage exit
of the embedding kernel.

Each fixture molecule carries hand-written check tables that isolate one check, and a list of labelled geometries with
the verdict RDKit's definitions give them. Geometries are
- exact: small dyadic coordinates, so every product and cross product is exact in fp64 and the kernel (FMA-contracted)
  and the oracle (no contraction) take the same branch even on a tie;
- near: the guarded quantity 2^-20 relative either side of its threshold, far beyond any rounding difference between
  the kernel (which normalises by multiplying with 1 / l) and the oracle (which divides);
- generic: far from every threshold.
CPU: every check restated in numpy from RDKit's definitions (DistGeomUtils / Embedder: _volumeTest, _sameSide,
_centerInVolume, checkChiralCenters, _boundsFulfilled, doubleBondGeometryChecks, doubleBondStereoChecks, the improper
planarity test and the per-atom energy test), against the oracle and against the stated verdicts, under every switch.
GPU, check kernel: the same fixtures in one batch, bit for bit against the oracle; a check with more terms than the
CTA has threads, failing at one term placed at each edge of the strided loop; more slots than the grid, a molecule
whose coordinates exceed 48 KB of shared memory, a molecule without tables.
GPU, attempt kernel: molecules that fail one stage on every attempt end every attempt at that stage, with the same
histogram as the oracle's pipeline; two such stages count at the earlier one; switching the owning stage off embeds.
"""
import ctypes as C
import math
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

import oracle
from nvmolkit_b200 import synthetic as S
from nvmolkit_b200.embedMolecules import FlatEmbedMolecules
from nvmolkit_b200.forcefield import CheckTables, FlatSystem

DELTA = 2.0 ** -20
PARAMS = dict(seed=1234, boxSize=10.0, optimizerForceTol=1e-3, enforceChirality=1, useExpTorsions=1, useBasicKnowledge=1,
              maxAttempts=30, dgIters=400, fourthIters=200, etkIters=300, maxRestarts=20, useMetricStart=0)

# failure bits (include/b200mol.h): bit s = stage s failed
ENERGY, TET, CHIR1, PLAN, DBGEOM, CHIR2, CDIST, CIV, DBSTEREO = (1 << s for s in (1, 2, 3, 5, 6, 7, 8, 9, 10))
CHIR = CHIR1 | CHIR2
CHIRALITY_BITS = CHIR | CDIST | CIV | DBSTEREO  # owned by enforceChirality
KT = 256  # threads per CTA of the check and attempt kernels


@dataclass
class Geom:
    label: str
    pos: np.ndarray  # [n, 4]
    want: int  # failure mask with every switch on
    kind: str = "generic"  # generic | exact | near


@dataclass
class Fixture:
    name: str
    n: int
    checks: dict  # CHECK_LAYOUT table -> (idx, par)
    geoms: list = field(default_factory=list)
    num_impropers: int = 0
    dg: dict = field(default_factory=dict)
    etk: dict = field(default_factory=dict)


def p4(xyz, w=0.0):
    x = np.asarray(xyz, float)
    out = np.zeros((len(x), 4))
    out[:, :3] = x
    out[:, 3] = w
    return out


def _unit(v):
    v = np.asarray(v, float)
    return v / np.sqrt(v @ v)


_R = np.linalg.qr(np.random.default_rng(13).normal(size=(3, 3)))[0]  # a fixed rotation: generic = out of every plane


def rot(x):
    return np.asarray(x, float) @ _R.T + np.array([0.3, -0.2, 0.7])


# ------------------------------------------------------------------------------------------------ RDKit restated
def _unit_or_zero(v):
    # (as the kernel and the oracle do; which value a zero arm gets cannot change a verdict, see the "arm atom on the
    # centre" geometry)
    l = np.sqrt(v @ v)
    return v / l if l > 0.0 else v


def volume_fails(pos, row, fused):
    """Embedder _volumeTest: |(d_a x d_b) . d_c| >= 0.5 (x0.25 in fused small rings) for the four triples of unit arms."""
    p0 = pos[row[0], :3]
    d = [_unit_or_zero(p0 - pos[row[k], :3]) for k in (1, 2, 3, 4)]
    lim = 0.5 * (0.25 if fused else 1.0)
    return any(abs(np.cross(d[a], d[b]) @ d[c]) < lim for a, b, c in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)))


def _same_side(v1, v2, v3, v4, p0, tol):
    n = np.cross(v2 - v1, v3 - v1)
    d1, d2 = n @ (v4 - v1), n @ (p0 - v1)
    if abs(d1) < tol or abs(d2) < tol:
        return False
    return (d1 < 0.0) == (d2 < 0.0)


def centre_outside(pos, row, tol):
    """Embedder _centerInVolume (failure = not inside); a three-coordinate set (idx0 == idx4) is never judged."""
    if row[0] == row[4]:
        return False
    p0, p1, p2, p3, p4_ = (pos[row[k], :3] for k in range(5))
    return not (_same_side(p1, p2, p3, p4_, p0, tol) and _same_side(p2, p3, p4_, p1, p0, tol) and
                _same_side(p3, p4_, p1, p2, p0, tol) and _same_side(p4_, p1, p2, p3, p0, tol))


def chiral_volume(pos, a, b, c, d):
    """ChiralViolationContrib::calcChiralVolume on the first three coordinates."""
    v1, v2, v3 = pos[a, :3] - pos[d, :3], pos[b, :3] - pos[d, :3], pos[c, :3] - pos[d, :3]
    return v1 @ np.cross(v2, v3)


def chirality_fails(vol, lb, ub):
    """Embedder checkChiralCenters."""
    opposite = lambda x, y: np.signbit(x) != np.signbit(y)  # noqa: E731
    return bool((lb > 0 and vol < lb and (vol / lb < 0.8 or opposite(vol, lb))) or
                (ub < 0 and vol > ub and (vol / ub < 0.8 or opposite(vol, ub))))


def bounds_fail(dist, lb, ub):
    """Embedder _boundsFulfilled (failure): outside the bounds by more than a tenth of the UPPER bound, both sides."""
    return bool((dist < lb and abs(dist - lb) > 0.1 * ub) or (dist > ub and abs(dist - ub) > 0.1 * ub))


def dihedral(a0, a1, a2, a3):
    """RDGeom::computeDihedralAngle with Point3D::angleTo (the normalised dot clamped to [-1, 1] by returning 0 / pi)."""
    e = a2 - a1
    c1, c2 = np.cross(a0 - a1, e), np.cross(a3 - a2, e)
    dt = (c1 @ c2) / np.sqrt((c1 @ c1) * (c2 @ c2))
    if dt <= -1.0:
        return np.pi
    if dt >= 1.0:
        return 0.0
    return float(np.arccos(dt))


def linear_fails(a0, a1, a2):
    """Embedder doubleBondGeometryChecks: unit(a1 - a0) . unit(a1 - a2) + 1 < 1e-3."""
    return bool(_unit_or_zero(a1 - a0) @ _unit_or_zero(a1 - a2) + 1.0 < 1e-3)


def dg_energy(dg, pos):
    """DistViolationContrib + ChiralViolationContrib (weight 1) + FourthDimContrib (weight 0.1) in four dimensions."""
    e = 0.0
    if "dist" in dg:
        for (i, j), (lb2, ub2, w) in zip(*dg["dist"]):
            d2 = float(((pos[i] - pos[j]) ** 2).sum())
            val = d2 / ub2 - 1.0 if d2 > ub2 else (2.0 * lb2 / (lb2 + d2) - 1.0 if d2 < lb2 else 0.0)
            e += w * val * val
    if "chiral" in dg:
        for (a, b, c, d), (ub, lb) in zip(*dg["chiral"]):
            vol = chiral_volume(pos, a, b, c, d)
            e += (vol - lb) ** 2 if vol < lb else ((vol - ub) ** 2 if vol > ub else 0.0)
    if "fourth" in dg:
        for (a,) in dg["fourth"][0]:
            e += 0.1 * pos[a, 3] ** 2
    return e


def improper_energy(etk, pos):
    """UFF InversionContrib as ETKDG uses it: K (C0 + C1 sin Y + C2 cos 2W), cos Y from calculateCosY."""
    e = 0.0
    if "improper" not in etk:
        return e
    for (i, j, k, l), (c0, c1, c2, fk) in zip(*etk["improper"]):
        ji, jk, jl = pos[i, :3] - pos[j, :3], pos[k, :3] - pos[j, :3], pos[l, :3] - pos[j, :3]
        cos_y = 0.0
        if min(ji @ ji, jk @ jk, jl @ jl) >= 1e-16:
            n = np.cross(ji, jk) / (np.sqrt(ji @ ji) * np.sqrt(jk @ jk))
            if n @ n >= 1e-16:
                cos_y = (n @ jl) / (np.sqrt(jl @ jl) * np.sqrt(n @ n))
        s2 = 1.0 - cos_y * cos_y
        sin_y = np.sqrt(s2) if s2 > 0.0 else 0.0
        e += fk * (c0 + c1 * sin_y + c2 * (2.0 * sin_y * sin_y - 1.0))
    return e


def _rows(fx, name):
    return zip(*fx.checks[name]) if name in fx.checks else ()


def rdkit_mask(fx, pos, params=PARAMS):
    """The failure mask of one geometry, from RDKit's definitions (every check evaluated, none stops the others)."""
    ec, ubk = params["enforceChirality"], params["useBasicKnowledge"]
    m = 0
    if dg_energy(fx.dg, pos) / fx.n >= 0.05:
        m |= ENERGY
    if any(volume_fails(pos, r, p[0] != 0.0) or centre_outside(pos, r, 0.3) for r, p in _rows(fx, "tetrahedral")):
        m |= TET
    chir = any(chirality_fails(chiral_volume(pos, *r[1:]), p[0], p[1]) for r, p in _rows(fx, "chiral"))
    if ec and chir:
        m |= CHIR
    if ubk and improper_energy(fx.etk, pos) > 0.7 * fx.num_impropers:
        m |= PLAN
    if any(linear_fails(*(pos[a, :3] for a in r)) for r, _p in _rows(fx, "dbGeom")):
        m |= DBGEOM
    if ec:
        if any(bounds_fail(np.linalg.norm(pos[a, :3] - pos[b, :3]), p[0], p[1]) for (a, b), p in _rows(fx, "chiralDist")):
            m |= CDIST
        if any(centre_outside(pos, r, 0.1) for r, _p in _rows(fx, "chiral")):
            m |= CIV
        if any((dihedral(*(pos[a, :3] for a in r)) - np.pi / 2) * p[0] < 0.0 for r, p in _rows(fx, "dbStereo")):
            m |= DBSTEREO
    return m


def switched(want, params):
    off = (0 if params["enforceChirality"] else CHIRALITY_BITS) | (0 if params["useBasicKnowledge"] else PLAN)
    return want & ~off


SWITCHES = [dict(PARAMS, enforceChirality=ec, useBasicKnowledge=ubk) for ec in (1, 0) for ubk in (1, 0)]
SWITCH_IDS = [f"chirality{ec}-basic{ubk}" for ec in (1, 0) for ubk in (1, 0)]


# ------------------------------------------------------------------------------------------------ fixtures
def _tables(idx, par, k, p):
    return (np.asarray(idx, np.int16).reshape(-1, k), np.asarray(par, float).reshape(len(idx), p))


def tet_arms(which, t):
    """Four unit arms whose triple product number `which` ((1,2,3), (1,2,4), (1,3,4), (2,3,4)) is -t or t, the others
    +-1 or +-sqrt((1 - t^2) / 2) (> 0.6 for t <= 0.5)."""
    a = np.sqrt((1.0 - t * t) / 2.0)
    x, y, z = np.eye(3)
    if which == 0:
        return [x, y, -np.array([a, a, t]), z]
    return [x, y, z, -np.array({1: (a, a, t), 2: (a, t, a), 3: (t, a, a)}[which])]


def tet_geom(arms, length=4.0):
    """Centre atom 0 at the origin, atom k at -length * arm k (length a power of two: p0 - pk = length * arm exactly)."""
    return p4([[0.0, 0.0, 0.0]] + [-length * np.asarray(d) for d in arms])


REG = np.array([[1.0, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]])  # a regular tetrahedron around the origin


def tetrahedral_fixtures():
    out = []
    for fused in (0.0, 1.0):
        lim = 0.125 if fused else 0.5
        g = []
        for which in range(4):
            g.append(Geom(f"triple {which} above limit", tet_geom(tet_arms(which, lim * (1 + DELTA))), 0, "near"))
            g.append(Geom(f"triple {which} below limit", tet_geom(tet_arms(which, lim * (1 - DELTA))), TET, "near"))
        # between the fused and the unfused limit: the flag decides
        g.append(Geom("triple 0.3", tet_geom(tet_arms(1, 0.3)), 0 if fused else TET))
        g.append(Geom("regular", p4(np.concatenate([[[0.0, 0, 0]], rot(REG) - rot([0, 0, 0])])), 0))
        # an arm atom on the centre: the centre lies in three face planes (same-side products 0), so the centre-in-volume
        # test fails it whatever its volumes are, zero (a zero arm kept zero) or NaN (a division by the zero length)
        g.append(Geom("arm atom on the centre", p4([[0.0, 0, 0], [0, 0, 0], [0, 2.0, 0], [0, 0, 2.0], [-2.0, -2.0, -2.0]]),
                      TET, "exact"))
        g.append(Geom("coplanar arms", p4([[0.0, 0, 0], [2.0, 0, 0], [0, 2.0, 0], [-2.0, 0, 0], [0, -2.0, 1.0]]), TET, "exact"))
        out.append(Fixture(f"tetrahedral fused={fused:g}", 5,
                           {"tetrahedral": _tables([(0, 1, 2, 3, 4)], [fused], 5, 1)}, g))
    return out


def centre_in_volume_fixture():
    """A tetrahedral row and a chiral row (bounds 0, 0: chirality never fails) on the same centre: stage 2 judges the
    centre at tolerance 0.3, stage 9 at 0.1. Regular tetrahedron scaled by s: every same-side product is 4 s^3."""
    rows = {"tetrahedral": _tables([(0, 1, 2, 3, 4)], [0.0], 5, 1), "chiral": _tables([(0, 1, 2, 3, 4)], [(0.0, 0.0)], 5, 2)}
    g = [Geom("centroid", p4(np.concatenate([[[0.0, 0, 0]], REG])), 0, "exact"),
         Geom("same-side 0.2109 (s = 3/8)", p4(np.concatenate([[[0.0, 0, 0]], 0.375 * REG])), TET, "exact")]
    for k in range(4):  # centre at -v_k: outside the face opposite v_k only; the arms stay > 0.57 in volume
        g.append(Geom(f"outside face {k}", p4(np.concatenate([[-REG[k]], REG])), TET | CIV, "exact"))
    for tol, want_above, want_below in ((0.3, 0, TET), (0.1, TET, TET | CIV)):
        for sgn, want in ((1, want_above), (-1, want_below)):
            s = (tol * (1 + sgn * DELTA) / 4.0) ** (1.0 / 3.0)
            g.append(Geom(f"same-side {tol:g} {'above' if sgn > 0 else 'below'}", p4(np.concatenate([[[0.0, 0, 0]], s * REG])),
                          want, "near"))
    return Fixture("centre in volume", 5, rows, g)


def _chiral_geom(vol):
    """Centre 0 at the origin, neighbours 1-4 a regular tetrahedron of chiral volume vol (16 s^3, sign by a swap)."""
    s = (abs(vol) / 16.0) ** (1.0 / 3.0)
    v = s * REG
    if vol < 0:
        v = v[[1, 0, 2, 3]]
    return p4(np.concatenate([[[0.0, 0, 0]], v]))


def chirality_fixtures():
    out = []
    for lb, ub in ((5.0, 100.0), (-100.0, -5.0)):
        b = lb if lb > 0 else ub  # the bound the check compares with
        sg = 1.0 if lb > 0 else -1.0
        g = [Geom("0.8 bound, inside", _chiral_geom(0.8 * b * (1 + DELTA)), 0, "near"),
             Geom("0.8 bound, outside", _chiral_geom(0.8 * b * (1 - DELTA)), CHIR, "near"),
             Geom("bound, inside", _chiral_geom(b * (1 + DELTA)), 0, "near"),
             Geom("bound, short", _chiral_geom(b * (1 - DELTA)), 0, "near"),
             Geom("opposite sign", _chiral_geom(-0.8 * b), CHIR),
             Geom("beyond the far bound", _chiral_geom(2.0 * (ub if lb > 0 else lb)), 0),  # RDKit accepts it
             Geom("volume 16 (s = 1)", _chiral_geom(16.0 * sg), 0, "exact"),
             Geom("volume 2 (s = 1/2)", _chiral_geom(2.0 * sg), CHIR, "exact"),
             Geom("volume -16", _chiral_geom(-16.0 * sg), CHIR, "exact"),
             Geom("zero volume", p4([[0.0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [-1.0, 0, 0], [0, -1.0, 0]]), CHIR | CIV, "exact")]
        out.append(Fixture(f"chirality ({lb:g}, {ub:g})", 5, {"chiral": _tables([(0, 1, 2, 3, 4)], [(lb, ub)], 5, 2)}, g))
    # RDKit's three-coordinate set: idx4 = idx0 (the centre stands in for the fourth neighbour), lower bound 2; the
    # centre-in-volume test never judges it. Neighbours at s * (x, y, z): volume s^3.
    g = []
    for lab, vol, want, kind in (("0.8 bound, inside", 1.6 * (1 + DELTA), 0, "near"),
                                 ("0.8 bound, outside", 1.6 * (1 - DELTA), CHIR, "near"),
                                 ("bound, short", 2.0 * (1 - DELTA), 0, "near"),
                                 ("volume 1", 1.0, CHIR, "exact"), ("volume 8", 8.0, 0, "exact"),
                                 ("opposite sign", -8.0, CHIR, "exact")):
        s = np.cbrt(vol)
        g.append(Geom(lab, p4([[0.0, 0, 0], [s, 0, 0], [0, s, 0], [0, 0, s]]), want, kind))
    out.append(Fixture("chirality three-coordinate", 4, {"chiral": _tables([(0, 1, 2, 3, 0)], [(2.0, 100.0)], 5, 2)}, g))
    return out


def chiral_dist_fixture():
    """lb = 1, ub = 4: the tolerance is 0.1 * ub = 0.4 on both sides (0.1 * lb would be 0.1)."""
    lb, ub = 1.0, 4.0
    u = _unit([0.31, -0.62, 0.72])
    pair = lambda d: p4([[0.1, 0.2, -0.3], np.array([0.1, 0.2, -0.3]) + d * u])  # noqa: E731
    g = [Geom("below lb, inside tolerance", pair(lb - 0.1 * ub * (1 - DELTA)), 0, "near"),
         Geom("below lb, outside tolerance", pair(lb - 0.1 * ub * (1 + DELTA)), CDIST, "near"),
         Geom("above ub, inside tolerance", pair(ub + 0.1 * ub * (1 - DELTA)), 0, "near"),
         Geom("above ub, outside tolerance", pair(ub + 0.1 * ub * (1 + DELTA)), CDIST, "near"),
         Geom("inside", pair(2.5), 0),
         Geom("3-4-5", p4([[0.0, 0, 0], [3.0, 4.0, 0]]), CDIST, "exact"),
         Geom("on ub", p4([[0.0, 0, 0], [0, 4.0, 0]]), 0, "exact"),
         Geom("0.5", p4([[0.0, 0, 0], [0, 0, 0.5]]), CDIST, "exact"),
         Geom("coincident", p4([[0.25, 0, 0], [0.25, 0, 0]]), CDIST, "exact")]
    return Fixture("chiral distance", 2, {"chiralDist": _tables([(0, 1)], [(lb, ub)], 2, 2)}, g)


def planarity_fixtures():
    """One improper centre (atom 0) = three terms, numImpropers = 1 (RDKit counts centres): threshold 0.7. The centre
    is lifted by h above the plane of its neighbours; the energy grows with h."""
    imp = _tables([(1, 0, 2, 3), (1, 0, 3, 2), (2, 0, 3, 1)], [(1.0, -1.0, 0.0, 10.0 / 3.0)] * 3, 4, 4)
    flat_nb = np.array([[1.0, 0, 0], [-0.5, 0.75, 0], [-0.5, -0.75, 0]])  # (dyadic, not quite 120 degrees)

    def lifted(h):
        return p4(np.concatenate([[[0.0, 0.0, h]], flat_nb]))

    fx = Fixture("planarity", 4, {}, num_impropers=1, etk={"improper": imp})

    def energy(h):
        return improper_energy(fx.etk, lifted(h))

    g = [Geom("planar", lifted(0.0), 0, "exact"), Geom("lifted 0.05", lifted(0.05), 0), Geom("lifted 1.0", lifted(1.0), PLAN)]
    for sgn, want in ((1, PLAN), (-1, 0)):
        h = _solve(energy, 0.7 * (1 + sgn * DELTA), 0.0, 1.0)
        g.append(Geom(f"energy 0.7 {'above' if sgn > 0 else 'below'}", lifted(h), want, "near"))
    fx.geoms = g
    # no centre counted: an exactly planar centre has energy exactly 0, and 0 > 0 is false
    zero = Fixture("planarity numImpropers=0", 4, {}, [Geom("planar", lifted(0.0), 0, "exact"),
                                                       Geom("lifted 0.05", lifted(0.05), PLAN)], 0, etk={"improper": imp})
    return [fx, zero]


def db_geometry_fixture():
    """Atom 1 at the origin, atom 0 on -x, atom 2 at angle theta from +x: unit(1 - 0) . unit(1 - 2) + 1 = 1 - cos(theta)."""
    def at(c):
        s = np.sqrt(1.0 - c * c)
        return p4([[-1.5, 0, 0], [0, 0, 0], [1.25 * c, 1.25 * s, 0]])

    g = [Geom("inside tolerance", at(1.0 - 1e-3 * (1 - DELTA)), DBGEOM, "near"),
         Geom("outside tolerance", at(1.0 - 1e-3 * (1 + DELTA)), 0, "near"),
         Geom("linear", p4([[-1.0, 0, 0], [0, 0, 0], [2.0, 0, 0]]), DBGEOM, "exact"),
         Geom("right angle", p4([[-1.0, 0, 0], [0, 0, 0], [0, 2.0, 0]]), 0, "exact"),
         Geom("generic", p4(rot([[-1.3, 0, 0], [0, 0, 0], [0.6, 1.1, 0]])), 0),
         Geom("folded", p4([[-1.0, 0, 0], [0, 0, 0], [-2.0, 0, 0]]), 0, "exact")]
    return Fixture("double-bond geometry", 3, {"dbGeom": _tables([(0, 1, 2)], np.zeros((1, 0)), 3, 0)}, g)


CIS = np.array([[0.0, 1.0, 0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [1.0, 1.0, 0.0]])
TRANS = np.array([[0.0, 1.0, 0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [1.0, -1.0, 0.0]])


def _stereo_dot(x):
    """The normalised dot of the double-bond stereo check in the oracle's operation order, in plain float arithmetic
    (no BLAS, no contraction)."""
    p0, p1, p2, p3 = ([float(c) for c in row[:3]] for row in x)
    d1, d2, d3 = ([a[i] - b[i] for i in range(3)] for a, b in ((p2, p1), (p0, p1), (p3, p2)))

    def crs(a, b):
        return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]

    def dot(a, b):
        return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]

    c1, c2 = crs(d2, d1), crs(d3, d1)
    return dot(c1, c2) / math.sqrt(dot(c1, c1) * dot(c2, c2))


def _rotations_past_one(base, sign, count, seed):
    """Random rotations of an exactly planar set whose normalised dot, as the oracle computes it, rounds beyond +-1.
    (The kernel's contracted arithmetic rounds some of the same sets past +-1 and others not; taking many makes it
    likely that some are, which is what the clamp before acos is there for.)"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        x = base @ q.T
        if _stereo_dot(x) * sign > 1.0:
            out.append(x)
    return out


def db_stereo_fixtures():
    out = []
    for sign in (1.0, -1.0):
        want_cis, want_trans = (DBSTEREO, 0) if sign > 0 else (0, DBSTEREO)
        g = [Geom("cis", p4(CIS), want_cis, "exact"), Geom("trans", p4(TRANS), want_trans, "exact"),
             # dot exactly 0: acos(0) must equal pi / 2 exactly for both signs to pass
             Geom("90 degrees", p4([[0.0, 1.0, 0], [0, 0, 0], [1.0, 0, 0], [1.0, 0, 1.0]]), 0, "exact"),
             Geom("89.99 degrees", p4([[0.0, 1.0, 0], [0, 0, 0], [1.0, 0, 0], [1.0, np.sin(1e-4), np.cos(1e-4)]]),
                  want_cis, "near"),
             Geom("90.01 degrees", p4([[0.0, 1.0, 0], [0, 0, 0], [1.0, 0, 0], [1.0, -np.sin(1e-4), np.cos(1e-4)]]),
                  want_trans, "near"),
             Geom("60 degrees", p4(rot([[0.0, 1.0, 0], [0, 0, 0], [1.4, 0, 0], [1.4, 0.5, 0.866]])), want_cis),
             Geom("130 degrees", p4(rot([[0.0, 1.0, 0], [0, 0, 0], [1.4, 0, 0], [1.4, -0.643, 0.766]])), want_trans)]
        for k, x in enumerate(_rotations_past_one(TRANS, -1.0, 64, 17)):
            g.append(Geom(f"trans rotated {k} (dot < -1)", p4(x), want_trans, "near"))
        for k, x in enumerate(_rotations_past_one(CIS, 1.0, 64, 19)):
            g.append(Geom(f"cis rotated {k} (dot > 1)", p4(x), want_cis, "near"))
        out.append(Fixture(f"double-bond stereo sign {sign:+g}", 4, {"dbStereo": _tables([(0, 1, 2, 3)], [sign], 4, 1)}, g))
    return out


def _solve(f, target, lo, hi):
    """A point where the increasing-through-target function f is within 2^-30 relative of target (bisection)."""
    flo, fhi = f(lo) - target, f(hi) - target
    assert flo < 0.0 < fhi, (flo, fhi)
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        fm = f(mid) - target
        if abs(fm) <= 2.0 ** -30 * abs(target):
            return mid
        lo, hi = (mid, hi) if fm < 0.0 else (lo, mid)
    raise AssertionError("bisection did not reach the target")


def _synthetic_tables(n_heavy_lo, n_heavy_hi, seed):
    flat, _ = S.random_embed_molecules(1, n_heavy_lo, n_heavy_hi, seed=seed)
    dg = {k: (ix, pr) for k, (_st, ix, pr) in flat.dg.tables.items()}
    etk = {k: (ix, pr) for k, (_st, ix, pr) in flat.etk.tables.items()}
    return int(flat.atom_counts[0]), dg, etk


def _dg_oracle_energy(fx, pos):
    sysf = FlatSystem.from_molecules("dg", [fx.n], [fx.dg])
    return oracle.ff_energy_grad("dg", sysf.atom_counts, sysf.tables, 0, pos, False, dim=4, chiral_weight=1.0,
                                 fourth_dim_weight=0.1)[0]


def energy_fixture():
    """DG tables of a small synthetic molecule, no check tables. From a DG minimum the geometry moves along a fixed
    direction; the points where the oracle's energy is 0.05 nA (1 -+ 2^-20) are found by bisection."""
    n, dg, _ = _synthetic_tables(6, 9, 32)
    fx = Fixture("energy per atom", n, {}, dg=dg)
    sysf = FlatSystem.from_molecules("dg", [n], [dg])
    rng = np.random.default_rng(3)
    pos, e, _c, _i = oracle.ff_minimize("dg", sysf.atom_counts, sysf.tables, [0], [0, n], (rng.random((n, 4)) - 0.5) * 8.0,
                                        3000, 1e-6, dim=4, chiral_weight=1.0, fourth_dim_weight=0.1)
    assert e[0] / n < 0.025
    step = rng.normal(0.0, 1.0, (n, 4))
    thr = 0.05 * n
    g = [Geom("minimum", pos, 0), Geom("far", pos + 3.0 * step, ENERGY)]
    f = lambda t: _dg_oracle_energy(fx, pos + t * step)  # noqa: E731
    hi = 0.05
    while f(hi) < 2.0 * thr:
        hi *= 2.0
    for sgn, want in ((1, ENERGY), (-1, 0)):
        t = _solve(f, thr * (1 + sgn * DELTA), 0.0, hi)
        g.append(Geom(f"energy 0.05 nA {'above' if sgn > 0 else 'below'}", pos + t * step, want, "near"))
    fx.geoms = g
    return fx


def empty_fixture():
    return Fixture("no tables", 3, {}, [Geom("generic", np.random.default_rng(1).normal(0, 1.0, (3, 4)), 0)])


_FIXTURES = []


def fixtures():
    if not _FIXTURES:
        _FIXTURES.extend(tetrahedral_fixtures() + [centre_in_volume_fixture()] + chirality_fixtures() +
                         [chiral_dist_fixture()] + planarity_fixtures() + [db_geometry_fixture()] + db_stereo_fixtures() +
                         [energy_fixture(), empty_fixture()])
    return _FIXTURES


def flat_of(fxs):
    counts = [f.n for f in fxs]
    return FlatEmbedMolecules(FlatSystem.from_molecules("dg", counts, [f.dg for f in fxs]),
                              FlatSystem.from_molecules("etk", counts, [f.etk for f in fxs]),
                              CheckTables.from_molecules(counts, [f.checks for f in fxs], [f.num_impropers for f in fxs]))


def oracle_mask(flat, mol, pos, params=PARAMS):
    return oracle.etkdg_check((flat.dg.atom_counts, flat.dg.tables), (flat.etk.atom_counts, flat.etk.tables),
                              flat.checks.tables, flat.checks.num_impropers, params, int(mol), pos)


# ------------------------------------------------------------------------------------------------ CPU
def test_fixtures_cover_both_verdicts_of_every_check():
    seen = {}
    for fx in fixtures():
        for g in fx.geoms:
            assert g.pos.shape == (fx.n, 4) and np.isfinite(g.pos).all(), (fx.name, g.label)
            for bit in (ENERGY, TET, CHIR, PLAN, DBGEOM, CDIST, CIV, DBSTEREO):
                seen.setdefault(bit, set()).add(bool(g.want & bit))
    assert all(v == {False, True} for v in seen.values()), seen


def test_arm_atom_on_the_centre_fails_the_centre_in_volume_test():
    """Whether a zero-length arm is kept zero or divided by its zero length (NaN volumes, which pass the volume test),
    the row fails: the centre lies in three of the four face planes."""
    for fx in tetrahedral_fixtures():
        g = next(g for g in fx.geoms if g.label == "arm atom on the centre")
        row = fx.checks["tetrahedral"][0][0]
        assert centre_outside(g.pos, row, 0.3) and centre_outside(g.pos, row, 0.1)
        with np.errstate(invalid="ignore", divide="ignore"):
            p0 = g.pos[row[0], :3]
            d = [(p0 - g.pos[row[k], :3]) / np.linalg.norm(p0 - g.pos[row[k], :3]) for k in (1, 2, 3, 4)]
            vols = [abs(np.cross(d[a], d[b]) @ d[c]) for a, b, c in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3))]
        assert not any(v < 0.125 for v in vols) and any(np.isnan(v) for v in vols)  # NaN volumes: no volume verdict


@pytest.mark.parametrize("params", SWITCHES, ids=SWITCH_IDS)
def test_oracle_checks_equal_rdkit_restatement(params):
    """The oracle's mask = the numpy restatement of RDKit's checks = the stated verdict, on every fixture geometry."""
    fxs = fixtures()
    flat = flat_of(fxs)
    for m, fx in enumerate(fxs):
        for g in fx.geoms:
            ref = rdkit_mask(fx, g.pos, params)
            assert ref == switched(g.want, params), (fx.name, g.label, bin(ref), bin(g.want))
            assert oracle_mask(flat, m, g.pos, params) == ref, (fx.name, g.label)


# ------------------------------------------------------------------------------------------------ attempt-kernel fixtures
EXIT_PARAMS = dict(PARAMS, seed=99, maxAttempts=4)


def exit_molecule(checks, dg_extra=None, imp_const=False, linear=False):
    """A 21-atom synthetic molecule with its own DG and ETK tables (without the DG chiral-volume terms, which make a
    few minimisations from random starts settle above 0.05 per atom, so that no attempt fails the energy test of stage
    1 by the path its minimiser took) and the given check tables only.
    dg_extra: extra DG distance terms; imp_const: an improper term of constant energy 10 (numImpropers = 1);
    linear: three more atoms made straight for the double-bond geometry check: DG distance terms that any angle above
    97 degrees satisfies (bonds 1, ends 1.5-2 apart, so the DG energy still reaches 0), then an ETK angle term of
    179-180 degrees."""
    n, dg, etk = _synthetic_tables(6, 8, 3)
    dg["chiral"] = (np.zeros((0, 4), np.int16), np.zeros((0, 2)))
    dist_i, dist_p = [dg["dist"][0]], [dg["dist"][1]]
    four_i = [dg["fourth"][0]]
    if dg_extra is not None:
        dist_i.append(np.asarray(dg_extra[0], np.int16))
        dist_p.append(np.asarray(dg_extra[1], float))
    if linear:
        a = n
        dist_i.append(np.array([(a, a + 1), (a + 1, a + 2), (a, a + 2)], np.int16))
        dist_p.append(np.array([(1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (2.25, 4.0, 1.0)]))
        four_i.append(np.array([[a], [a + 1], [a + 2]], np.int16))
        # the ETK refinement brings the angle between 179 and 180 degrees (as RDKit does for linear centres)
        ang_i, ang_p = etk["angle13"]
        etk = dict(etk, angle13=(np.concatenate([ang_i, [(a, a + 1, a + 2)]]), np.concatenate([ang_p, [(179.0, 180.0)]])))
        n += 3
    dg = dict(dg, dist=(np.concatenate(dist_i), np.concatenate(dist_p)),
              fourth=(np.concatenate(four_i), np.zeros((sum(len(f) for f in four_i), 0))))
    n_imp = 0
    if imp_const:
        etk = dict(etk, improper=(np.array([(1, 0, 2, 3)], np.int16), np.array([(10.0, 0.0, 0.0, 1.0)])))
        n_imp = 1
    return Fixture("exit", n, checks, [], n_imp, dg, etk)


def exit_fixtures():
    """stage -> molecule that fails that stage on every attempt (checks of the stages before it cannot fail)."""
    return {
        1: exit_molecule({}, dg_extra=([(0, 1)], [(400.0, 441.0, 100.0)])),  # bond 0-1 also held at 20-21: inconsistent
        2: exit_molecule({"tetrahedral": _tables([(4, 1, 1, 2, 3)], [0.0], 5, 1)}),  # a repeated arm: volume 0
        3: exit_molecule({"chiral": _tables([(4, 1, 2, 3, 5)], [(1e6, 2e6)], 5, 2)}),
        5: exit_molecule({}, imp_const=True),  # energy 10 > 0.7
        6: exit_molecule({"dbGeom": _tables([(21, 22, 23)], np.zeros((1, 0)), 3, 0)}, linear=True),
        8: exit_molecule({"chiralDist": _tables([(0, 5)], [(40.0, 41.0)], 2, 2)}),
        9: exit_molecule({"chiral": _tables([(1, 1, 2, 3, 4)], [(0.0, 0.0)], 5, 2)}),  # centre on an arm: same-side 0
        10: exit_molecule({"dbStereo": _tables([(1, 2, 3, 1)], [1.0], 4, 1)}),  # i = l: dihedral 0, trans demanded
    }


def _oracle_embed(flat, slot_mol, params):
    return oracle.etkdg_embed((flat.dg.atom_counts, flat.dg.tables), (flat.etk.atom_counts, flat.etk.tables),
                              flat.checks.tables, flat.checks.num_impropers, params, list(slot_mol))


def _settle(fx, total):
    """Attempts allowed to end at stage 1. None for the plain molecule. The one with the straight triple carries three
    atoms held by nothing but their own terms: about one minimisation from a random start in a thousand (on the
    device, none seen in the oracle) settles above 0.05 per atom there, which the trajectory, not a check, decides."""
    return total // 100 if fx.n > 21 else 0


def _assert_exits_at(fails, stage, total, settle=0):
    """Every attempt failed, at `stage`, apart from at most `settle` at the energy test of stage 1."""
    early = 0 if stage == 1 else int(fails[1])
    assert fails.sum() == total and early <= settle, fails
    want = np.zeros(11, np.int64)
    want[1] = early
    want[stage] += total - early
    assert np.array_equal(fails, want), fails


def both_fixture(stages):
    """The tables of two always-failing stages on one molecule (the one with the straight triple when stage 6 is in)."""
    ex = exit_fixtures()
    first, second = (ex[s] for s in stages)
    fx = ex[6] if 6 in stages else first
    return Fixture("both", fx.n, dict(first.checks, **second.checks), [], 0, fx.dg, fx.etk)


@pytest.mark.parametrize("stage", [1, 2, 3, 5, 6, 8, 9, 10])
def test_oracle_pipeline_fails_every_attempt_at_its_stage(stage):
    flat = flat_of([exit_fixtures()[stage]])
    out, att, _e, fails = _oracle_embed(flat, [0] * 6, EXIT_PARAMS)
    assert all(o is None for o in out) and (att == EXIT_PARAMS["maxAttempts"]).all()
    _assert_exits_at(fails, stage, 6 * EXIT_PARAMS["maxAttempts"])


@pytest.mark.parametrize("stages", [(8, 10), (6, 8)], ids=["8+10", "6+8"])
def test_oracle_pipeline_counts_two_failing_stages_at_the_earlier(stages):
    out, _att, _e, fails = _oracle_embed(flat_of([both_fixture(stages)]), [0] * 6, EXIT_PARAMS)
    assert all(o is None for o in out)
    _assert_exits_at(fails, stages[0], 6 * EXIT_PARAMS["maxAttempts"])


# ------------------------------------------------------------------------------------------------ GPU: check kernel
def _check_masks_gpu(flat, slot_mol, pos4_list, params=PARAMS):
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.embedMolecules import EmbedParamsC

    dev = torch.device("cuda", 0)
    dg, _a = flat.dg.to_device(dev)
    etk, _b = flat.etk.to_device(dev)
    chk, _c = flat.checks.to_device(dev)
    pc = EmbedParamsC(**params)
    starts = np.concatenate([[0], np.cumsum([len(p) for p in pos4_list])]).astype(np.int32)
    d_pos = torch.from_numpy(np.concatenate(pos4_list)).to(dev)
    d_mol = torch.from_numpy(np.asarray(slot_mol, dtype=np.int32)).to(dev)
    d_st = torch.from_numpy(starts).to(dev)
    masks = torch.full((len(slot_mol),), -1, dtype=torch.int32, device=dev)
    _lib.call("b200mol_etkdg_check", C.byref(dg), C.byref(etk), C.byref(chk), C.byref(pc), len(slot_mol), d_mol.data_ptr(),
              d_st.data_ptr(), int(np.max(flat.atom_counts[np.asarray(slot_mol)])), d_pos.data_ptr(), masks.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    return masks.cpu().numpy().astype(np.uint32)


def _fixture_slots(fxs):
    slots = [(m, g) for m, fx in enumerate(fxs) for g in fx.geoms]
    return [m for m, _ in slots], [g.pos for _, g in slots], slots


@pytest.mark.gpu
@pytest.mark.parametrize("params", SWITCHES, ids=SWITCH_IDS)
def test_check_kernel_matches_oracle_and_verdicts(cuda, params):
    fxs = fixtures()
    flat = flat_of(fxs)
    slot_mol, pos, slots = _fixture_slots(fxs)
    got = _check_masks_gpu(flat, slot_mol, pos, params)
    for s, (m, g) in enumerate(slots):
        where = (fxs[m].name, g.label, bin(got[s]))
        assert got[s] == oracle_mask(flat, m, g.pos, params), where
        assert got[s] == switched(g.want, params), where


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["chiralDist", "tetrahedral"])
def test_check_kernel_finds_one_failing_term_anywhere_in_the_strided_loop(cuda, table):
    """520 terms (> 2 x 256 threads), all passing but one, placed at each edge of the per-thread loop: the verdict is
    the OR over the CTA (thread 0, a lane of the first warp, the first of the second warp, the last thread, the second
    trip of thread 0, the last term)."""
    n_terms, bit = 2 * KT + 8, {"chiralDist": CDIST, "tetrahedral": TET}[table]
    # atoms 0-4: a regular tetrahedron around atom 0 (passes), atoms 5-9: a flat one (fails); pair 0-1 at 1.73
    pos = p4(np.concatenate([[[0.0, 0, 0]], REG, [[0.0, 0, 0]], REG * [1, 1, 0]]))
    good = {"chiralDist": ((0, 1), (1.5, 2.0)), "tetrahedral": ((0, 1, 2, 3, 4), (0.0,))}[table]
    bad = {"chiralDist": ((0, 1), (5.0, 6.0)), "tetrahedral": ((5, 6, 7, 8, 9), (0.0,))}[table]
    k, p = {"chiralDist": (2, 2), "tetrahedral": (5, 1)}[table]
    fxs, wants = [], []
    for where in (0, 31, 32, KT - 1, KT, n_terms - 1, None):
        idx, par = [good[0]] * n_terms, [good[1]] * n_terms
        if where is not None:
            idx[where], par[where] = bad
        fxs.append(Fixture(f"fail at {where}", 10, {table: _tables(idx, par, k, p)}, [Geom("", pos, 0)]))
        wants.append(0 if where is None else bit)
    flat = flat_of(fxs)
    got = _check_masks_gpu(flat, list(range(len(fxs))), [pos] * len(fxs))
    for m in range(len(fxs)):
        assert got[m] == wants[m] == oracle_mask(flat, m, pos), (fxs[m].name, bin(got[m]))


def big_fixture(n=2000):
    """2000 atoms (4 n doubles = 64 KB of shared memory): fourth-dimension terms on every atom, and a tetrahedral row
    and a distance pair on the last atoms."""
    rng = np.random.default_rng(8)
    base = p4(rng.normal(0, 6.0, (n, 3)))
    base[n - 5:, :3] = np.concatenate([[[0.0, 0, 0]], REG]) + 50.0
    base[n - 7:n - 5, :3] = [[60.0, 0, 0], [60.0, 1.75, 0]]
    fx = Fixture("2000 atoms", n, {"tetrahedral": _tables([tuple(range(n - 5, n))], [0.0], 5, 1),
                                   "chiralDist": _tables([(n - 7, n - 6)], [(1.5, 2.0)], 2, 2)},
                 dg={"fourth": (np.arange(n).reshape(-1, 1), np.zeros((n, 0)))})
    ok = base.copy()
    ok[:, 3] = 0.7  # 0.1 * 0.49 per atom
    heavy = base.copy()
    heavy[:, 3] = 0.71  # 0.1 * 0.5041 per atom >= 0.05
    far = ok.copy()
    far[n - 6, :3] = [60.0, 5.0, 0]
    flat4 = ok.copy()
    flat4[n - 4:, 2] = 50.0
    fx.geoms = [Geom("fourth 0.7", ok, 0), Geom("fourth 0.71", heavy, ENERGY), Geom("last pair apart", far, CDIST),
                Geom("last centre flat", flat4, TET)]
    return fx


@pytest.mark.gpu
def test_check_kernel_batch_shapes(cuda):
    """More slots than the kernel's grid (4 x SMs), alternating by grid pass between a 2000-atom molecule and the small
    fixtures, so one CTA checks a small molecule right after a large one in the same shared memory; an empty molecule."""
    small = fixtures()
    big = big_fixture()
    fxs = small + [big]
    flat = flat_of(fxs)
    grid = 4 * torch.cuda.get_device_properties(0).multi_processor_count
    small_slots = [(m, g) for m, fx in enumerate(small) for g in fx.geoms]
    big_slots = [(len(small), g) for g in big.geoms]
    slots = []
    for s in range(2000):
        pool = big_slots if (s // grid) % 2 == 0 else small_slots
        slots.append(pool[(s * 7) % len(pool)])
    assert len(slots) > 3 * grid
    got = _check_masks_gpu(flat, [m for m, _ in slots], [g.pos for _, g in slots])
    memo = {}
    for s, (m, g) in enumerate(slots):
        if id(g) not in memo:
            memo[id(g)] = oracle_mask(flat, m, g.pos)
            assert memo[id(g)] == g.want, (fxs[m].name, g.label)
        assert got[s] == memo[id(g)], (s, fxs[m].name, g.label, bin(got[s]))
    # the large molecule alone (one CTA per slot) and the empty one alone
    got = _check_masks_gpu(flat, [len(small)] * len(big.geoms), [g.pos for g in big.geoms])
    assert [int(x) for x in got] == [g.want for g in big.geoms]
    empty = [m for m, fx in enumerate(small) if fx.name == "no tables"][0]
    assert _check_masks_gpu(flat, [empty], [small[empty].geoms[0].pos])[0] == 0


# ------------------------------------------------------------------------------------------------ GPU: attempt kernel
def _embed_gpu(flat, slot_mol, params):
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.embedMolecules import EmbedParamsC

    dev = torch.device("cuda", 0)
    dg, _a = flat.dg.to_device(dev)
    etk, _b = flat.etk.to_device(dev)
    chk, _c = flat.checks.to_device(dev)
    slot_mol = np.asarray(slot_mol, np.int32)
    starts = np.concatenate([[0], np.cumsum(flat.atom_counts[slot_mol])]).astype(np.int32)
    n = len(slot_mol)
    coords = torch.zeros((int(starts[-1]), 3), dtype=torch.float64, device=dev)
    ok = torch.full((n,), -1, dtype=torch.int8, device=dev)
    attempts = torch.full((n,), -1, dtype=torch.int32, device=dev)
    energy = torch.zeros(n, dtype=torch.float64, device=dev)
    fails = torch.full((11,), -1, dtype=torch.int64, device=dev)
    d_mol, d_st = torch.from_numpy(slot_mol).to(dev), torch.from_numpy(starts).to(dev)  # (alive until the kernel ends)
    _lib.call("b200mol_etkdg_embed", C.byref(dg), C.byref(etk), C.byref(chk), C.byref(EmbedParamsC(**params)), n,
              d_mol.data_ptr(), d_st.data_ptr(), int(flat.atom_counts[slot_mol].max()), coords.data_ptr(), ok.data_ptr(),
              attempts.data_ptr(), energy.data_ptr(), fails.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return (ok.cpu().numpy(), attempts.cpu().numpy(), fails.cpu().numpy(), coords.cpu().numpy(), starts)


def _n_ctas():
    """The embedder's grid at most: SMs x the resident CTAs per SM it allows itself (option bfgs_ctas_per_sm)."""
    from nvmolkit_b200 import _lib

    return _lib.get_option("bfgs_ctas_per_sm") * torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [1, 2, 3, 5, 6, 8, 9, 10])
def test_embed_ends_every_attempt_at_the_failing_stage(cuda, stage):
    """As many slots as the kernel has CTAs at most, so that CTAs run speculative attempts of other slots; then a
    small batch against the oracle's pipeline on the same random streams."""
    fx = exit_fixtures()[stage]
    flat = flat_of([fx])
    n_slots, a = _n_ctas(), EXIT_PARAMS["maxAttempts"]
    ok, att, fails, _x, _s = _embed_gpu(flat, [0] * n_slots, EXIT_PARAMS)
    assert (ok == 0).all() and (att == a).all()
    _assert_exits_at(fails, stage, n_slots * a, _settle(fx, n_slots * a))
    n_small = 16
    ok, att, fails, _x, _s = _embed_gpu(flat, [0] * n_small, EXIT_PARAMS)
    _out, cpu_att, _e, cpu_fails = _oracle_embed(flat, [0] * n_small, EXIT_PARAMS)
    assert (ok == 0).all() and np.array_equal(att, cpu_att)
    _assert_exits_at(cpu_fails, stage, n_small * a)
    _assert_exits_at(fails, stage, n_small * a, _settle(fx, n_small * a))
    if not _settle(fx, n_small * a):
        assert np.array_equal(fails, cpu_fails), (fails, cpu_fails)


@pytest.mark.gpu
@pytest.mark.parametrize("stages", [(8, 10), (6, 8)], ids=["8+10", "6+8"])
def test_embed_counts_two_failing_stages_at_the_earlier(cuda, stages):
    fx = both_fixture(stages)
    flat = flat_of([fx])
    n_slots, a = _n_ctas(), EXIT_PARAMS["maxAttempts"]
    ok, att, fails, _x, _s = _embed_gpu(flat, [0] * n_slots, EXIT_PARAMS)
    assert not ok.any()
    _assert_exits_at(fails, stages[0], n_slots * a, _settle(fx, n_slots * a))


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [3, 5, 8, 9, 10])
def test_embed_succeeds_with_the_owning_switch_off(cuda, stage):
    switch = "useBasicKnowledge" if stage == 5 else "enforceChirality"
    params = dict(EXIT_PARAMS, maxAttempts=10, **{switch: 0})
    flat = flat_of([exit_fixtures()[stage]])
    ok, att, fails, coords, starts = _embed_gpu(flat, [0] * 16, params)
    assert ok.all() and not fails[stage], (ok, fails)
    for s in np.nonzero(ok)[0]:
        x = coords[starts[s]:starts[s + 1]]
        mask = oracle_mask(flat, 0, p4(x), params)
        assert mask & 0b11111100000 == 0, (s, bin(mask))  # stages 5-10 hold on the accepted conformer
