"""CPU oracle — TEST INFRASTRUCTURE ONLY.

ctypes front-end to ``oracle/liboracle.so`` (plain-C restatements of the reference algorithms, see the header of each
``oracle_*.c``). Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline leg may import this
package; nothing under ``nvmolkit_b200/`` does.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (no GPU involved). Returns the library path."""
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.startswith("oracle_") and f.endswith(".c")]
    stale = (not os.path.exists(_LIB_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs)
    if force or stale:
        subprocess.run(["make", "-C", _HERE, "-s"] + (["-B"] if force else []), check=True)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _declare(_lib)
    return _lib


def set_threads(n: int = 0) -> int:
    """Use n OpenMP threads (0 = leave as is); returns the team size the library will use."""
    L = lib()
    L.oracle_set_threads.argtypes = [C.c_int]
    L.oracle_set_threads.restype = C.c_int
    return int(L.oracle_set_threads(int(n)))


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(C.POINTER(t))


def _declare(L: C.CDLL) -> None:
    u32p, i32p, f64p, u16p = C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_uint16)
    L.oracle_similarity_cross.argtypes = [u32p, C.c_long, u32p, C.c_long, C.c_int, C.c_int, f64p]
    L.oracle_similarity_cross.restype = None
    L.oracle_count_ge.argtypes = [u32p, C.c_long, u32p, C.c_long, C.c_int, C.c_int, C.c_double, C.c_int, i32p]
    L.oracle_count_ge.restype = None
    L.oracle_butina_dense.argtypes = [f64p, C.c_long, C.c_double, i32p, i32p]
    L.oracle_butina_dense.restype = C.c_int
    L.oracle_butina_fp.argtypes = [u32p, C.c_long, C.c_int, C.c_int, C.c_double, i32p, i32p]
    L.oracle_butina_fp.restype = C.c_int
    L.oracle_morgan_atom_invariant.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32, C.c_int]
    L.oracle_morgan_atom_invariant.restype = C.c_uint32
    L.oracle_morgan_one.argtypes = [C.c_int, C.c_int, u32p, u32p, u16p, u16p, C.c_int, C.c_int, u32p, u32p]
    L.oracle_morgan_one.restype = C.c_int
    L.oracle_morgan.argtypes = [i32p, i32p, u32p, u32p, u16p, u16p, C.c_long, C.c_int, C.c_int, u32p]
    L.oracle_morgan.restype = None
    L.oracle_recip_quotient_mismatches.argtypes = [C.c_int, C.c_int]
    L.oracle_recip_quotient_mismatches.restype = C.c_long
    for name, fn in _LATE_DECL.items():
        if hasattr(L, name):
            fn(getattr(L, name))


_LATE_DECL: dict = {}

METRIC = {"tanimoto": 0, "cosine": 1}


def _fp(a) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(a).view(np.uint32) if np.asarray(a).dtype == np.int32 else a, dtype=np.uint32)
    assert a.ndim == 2
    return a


# ------------------------------------------------------------------ path A
def similarity_cross(a, b=None, metric: str = "tanimoto") -> np.ndarray:
    a = _fp(a)
    b = a if b is None else _fp(b)
    out = np.empty((a.shape[0], b.shape[0]), dtype=np.float64)
    lib().oracle_similarity_cross(_p(a, C.c_uint32), a.shape[0], _p(b, C.c_uint32), b.shape[0], a.shape[1],
                                  METRIC[metric], _p(out, C.c_double))
    return out


def count_ge(x, y, cutoff: float, metric: str = "tanimoto", sign: int = 1, counts=None) -> np.ndarray:
    x, y = _fp(x), _fp(y)
    if counts is None:
        counts = np.zeros(x.shape[0], dtype=np.int32)
    lib().oracle_count_ge(_p(x, C.c_uint32), x.shape[0], _p(y, C.c_uint32), y.shape[0], x.shape[1], METRIC[metric],
                          float(cutoff), int(sign), _p(counts, C.c_int32))
    return counts


def recip_quotient_mismatches(umax: int, newton: bool = True) -> int:
    """Pairs 1 <= c <= u <= umax where the tensor tile's c / u = fma(fma(-q0, u, c), r, q0) (r = RN(1/u), q0 = RN(c r))
    is not the correctly rounded quotient; newton=False counts those of q0 alone."""
    return int(lib().oracle_recip_quotient_mismatches(int(umax), int(bool(newton))))


def butina_dense(dist, cutoff: float):
    dist = np.ascontiguousarray(dist, dtype=np.float64)
    n = dist.shape[0]
    ids = np.empty(n, dtype=np.int32)
    cen = np.empty(max(n, 1), dtype=np.int32)
    k = lib().oracle_butina_dense(_p(dist, C.c_double), n, float(cutoff), _p(ids, C.c_int32), _p(cen, C.c_int32))
    return ids, cen[:k].copy()


def butina_fp(fp, cutoff: float, metric: str = "tanimoto"):
    fp = _fp(fp)
    n = fp.shape[0]
    ids = np.empty(n, dtype=np.int32)
    cen = np.empty(max(n, 1), dtype=np.int32)
    k = lib().oracle_butina_fp(_p(fp, C.c_uint32), n, fp.shape[1], METRIC[metric], float(cutoff), _p(ids, C.c_int32),
                               _p(cen, C.c_int32))
    return ids, cen[:k].copy()


def morgan_atom_invariant(z, total_degree, total_hs, charge=0, delta_mass=0, in_ring=False) -> int:
    return int(lib().oracle_morgan_atom_invariant(z, total_degree, total_hs, charge, delta_mass, int(bool(in_ring))))


def morgan_codes(atom_inv, bond_inv, bond_a, bond_b, radius: int) -> np.ndarray:
    """Unfolded environment codes of one molecule (what RDKit's sparse fingerprint counts)."""
    atom_inv = np.ascontiguousarray(atom_inv, dtype=np.uint32)
    bond_inv = np.ascontiguousarray(bond_inv, dtype=np.uint32)
    bond_a = np.ascontiguousarray(bond_a, dtype=np.uint16)
    bond_b = np.ascontiguousarray(bond_b, dtype=np.uint16)
    codes = np.zeros((radius + 1) * max(len(atom_inv), 1), dtype=np.uint32)
    n = lib().oracle_morgan_one(len(atom_inv), len(bond_inv), _p(atom_inv, C.c_uint32), _p(bond_inv, C.c_uint32),
                                _p(bond_a, C.c_uint16), _p(bond_b, C.c_uint16), radius, 2048, None,
                                _p(codes, C.c_uint32))
    return codes[:n].copy()


def morgan(atom_starts, bond_starts, atom_inv, bond_inv, bond_a, bond_b, radius: int, fp_bits: int) -> np.ndarray:
    atom_starts = np.ascontiguousarray(atom_starts, dtype=np.int32)
    bond_starts = np.ascontiguousarray(bond_starts, dtype=np.int32)
    atom_inv = np.ascontiguousarray(atom_inv, dtype=np.uint32)
    bond_inv = np.ascontiguousarray(bond_inv, dtype=np.uint32)
    bond_a = np.ascontiguousarray(bond_a, dtype=np.uint16)
    bond_b = np.ascontiguousarray(bond_b, dtype=np.uint16)
    n = len(atom_starts) - 1
    out = np.zeros((n, fp_bits // 32), dtype=np.uint32)
    lib().oracle_morgan(_p(atom_starts, C.c_int32), _p(bond_starts, C.c_int32), _p(atom_inv, C.c_uint32),
                        _p(bond_inv, C.c_uint32), _p(bond_a, C.c_uint16), _p(bond_b, C.c_uint16), n, radius, fp_bits,
                        _p(out, C.c_uint32))
    return out


# ------------------------------------------------------------------ path B (force fields + BFGS)
class _TermTableC(C.Structure):
    _fields_ = [("starts", C.c_void_p), ("idx", C.c_void_p), ("par", C.c_void_p)]


_FF_LAYOUT = {
    "mmff": ("bond", "angle", "strbend", "oop", "torsion", "vdw", "ele", "distc", "posc", "anglec", "torsc"),
    "uff": ("bond", "angle", "torsion", "inversion", "vdw", "distc", "posc", "anglec", "torsc"),
    "dg": ("dist", "chiral", "fourth"),
    "etk": ("torsion", "improper", "dist12", "dist13", "angle13", "longrange"),
}


def _ff_struct(kind):
    fields = [("nMols", C.c_int32), ("atomCounts", C.c_void_p)] + [(n, _TermTableC) for n in _FF_LAYOUT[kind]]
    return type(f"Oracle{kind}System", (C.Structure,), {"_fields_": fields})


_FF_STRUCT = {k: _ff_struct(k) for k in _FF_LAYOUT}


def _host_system(kind: str, atom_counts: np.ndarray, tables: dict):
    """tables[name] = (starts int32, idx int16 [n,K], par float64 [n,P]); arrays must stay alive during the call."""
    st = _FF_STRUCT[kind]()
    st.nMols = len(atom_counts)
    st.atomCounts = atom_counts.ctypes.data
    keep = []
    for name in _FF_LAYOUT[kind]:
        if name not in tables:  # restraint tables are optional
            z = np.zeros(len(atom_counts) + 1, dtype=np.int32)
            keep.append(z)
            setattr(st, name, _TermTableC(z.ctypes.data, None, None))
            continue
        starts, idx, par = tables[name]
        setattr(st, name, _TermTableC(starts.ctypes.data, idx.ctypes.data, par.ctypes.data if par.size else None))
    st._keep = keep
    return st


def _declare_ff(L):
    vp, f64p, i32p, i8p = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_int8)
    L.oracle_mmff_energy_grad.argtypes = [vp, C.c_int, f64p, f64p, f64p]
    L.oracle_mmff_energy_grad.restype = C.c_double
    L.oracle_uff_energy_grad.argtypes = [vp, C.c_int, f64p, f64p]
    L.oracle_uff_energy_grad.restype = C.c_double
    L.oracle_uff_minimize.argtypes = [vp, C.c_int, i32p, i32p, f64p, C.c_int, C.c_double, f64p, i8p, i32p]
    L.oracle_uff_minimize.restype = None
    L.oracle_dg_energy_grad.argtypes = [vp, C.c_int, C.c_int, C.c_double, C.c_double, f64p, f64p]
    L.oracle_dg_energy_grad.restype = C.c_double
    L.oracle_etk_energy_grad.argtypes = [vp, C.c_int, f64p, f64p, C.c_int]
    L.oracle_etk_energy_grad.restype = C.c_double
    L.oracle_mmff_minimize.argtypes = [vp, C.c_int, i32p, i32p, f64p, C.c_int, C.c_double, f64p, i8p, i32p]
    L.oracle_mmff_minimize.restype = None
    L.oracle_dg_minimize.argtypes = [vp, C.c_int, C.c_double, C.c_double, C.c_int, i32p, i32p, f64p, C.c_int, C.c_double,
                                     f64p, i8p, i32p]
    L.oracle_dg_minimize.restype = None
    L.oracle_etk_minimize.argtypes = [vp, C.c_int, C.c_int, C.c_int, i32p, i32p, f64p, C.c_int, C.c_double, f64p, i8p, i32p]
    L.oracle_etk_energy_grad_ref.argtypes = [vp, C.c_int, f64p, f64p, C.c_int, f64p]
    L.oracle_etk_energy_grad_ref.restype = C.c_double
    L.oracle_etk_minimize.restype = None
    L.oracle_poly_minimize.argtypes = [C.c_int, C.c_int, f64p, f64p, f64p, C.c_int, C.c_double, C.c_int, f64p, i32p]
    L.oracle_poly_minimize.restype = C.c_int
    L.oracle_poly_energy_grad.argtypes = [C.c_int, C.c_int, f64p, f64p, f64p, f64p]
    L.oracle_poly_energy_grad.restype = C.c_double


_late_lib = [None]


def _ensure_ff():
    L = lib()
    if _late_lib[0] is None:
        _late_lib[0] = L
        _declare_ff(L)
    return L


def ff_energy_grad(kind: str, atom_counts, tables, mol: int, pos, want_grad=True, *, dim=0, chiral_weight=1.0,
                   fourth_dim_weight=0.1, plain=False, ref_pos=None):
    """Energy (and gradient) of one conformer of molecule `mol`. pos: float64 [nAtoms, dim]."""
    L = _ensure_ff()
    atom_counts = np.ascontiguousarray(atom_counts, dtype=np.int32)
    st = _host_system(kind, atom_counts, tables)
    pos = np.ascontiguousarray(pos, dtype=np.float64)
    grad = np.zeros_like(pos) if want_grad else None
    gp = _p(grad, C.c_double) if want_grad else None
    if kind == "mmff":
        per = np.zeros(7)
        e = L.oracle_mmff_energy_grad(C.addressof(st), mol, _p(pos, C.c_double), gp, _p(per, C.c_double))
        return e, grad, per
    if kind == "uff":
        return L.oracle_uff_energy_grad(C.addressof(st), mol, _p(pos, C.c_double), gp), grad, None
    if kind == "dg":
        e = L.oracle_dg_energy_grad(C.addressof(st), mol, dim or 4, chiral_weight, fourth_dim_weight, _p(pos, C.c_double), gp)
        return e, grad, None
    rp = None
    if ref_pos is not None:
        ref_pos = np.ascontiguousarray(ref_pos, dtype=np.float64)
        rp = _p(ref_pos, C.c_double)
    e = L.oracle_etk_energy_grad_ref(C.addressof(st), mol, _p(pos, C.c_double), gp, int(plain), rp)
    return e, grad, None


def ff_minimize(kind: str, atom_counts, tables, conf_mol, conf_atom_start, positions, max_iters=200, grad_tol=1e-4, *,
                dim=0, chiral_weight=1.0, fourth_dim_weight=0.1, plain=False, recentre=True):
    """RDKit-faithful BFGS on every conformer (OpenMP over conformers). Returns (positions, energies, converged, iters)."""
    L = _ensure_ff()
    atom_counts = np.ascontiguousarray(atom_counts, dtype=np.int32)
    st = _host_system(kind, atom_counts, tables)
    conf_mol = np.ascontiguousarray(conf_mol, dtype=np.int32)
    starts = np.ascontiguousarray(conf_atom_start, dtype=np.int32)
    pos = np.array(positions, dtype=np.float64, order="C", copy=True)
    n = len(conf_mol)
    e = np.zeros(n)
    conv = np.zeros(n, dtype=np.int8)
    iters = np.zeros(n, dtype=np.int32)
    a = (n, _p(conf_mol, C.c_int32), _p(starts, C.c_int32), _p(pos, C.c_double), int(max_iters), float(grad_tol),
         _p(e, C.c_double), _p(conv, C.c_int8), _p(iters, C.c_int32))
    if kind == "mmff":
        L.oracle_mmff_minimize(C.addressof(st), *a)
    elif kind == "uff":
        L.oracle_uff_minimize(C.addressof(st), *a)
    elif kind == "dg":
        L.oracle_dg_minimize(C.addressof(st), dim or 4, chiral_weight, fourth_dim_weight, *a)
    else:
        L.oracle_etk_minimize(C.addressof(st), int(plain), int(recentre), *a)
    return pos, e, conv, iters


def poly_minimize(power, w, c, x0, max_iters, grad_tol, scale_grads=False):
    L = _ensure_ff()
    w = np.ascontiguousarray(w, dtype=np.float64)
    c = np.ascontiguousarray(c, dtype=np.float64)
    x = np.array(x0, dtype=np.float64, copy=True)
    e = C.c_double(0)
    it = C.c_int32(0)
    st = L.oracle_poly_minimize(len(x), power, _p(w, C.c_double), _p(c, C.c_double), _p(x, C.c_double), max_iters,
                                grad_tol, int(scale_grads), C.byref(e), C.byref(it))
    return x, e.value, st, it.value


# ------------------------------------------------------------------ DG preparation + ETKDG
class _ChecksC(C.Structure):
    _fields_ = [(n, _TermTableC) for n in ("tetrahedral", "chiral", "chiralDist", "dbStereo", "dbGeom")] + \
               [("numImpropers", C.c_void_p)]


class _EmbedParamsC(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("boxSize", C.c_double), ("optimizerForceTol", C.c_double),
                ("enforceChirality", C.c_int32), ("useExpTorsions", C.c_int32), ("useBasicKnowledge", C.c_int32),
                ("maxAttempts", C.c_int32), ("dgIters", C.c_int32), ("fourthIters", C.c_int32), ("etkIters", C.c_int32),
                ("maxRestarts", C.c_int32), ("useMetricStart", C.c_int32)]


def _checks_struct(tables: dict, num_impropers: np.ndarray):
    st = _ChecksC()
    for name in ("tetrahedral", "chiral", "chiralDist", "dbStereo", "dbGeom"):
        starts, idx, par = tables[name]
        setattr(st, name, _TermTableC(starts.ctypes.data, idx.ctypes.data, par.ctypes.data if par.size else None))
    st.numImpropers = num_impropers.ctypes.data
    return st


def _embed_params(p: dict):
    return _EmbedParamsC(**p)


def triangle_smooth(bounds: np.ndarray, tol: float = 0.0):
    """In-place smoothing of one RDKit-layout bounds matrix copy. Returns (matrix, ok)."""
    L = lib()
    b = np.array(bounds, dtype=np.float64, order="C", copy=True)
    L.oracle_triangle_smooth.restype = C.c_int
    ok = L.oracle_triangle_smooth(b.ctypes.data_as(C.c_void_p), C.c_int(b.shape[0]), C.c_double(tol))
    return b, bool(ok)


def power_eigen(mat: np.ndarray, num_eigs: int, v0: np.ndarray):
    L = lib()
    m = np.array(mat, dtype=np.float64, order="C", copy=True)
    n = m.shape[0]
    v0 = np.ascontiguousarray(v0, dtype=np.float64)
    vals = np.zeros(num_eigs)
    vecs = np.zeros((num_eigs, n))
    L.oracle_power_eigen.restype = C.c_int
    k = L.oracle_power_eigen(m.ctypes.data_as(C.c_void_p), C.c_int(n), C.c_int(num_eigs), v0.ctypes.data_as(C.c_void_p),
                             vals.ctypes.data_as(C.c_void_p), vecs.ctypes.data_as(C.c_void_p))
    return vals, vecs, k


def metric_embed(dist: np.ndarray, dim: int, v0: np.ndarray):
    """Distance matrix -> coordinates [n, dim] (or None when an eigenvalue is not positive)."""
    L = lib()
    d = np.ascontiguousarray(dist, dtype=np.float64)
    n = d.shape[0]
    T = np.zeros((n, n))
    L.oracle_metric_matrix(d.ctypes.data_as(C.c_void_p), C.c_int(n), T.ctypes.data_as(C.c_void_p))
    vals, vecs, k = power_eigen(T, dim, v0)
    if k < dim:
        return None
    coords = np.zeros((n, dim))
    L.oracle_coords_from_eigen.restype = C.c_int
    ok = L.oracle_coords_from_eigen(vals.ctypes.data_as(C.c_void_p), vecs.ctypes.data_as(C.c_void_p), C.c_int(n), C.c_int(dim),
                                    coords.ctypes.data_as(C.c_void_p))
    return coords if ok else None


def etkdg_check(dg, etk, checks, num_impropers, params: dict, mol: int, pos4: np.ndarray) -> int:
    """dg / etk = (atom_counts, tables); checks = tables dict. Returns the failure bit mask of include/b200mol.h."""
    L = _ensure_ff()
    d = _host_system("dg", np.ascontiguousarray(dg[0], dtype=np.int32), dg[1])
    e = _host_system("etk", np.ascontiguousarray(etk[0], dtype=np.int32), etk[1])
    ck = _checks_struct(checks, np.ascontiguousarray(num_impropers, dtype=np.int32))
    pr = _embed_params(params)
    pos4 = np.ascontiguousarray(pos4, dtype=np.float64)
    L.oracle_etkdg_check.restype = C.c_uint
    L.oracle_etkdg_check.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_void_p]
    return int(L.oracle_etkdg_check(C.addressof(d), C.addressof(e), C.addressof(ck), C.addressof(pr), mol, pos4.ctypes.data))


def etkdg_embed(dg, etk, checks, num_impropers, params: dict, slot_mol):
    """CPU pipeline over slots (serial). Returns (list of coords3 | None, attempts, energies, stage failure counts[11])."""
    L = _ensure_ff()
    counts = np.ascontiguousarray(dg[0], dtype=np.int32)
    d = _host_system("dg", counts, dg[1])
    e = _host_system("etk", np.ascontiguousarray(etk[0], dtype=np.int32), etk[1])
    nimp = np.ascontiguousarray(num_impropers, dtype=np.int32)
    ck = _checks_struct(checks, nimp)
    pr = _embed_params(params)
    L.oracle_etkdg_embed_one.restype = C.c_int
    L.oracle_etkdg_embed_one.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    fails = np.zeros(11, dtype=np.int64)
    out, attempts, energies = [], [], []
    for slot, mol in enumerate(slot_mol):
        xyz = np.zeros((counts[mol], 3))
        att = C.c_int32(0)
        en = C.c_double(0.0)
        ok = L.oracle_etkdg_embed_one(C.addressof(d), C.addressof(e), C.addressof(ck), C.addressof(pr), slot, int(mol),
                                      xyz.ctypes.data, C.addressof(att), C.addressof(en), fails.ctypes.data)
        out.append(xyz if ok else None)
        attempts.append(att.value)
        energies.append(en.value)
    return out, np.array(attempts), np.array(energies), fails


def etkdg_initial_coords(dg, params: dict, slot: int, mol: int, attempt: int):
    """Stage 0 of one attempt: (pos4 [nAtoms, 4], ok)."""
    L = _ensure_ff()
    d = _host_system("dg", np.ascontiguousarray(dg[0], dtype=np.int32), dg[1])
    pr = _embed_params(params)
    n = int(np.asarray(dg[0])[mol])
    pos = np.zeros((n, 4))
    L.oracle_etkdg_initial_coords.restype = C.c_int
    L.oracle_etkdg_initial_coords.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    ok = L.oracle_etkdg_initial_coords(C.addressof(d), C.addressof(pr), int(slot), int(mol), int(attempt), pos.ctypes.data)
    return pos, bool(ok)


def uniform01(seed: int, slot: int, attempt: int, element: int) -> float:
    L = lib()
    L.oracle_uniform01.restype = C.c_double
    L.oracle_uniform01.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32]
    return float(L.oracle_uniform01(seed, slot, attempt, element))


def etkdg_embed_batch(dg, etk, checks, num_impropers, params: dict, slot_mol, slot_atom_start):
    """OpenMP CPU pipeline over all slots. Returns (coords3 [totalAtoms,3], ok int8, attempts, energies)."""
    L = _ensure_ff()
    counts = np.ascontiguousarray(dg[0], dtype=np.int32)
    d = _host_system("dg", counts, dg[1])
    e = _host_system("etk", np.ascontiguousarray(etk[0], dtype=np.int32), etk[1])
    nimp = np.ascontiguousarray(num_impropers, dtype=np.int32)
    ck = _checks_struct(checks, nimp)
    pr = _embed_params(params)
    slot_mol = np.ascontiguousarray(slot_mol, dtype=np.int32)
    starts = np.ascontiguousarray(slot_atom_start, dtype=np.int32)
    n = len(slot_mol)
    coords = np.zeros((int(starts[-1]), 3))
    ok = np.zeros(n, dtype=np.int8)
    att = np.zeros(n, dtype=np.int32)
    en = np.zeros(n)
    L.oracle_etkdg_embed_batch.restype = None
    L.oracle_etkdg_embed_batch.argtypes = [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 6
    L.oracle_etkdg_embed_batch(C.addressof(d), C.addressof(e), C.addressof(ck), C.addressof(pr), n, slot_mol.ctypes.data,
                               starts.ctypes.data, coords.ctypes.data, ok.ctypes.data, att.ctypes.data, en.ctypes.data)
    return coords, ok, att, en


# ------------------------------------------------------------------------------------------------ term construction
def dg_dist_terms(bounds: np.ndarray, basin: float = 1e8):
    """(idx [n,2] int32 with i > j, par [n,3] = lb^2, ub^2, weight) — oracle_build.c oracle_dg_dist_terms."""
    L = lib()
    b = np.ascontiguousarray(bounds, np.float64)
    n = b.shape[0]
    idx = np.empty((n * (n - 1) // 2, 2), np.int32)
    par = np.empty((n * (n - 1) // 2, 3))
    L.oracle_dg_dist_terms.restype = C.c_int
    L.oracle_dg_dist_terms.argtypes = [C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
    k = L.oracle_dg_dist_terms(n, b.ctypes.data, float(basin), idx.ctypes.data, par.ctypes.data)
    return idx[:k], par[:k]


def inversion_coefficients(z: int, c_bound_to_o: bool):
    """(k / 3, C0, C1, C2) of an improper centre of atomic number z."""
    L = lib()
    out = (C.c_double * 4)()
    L.oracle_inversion_coefficients.restype = None
    L.oracle_inversion_coefficients.argtypes = [C.c_int, C.c_int, C.c_void_p]
    L.oracle_inversion_coefficients(int(z), 1 if c_bound_to_o else 0, out)
    return tuple(out)


def etk_terms(bounds, torsion_atoms, improper_atoms, bond_atoms, angle_atoms, scaling: float, basic: bool):
    """ETK tables other than the torsions (which are copied through) as dict name -> (idx int32, par)."""
    L = lib()
    b = np.ascontiguousarray(bounds, np.float64)
    n = b.shape[0]
    ta = np.ascontiguousarray(torsion_atoms, np.int32).reshape(-1, 4)
    ia = np.ascontiguousarray(improper_atoms, np.int32).reshape(-1, 6)
    ba = np.ascontiguousarray(bond_atoms, np.int32).reshape(-1, 2)
    aa = np.ascontiguousarray(angle_atoms, np.int32).reshape(-1, 4)
    npair = n * (n - 1) // 2
    imp_i, imp_p = np.empty((3 * len(ia), 4), np.int32), np.empty((3 * len(ia), 4))
    d12_p = np.empty((len(ba), 4))
    d13_i, d13_p = np.empty((len(aa), 2), np.int32), np.empty((len(aa), 4))
    a13_i, a13_p = np.empty((len(aa), 3), np.int32), np.empty((len(aa), 2))
    lr_i, lr_p = np.empty((npair, 2), np.int32), np.empty((npair, 3))
    counts = (C.c_int32 * 5)()
    L.oracle_etk_terms.restype = None
    L.oracle_etk_terms.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                   C.c_void_p, C.c_double, C.c_int] + [C.c_void_p] * 10
    L.oracle_etk_terms(n, b.ctypes.data, len(ta), ta.ctypes.data, len(ia), ia.ctypes.data, len(ba), ba.ctypes.data, len(aa),
                       aa.ctypes.data, float(scaling), 1 if basic else 0, imp_i.ctypes.data, imp_p.ctypes.data,
                       d12_p.ctypes.data, d13_i.ctypes.data, d13_p.ctypes.data, a13_i.ctypes.data, a13_p.ctypes.data,
                       lr_i.ctypes.data, lr_p.ctypes.data, counts)
    return {"improper": (imp_i[: counts[0]], imp_p[: counts[0]]), "dist12": (ba.copy(), d12_p),
            "dist13": (d13_i[: counts[1]], d13_p[: counts[1]]), "angle13": (a13_i[: counts[2]], a13_p[: counts[2]]),
            "longrange": (lr_i[: counts[3]], lr_p[: counts[3]])}, int(counts[4])


# ------------------------------------------------------------------------------------------------ conformer pruning
def best_ssd(a: np.ndarray, b: np.ndarray) -> float:
    """Best-alignment sum of squared deviations of two [n, 3] point sets (Horn quaternion eigenproblem, oracle_prune.c)."""
    L = lib()
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    L.oracle_best_ssd.restype = C.c_double
    L.oracle_best_ssd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    return float(L.oracle_best_ssd(a.ctypes.data, None, b.ctypes.data, None, len(a)))


def rms_prune(xyz, conf_atom_start, mol_conf_start, thresh, matches=None, valid=None) -> np.ndarray:
    """keep flags [nConf]; matches[m] = [K, L] index array or None (all atoms)."""
    L = lib()
    xyz = np.ascontiguousarray(xyz, np.float64)
    cas = np.ascontiguousarray(conf_atom_start, np.int32)
    keep = np.zeros(len(cas) - 1, dtype=np.uint8)
    v = np.ascontiguousarray(valid, np.uint8) if valid is not None else None
    L.oracle_rms_prune_mol.restype = None
    L.oracle_rms_prune_mol.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_double,
                                       C.c_void_p, C.c_void_p]
    for m in range(len(mol_conf_start) - 1):
        c0, c1 = int(mol_conf_start[m]), int(mol_conf_start[m + 1])
        if c1 <= c0:
            continue
        mt = None if matches is None or matches[m] is None else np.ascontiguousarray(matches[m], np.int16)
        k, ln = (1, int(cas[c0 + 1] - cas[c0])) if mt is None else mt.shape
        L.oracle_rms_prune_mol(c0, c1, cas.ctypes.data, xyz.ctypes.data, int(k), int(ln), mt.ctypes.data if mt is not None else None,
                               float(thresh), v.ctypes.data if v is not None else None, keep.ctypes.data)
    return keep
