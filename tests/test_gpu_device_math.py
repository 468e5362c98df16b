"""The engine's device math, routine by routine, against 50-digit references (mpmath) and the oracle's taps.

tests/cuda/device_math.cu runs the routines of the csrc headers unchanged (same NVFLAGS as the library, so the same
FMA contraction) on batches of cases; every check here is one of
  (a) truth   — the operation restated in mpmath at 50 digits on the same fp64 inputs, error within a bound that
                follows from the routine's conditioning (table below);
  (b) oracle  — the oracle's tap on the same inputs (the parity the end-to-end tests rely on);
  (c) paths   — the two device paths of one operation (fast eigen-solver vs Jacobi, register vs compact solve).
Each regime prints its worst error / bound ratio; every assertion is ratio <= 1.

u = 2^-53. Bounds (c = 64 unless stated; c covers the O(10) roundings of each closed form, with headroom 4x):

| routine                         | quantity                 | bound                                                       |
|---------------------------------|--------------------------|-------------------------------------------------------------|
| sym_eig3_fast / _full on C      | |sv_k - lambda_k|        | c u lambda_1 (Weyl; both are backward stable: see below)    |
|                                 | sin angle(normal, v_3)   | c u lambda_1 / (lambda_2 - lambda_3) (Davis-Kahan)          |
| describe_*_from_sums (moments)  | |C_dev - C|              | E = c u (lambda_1 + |mu|^2): one-pass moments about the     |
|                                 |                          |   query lose the digits of |mu|^2 (mu = centroid - query)   |
|                                 | eigenvalues / normal     | as above with c u lambda_1 -> E                             |
|                                 | a2D                      | [dsq(s2) + dsq(s3)] / sqrt(s1) + a2D (E / s1 + 4u), with    |
|                                 |                          |   dsq(s) = min(sqrt(E), E / (2 sqrt(s))) (sqrt near 0)      |
| warp_ldlt_solve12(_compact)     | |D (x - x*)|_inf         | 3 n^2 sqrt(n) u kappa_2(M) |D x*|_inf, M = D^-1 A D^-1,     |
|                                 |                          |   D = sqrt(diag A): elimination without pivoting on an SPD  |
|                                 |                          |   matrix is backward stable with |L||U| <= n |A| (Higham    |
|                                 |                          |   10.1) and invariant under the diagonal scaling            |
|                                 | null coordinates         | exactly 0 (Eigen: pseudo-inverse of D)                      |
| warp_gn_solve                   | system (mode 1)          | 2 u |entry| (one rounding each; FMA may merge two)          |
|                                 | step x                   | the solve's bound                                           |
|                                 | pose after the step      | |dx| bound + c u (Euler / quaternion closed forms)           |
| ct_residual (duals)             | value, 12 partials       | c u S (1 + 1/theta^2): S = scale of the functor's terms,    |
|                                 |                          |   theta = acos|q_b . q_e|; dacos divides by                 |
|                                 |                          |   sqrt(1 - d^2) = sin(theta) formed from 1 - d^2, whose     |
|                                 |                          |   absolute error u becomes u / theta^2 relative             |
| quat_plus, qslerp_c, qfromR ... | components               | c u                                                         |
| loss_evaluate, corrector_1d     | rho[k], scales           | c u |value| (+ the published formula's conditioning)        |

Assumptions the bounds rest on: libdevice's acos, sin, cos, exp, log, cosh are within 2 ulp and sqrt / rsqrt within
1 ulp (CUDA C Programming Guide, "Mathematical functions", double precision table); the Jacobi solver converges in
its 12 sweeps (off-diagonal mass below 1e-32 of the diagonal's); the fast eigen-solver returns only what its residual
check accepts, and that check bounds the normal's error; its eigenvalues come from the trigonometric formula, which
hands a matrix with two coincident largest eigenvalues (half_det within 1e-4 of -1) to the Jacobi solver, because there
acos turns the rounding of half_det into a sqrt(u) error of the pair (regime "disc_exact" found it).
"""
import ctypes as C
import math
import os

import mpmath
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from ct_icp_b200 import _abi as abi

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
CC = 64.0
DPS = 50
_HERE = os.path.dirname(os.path.abspath(__file__))
HARNESS = os.environ.get("CTICP_DEVICE_MATH_LIB") or os.path.join(_HERE, "cuda", "libcticp_device_math.so")


# ------------------------------------------------------------------------------------------------ plumbing
class Harness:
    def __init__(self, path):
        self.lib = C.CDLL(path)

    def call(self, name, *args):
        conv = []
        for a in args:
            if isinstance(a, np.ndarray):
                assert a.flags["C_CONTIGUOUS"]
                conv.append(a.ctypes.data_as(C.c_void_p))
            elif isinstance(a, float):
                conv.append(C.c_double(a))
            else:
                conv.append(C.c_int(a))
        rc = getattr(self.lib, "dm_" + name)(*conv)
        assert rc == 0, "dm_%s: CUDA error %d" % (name, rc)

    def eig(self, full, a6):
        a6 = np.ascontiguousarray(a6, dtype=np.float64)
        out = np.zeros((len(a6), 12))
        self.call("sym_eig3", int(full), len(a6), a6, out)
        return out

    def describe(self, full, n, rel):
        n = np.ascontiguousarray(n, dtype=np.int32)
        rel = np.ascontiguousarray(rel, dtype=np.float64)
        out = np.zeros((len(n), 16))
        self.call("describe", int(full), len(n), n, rel, out)
        return out

    def solve(self, compact, A, b):
        A, b = np.ascontiguousarray(A, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
        x = np.zeros((len(A), 12))
        self.call("ldlt_solve12", int(compact), len(A), A, b, x)
        return x

    def gn(self, mode, acc, state, threshold):
        acc, state = np.ascontiguousarray(acc, dtype=np.float64), np.ascontiguousarray(state, dtype=np.float64)
        out, sys = np.zeros((len(acc), 40)), np.zeros((len(acc), 157))
        self.call("gn_solve", int(mode), len(acc), acc, state, float(threshold), out, sys)
        return out, sys

    def residual(self, robust, blk, kind, x):
        blk, x = np.ascontiguousarray(blk, dtype=np.float64), np.ascontiguousarray(x, dtype=np.float64)
        kind = np.ascontiguousarray(kind, dtype=np.int32)
        out = np.zeros((len(blk), 13))
        self.call("ct_residual", int(robust), len(blk), blk, kind, x, out)
        return out

    def dq_dot(self, x):
        x = np.ascontiguousarray(x, dtype=np.float64)
        out = np.zeros(len(x))
        self.call("dq_dot", len(x), x, out)
        return out

    def simple(self, name, width_out, *arrays, extra=()):
        arrays = [np.ascontiguousarray(a) for a in arrays]
        B = len(arrays[0])
        out = np.zeros((B, width_out) if width_out > 1 else B, dtype=np.int32 if name == "voxel_coord_rcp" else np.float64)
        self.call(name, B, *arrays, *extra, out)
        return out


@pytest.fixture(scope="module")
def dm():
    if not os.path.exists(HARNESS):
        pytest.fail("%s is missing: __graft_entry__.build() builds it (csrc/Makefile target device_math)" % HARNESS)
    return Harness(HARNESS)


def report(regime, ratio, extra=""):
    print("[device-math] %-40s worst error/bound = %.3g %s" % (regime, ratio, extra))
    assert ratio <= 1.0, (regime, ratio, extra)


def P(a):
    return a.ctypes.data_as(C.c_void_p)


RNG_SEED = 20261016


def rand_rot(rng, n):
    return Rotation.from_quat(rng.normal(size=(n, 4))).as_matrix()


def mpf(x):
    return mpmath.mpf(float(x))


# ------------------------------------------------------------------------------------------------ eigen / describe
def _points(kind, n, rng, B):
    """B neighbourhoods of n offsets from the query (fp64), shaped by `kind`; returns (n per case, rel[B, 32, 3])."""
    rel = np.zeros((B, 32, 3))
    ns = np.full(B, n, dtype=np.int32)
    for i in range(B):
        z = rng.normal(size=(n, 3))
        if kind.startswith("plane"):
            ratio = float(kind.split("_")[1])
            sig = np.array([0.4, 0.25, 0.4 * math.sqrt(ratio)])
            if ratio == 0.0:
                z[:, 2] = 0.0
            p = z * sig
            if kind.endswith("rot"):
                p = p @ rand_rot(rng, 1)[0].T
            else:   # axis-aligned, exactly planar fp32 points: z = const within the neighbourhood
                p = p.astype(np.float32).astype(np.float64)
                p[:, 2] = 0.0 if ratio == 0.0 else p[:, 2]
        elif kind == "line":
            p = np.outer(z[:, 0], rand_rot(rng, 1)[0][:, 0]) * 0.5
        elif kind == "disc":
            z[:, 2] = 0.0
            p = (z * np.array([0.3, 0.3, 0.0])) @ rand_rot(rng, 1)[0].T
        elif kind == "iso":
            p = z * 0.3
        elif kind == "offset_centroid":   # centimetre spread, centroid up to the 1 m search radius away from the query
            c = rng.normal(size=3)
            c *= rng.uniform(0.2, 1.0) / np.linalg.norm(c)
            p = c + 0.01 * z * np.array([1.0, 1.0, 0.05])
        else:
            raise ValueError(kind)
        rel[i, :n] = p
    return ns, rel


def _mp_cov(pts):
    n = len(pts)
    P_ = [[mpf(v) for v in row] for row in pts]
    mu = [sum(P_[k][d] for k in range(n)) / n for d in range(3)]
    Cm = mpmath.matrix(3, 3)
    for a in range(3):
        for b in range(3):
            Cm[a, b] = sum((P_[k][a] - mu[a]) * (P_[k][b] - mu[b]) for k in range(n)) / n
    return Cm, mu


def _mp_eig(Cm):
    E, Q = mpmath.eigsy(Cm)
    order = sorted(range(3), key=lambda k: -abs(E[k]))
    lam = [abs(E[k]) for k in order]
    vec = [[Q[r, k] for r in range(3)] for k in order]
    return lam, vec


def _sin_angle(v, w):
    """sin of the angle between two lines, from the cross product (accurate for tiny angles, unlike sqrt(1 - cos^2))"""
    v = np.asarray(v, dtype=float)
    w = np.array([float(t) for t in w])
    return float(np.linalg.norm(np.cross(v, w)) / (np.linalg.norm(v) * np.linalg.norm(w)))


def _a6(Cm):
    return [Cm[0, 0], Cm[0, 1], Cm[0, 2], Cm[1, 1], Cm[1, 2], Cm[2, 2]]


DESCRIBE_REGIMES = ["plane_1e-2_rot", "plane_1e-6_rot", "plane_1e-10_rot", "plane_1e-14_rot", "plane_0_rot",
                    "plane_1e-2_axis", "plane_1e-6_axis", "plane_1e-10_axis", "plane_1e-14_axis", "plane_0_axis",
                    "line", "disc", "iso", "offset_centroid"]


@pytest.mark.parametrize("kind", DESCRIBE_REGIMES)
def test_describe_and_eigen(dm, orc, kind):
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + sum(map(ord, kind)))
    ns, rel = [], []
    for n in (5, 6, 20, 32):
        a, b = _points(kind, n, rng, 50)
        ns.append(a); rel.append(b)
    ns, rel = np.concatenate(ns), np.concatenate(rel)
    fast = dm.describe(False, ns, rel)
    full = dm.describe(True, ns, rel)
    # the device's own covariance through both eigen-solvers
    a6 = np.ascontiguousarray(full[:, :6])
    e_fast, e_full = dm.eig(False, a6), dm.eig(True, a6)
    f_svd = orc.lib.orc_symmetric_svd3
    f_desc = orc.lib.orc_neighborhood_describe
    w = {"cov": 0, "sv": 0, "normal": 0, "a2D": 0, "svd_sv": 0, "svd_normal": 0, "oracle_normal": 0, "oracle_a2D": 0}
    fast_path = 0
    for i in range(len(ns)):
        n = int(ns[i])
        pts = rel[i, :n]
        Cm, mu = _mp_cov(pts)
        lam, vec = _mp_eig(Cm)
        l1, l2, l3 = (float(t) for t in lam)
        mu2 = float(sum(m * m for m in mu))
        E = CC * U * (l1 + mu2)
        # (a) covariance from the moments
        dC = max(abs(float(full[i, k] - c)) for k, c in enumerate(_a6(Cm)))
        w["cov"] = max(w["cov"], dC / E)
        # (a) eigen on the device's covariance: truth = eigsy of exactly that matrix
        Cd = mpmath.matrix([[full[i, 0], full[i, 1], full[i, 2]], [full[i, 1], full[i, 3], full[i, 4]],
                            [full[i, 2], full[i, 4], full[i, 5]]])
        dlam, dvec = _mp_eig(Cd)
        d1, d2, d3 = (float(t) for t in dlam)
        for out in (e_fast[i], e_full[i]):
            err = max(abs(out[k] - float(dlam[k])) for k in range(3))
            w["sv"] = max(w["sv"], err / (CC * U * d1) if d1 > 0 else (0.0 if err == 0 else np.inf))
            if d2 - d3 > CC * U * d1:   # otherwise the normal is not determined by the matrix (a line)
                w["normal"] = max(w["normal"], _sin_angle(out[3:6], dvec[2]) / (CC * U * d1 / (d2 - d3)))
        same = np.array_equal(e_fast[i, :6], e_full[i, :6])
        fast_path += not same
        # (a) describe_from_sums against the exact covariance of the offsets
        if l2 - l3 > 2 * E:
            w["normal"] = max(w["normal"], _sin_angle(fast[i, :3], vec[2]) / (2 * E / (l2 - l3)))
        if l1 > 0:
            a2 = (math.sqrt(l2) - math.sqrt(l3)) / math.sqrt(l1)
            def dsq(s):
                return min(math.sqrt(2 * E), 2 * E / (2 * math.sqrt(s))) if s > 0 else math.sqrt(2 * E)
            bound = (dsq(l2) + dsq(l3)) / math.sqrt(l1) + a2 * (2 * E / l1 + 4 * U)
            w["a2D"] = max(w["a2D"], abs(fast[i, 3] - a2) / bound)
        # (b) the oracle: SymmetricSVD3 on the same matrix, ComputeNeighborhood on the same points
        sv, V = np.zeros(3), np.zeros(9)
        f_svd(P(np.ascontiguousarray(_np3(full[i]))), P(sv), P(V))
        w["svd_sv"] = max(w["svd_sv"], np.abs(sv - e_full[i, :3]).max() / (2 * CC * U * max(d1, 1e-300)))
        if d2 - d3 > 2 * CC * U * d1:
            w["svd_normal"] = max(w["svd_normal"], _sin_angle(V.reshape(3, 3)[:, 2], e_fast[i, 3:6]) /
                                  (2 * CC * U * d1 / (d2 - d3)))
        on, oa = np.zeros(3), C.c_double()
        pl, li = C.c_double(), C.c_double()
        ok = f_desc(P(np.ascontiguousarray(pts)), C.c_size_t(n), P(on), C.byref(oa), C.byref(pl), C.byref(li), None)
        if ok and l2 - l3 > 4 * E:
            # the oracle's covariance is the uncentred world form: its own error is of the same kind as E
            w["oracle_normal"] = max(w["oracle_normal"], _sin_angle(on, fast[i, :3]) / (4 * E / (l2 - l3)))
            if l1 > 0:
                w["oracle_a2D"] = max(w["oracle_a2D"], abs(oa.value - fast[i, 3]) / (2 * bound))
    for k, v in w.items():
        report("%s / %s" % (kind, k), v)
    print("[device-math] %-40s fast path taken by %d of %d" % (kind, fast_path, len(ns)))
    if kind in ("plane_1e-2_rot", "plane_1e-6_rot", "offset_centroid"):
        assert fast_path > 0.9 * len(ns)   # well-separated regimes take the closed form


def _np3(r):
    return np.array([[r[0], r[1], r[2]], [r[1], r[3], r[4]], [r[2], r[4], r[5]]])


def _rand_spd_eig(rng, lam):
    Q = rand_rot(rng, 1)[0]
    Cm = Q @ np.diag(lam) @ Q.T
    return [Cm[0, 0], 0.5 * (Cm[0, 1] + Cm[1, 0]), 0.5 * (Cm[0, 2] + Cm[2, 0]), Cm[1, 1],
            0.5 * (Cm[1, 2] + Cm[2, 1]), Cm[2, 2]]


FALLBACKS = {
    # regime: (matrices, expected: True = the fallback (Jacobi) result, False = the closed form)
    "mx_zero": True,          # the zero matrix
    "nrm_zero": True,         # diagonal matrices: off-diagonals exactly 0
    "dm_zero": True,          # v [[1,1,0],[1,1,0],[0,0,0]]: e0 = 0 exactly, rows of A - e0 I parallel
    "verify_fail": True,      # lines: double eigenvalue at the bottom, the trigonometric e0 is off by ~sqrt(u)
    "v1_lt_v2": True,         # indefinite: |e0| is not the smallest |eigenvalue|
    "separated": False,       # eigenvalues 1 : 0.3 : 0.01, rotated
    "disc_exact": True,       # eigenvalues 1 : 1 : 0.01, rotated: double eigenvalue at the top, half_det at -1
}


def _fallback_inputs(regime, rng, B):
    out = []
    for _ in range(B):
        if regime == "mx_zero":
            out.append([0.0] * 6)
        elif regime == "nrm_zero":
            d = rng.uniform(0.01, 1.0, size=3)
            out.append([d[0], 0.0, 0.0, d[1], 0.0, d[2]])
        elif regime == "dm_zero":
            v = float(rng.uniform(0.01, 1.0))
            m = [v, v, 0.0, v, 0.0, 0.0]
            out.append([m[0], m[1], m[2], m[3], m[4], m[5]])
        elif regime == "verify_fail":
            out.append(_rand_spd_eig(rng, [rng.uniform(0.1, 1.0), 0.0, 0.0]))
        elif regime == "disc_exact":
            out.append(_rand_spd_eig(rng, [1.0, 1.0, 0.01]))
        elif regime == "v1_lt_v2":
            out.append(_rand_spd_eig(rng, [1.0, 0.5, -2.0]))
        else:
            out.append(_rand_spd_eig(rng, [1.0, 0.3, 0.01]))
    return np.array(out)


@pytest.mark.parametrize("regime", list(FALLBACKS))
def test_sym_eig3_fast_fallbacks(dm, orc, regime):
    """A fallback of sym_eig3_fast returns exactly what sym_eig3 (Jacobi) returns: bit identity with the harness's
    sym_eig3_full result marks it. Each regime meant to reach a fallback must reach it for most inputs; the truth bound
    holds either way."""
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + len(regime))
    a6 = _fallback_inputs(regime, rng, 300)
    f, j = dm.eig(False, a6), dm.eig(True, a6)
    same = np.array([np.array_equal(f[i, :6], j[i, :6]) for i in range(len(a6))])
    worst = 0.0
    for i in range(len(a6)):
        lam, vec = _mp_eig(mpmath.matrix(_np3(a6[i]).tolist()))
        l1, l2, l3 = (float(t) for t in lam)
        err = max(abs(f[i, k] - float(lam[k])) for k in range(3))
        worst = max(worst, err / (CC * U * l1) if l1 > 0 else (0.0 if err == 0 else np.inf))
        if l2 - l3 > CC * U * l1:
            worst = max(worst, _sin_angle(f[i, 3:6], vec[2]) / (CC * U * l1 / (l2 - l3)))
    report("fallback %s / eigen" % regime, worst, "(Jacobi result for %d of %d)" % (same.sum(), len(a6)))
    if FALLBACKS[regime]:
        assert same.mean() > 0.5, same.mean()
    elif FALLBACKS[regime] is False:
        assert same.mean() < 0.1, same.mean()


def test_coincident_points(dm, orc):
    """Coincident neighbours: sv0 = 0 and a2D = 0 * rsqrt(0) = NaN in the engine as in the reference
    ((sqrt(sv1) - sqrt(sv2)) / sqrt(sv0) = 0 / 0, neighborhood.h:302). The map's minimum distance between points of a
    voxel keeps such neighbourhoods out of real searches; a NaN weight would make the GN row NaN and the step
    non-finite, which warp_gn_solve reports as failed = 4 (test_gn_step_nonfinite_and_stop_test)."""
    rng = np.random.default_rng(RNG_SEED + 7)
    ns, rel = [], []
    for n in (5, 6, 20, 32):
        for _ in range(25):
            p = np.zeros((32, 3))
            # exactly representable offsets (multiples of 2^-10, a few bits): every moment is exact
            p[:n] = rng.integers(-64, 64, size=3) / 1024.0 if rng.uniform() < 0.5 else 0.0
            ns.append(n); rel.append(p)
    ns, rel = np.array(ns, dtype=np.int32), np.array(rel)
    d = dm.describe(False, ns, rel)
    f_desc = orc.lib.orc_neighborhood_describe
    agree = 0
    at_query = 0
    for i in range(len(ns)):
        on, oa, pl, li = np.zeros(3), C.c_double(), C.c_double(), C.c_double()
        f_desc(P(np.ascontiguousarray(rel[i, :ns[i]])), C.c_size_t(int(ns[i])), P(on), C.byref(oa), C.byref(pl),
               C.byref(li), None)
        same = (np.isnan(oa.value) and np.isnan(d[i, 3])) or oa.value == d[i, 3]
        agree += same
        if not rel[i].any():   # the query on the cluster: every moment is exactly 0 on both sides
            at_query += 1
            assert np.isnan(d[i, 3]) and np.isnan(oa.value), (d[i, 3], oa.value)
    # elsewhere the two covariance forms (query-centred moments here, the uncentred world form there) leave different
    # rounding noise in place of the zero matrix: a2D is then NaN, or a ratio of noise, on either side
    print("[device-math] coincident points: a2D engine == oracle (NaN included) for %d of %d, NaN on both at the "
          "query for %d of %d" % (agree, len(ns), at_query, at_query))
    assert at_query > 20


# ------------------------------------------------------------------------------------------------ 12x12 solve
PAIRS = [(i, j) for i in range(12) for j in range(i, 12)]


def _mp_solve(A, b, keep=None):
    idx = list(range(12)) if keep is None else keep
    M = mpmath.matrix([[A[r, c] for c in idx] for r in idx])
    y = mpmath.lu_solve(M, mpmath.matrix([b[r] for r in idx]))
    x = [mpmath.mpf(0)] * 12
    for k, r in enumerate(idx):
        x[r] = y[k]
    return x


def _solve_bound(A, x, keep=None):
    idx = list(range(12)) if keep is None else keep
    As = A[np.ix_(idx, idx)]
    d = np.sqrt(np.diag(As))
    M = As / np.outer(d, d)
    kappa = np.linalg.cond(M)
    n = 12
    return 3 * n * n * math.sqrt(n) * U * kappa * np.max(np.abs(d * np.array([float(x[r]) for r in idx]))), d, idx


def _systems(regime, rng, B, eng_tap):
    out = []
    for _ in range(B):
        J = rng.normal(size=(60, 12))
        if regime == "tap":
            A, b0 = eng_tap
            out.append((A, b0 + rng.normal(size=12) * np.abs(b0).max(), None))
            continue
        if regime.startswith("kappa"):
            kappa = float(regime.split("_")[1])
            Q = rand_rot(rng, 1)[0]
            Q12 = np.linalg.qr(rng.normal(size=(12, 12)))[0]
            M = Q12 @ np.diag(np.logspace(0, -math.log10(kappa), 12)) @ Q12.T
            D = np.logspace(0, 3, 12)[rng.permutation(12)]   # badly scaled columns: rotation vs translation
            A = M * np.outer(D, D)
            A = 0.5 * (A + A.T)
            del Q
            out.append((A, rng.normal(size=12) * D, None))
            continue
        J = J * np.logspace(0, 2, 12)
        null = []
        if regime.startswith("alpha1"):   # every alpha = 1: begin columns (rotation 0..2, translation 3..5) zero
            J[:, 0:6] = 0.0
            null = [0, 1, 2, 3, 4, 5]
        elif regime == "alpha0":          # every alpha = 0: end columns zero
            J[:, 6:12] = 0.0
            null = list(range(6, 12))
        elif regime == "mid_elimination":   # identical rows 0 and 1: the pivot of row 1 becomes exactly 0 at step 1
            J[:, 1] = J[:, 0]
            null = [1]
            J *= 1.0 / np.sqrt(np.sum(J[:, 0] ** 2) / 60.0)
        A = J.T @ J / 60.0
        A = 0.5 * (A + A.T)
        b = J.T @ rng.normal(size=60) / 60.0
        if regime == "alpha1_motion":   # the motion-model regulariser on the begin translation (warp_gn_solve)
            for d in range(3):
                A[3 + d, 3 + d] += 0.01
                b[3 + d] -= 0.01 * rng.normal()
            null = [0, 1, 2]
        if regime == "mid_elimination":
            # A[0][0] = 1 exactly: the elimination's multiplier a_10 * (1 / a_00) is exactly 1 and row 1 becomes exactly
            # zero, as it does with Eigen's division. (With a pivot whose reciprocal is inexact the product leaves a
            # remainder of ~u a_00 in place of the zero pivot: DESIGN.md section 2, documented deviations.)
            A[0, 0] = 1.0
            A[1, :] = A[0, :]
            A[:, 1] = A[:, 0]
            b[1] = b[0]
        out.append((A, b, null))
    return out


SOLVE_REGIMES = ["tap", "kappa_1e2", "kappa_1e6", "kappa_1e10", "kappa_1e14", "alpha1", "alpha1_motion", "alpha0",
                 "mid_elimination"]


@pytest.fixture(scope="module")
def gn_tap(orc, eng):
    """A, b of one linearisation from the engine's gn_normal_equations tap on the hdl64 parity scene."""
    from test_gpu_parity import _fill_world, _registration_case, small_map_options
    map_xyz, kp, frame, prev = _registration_case(orc, eng, "GN")
    me = eng.voxel_map(small_map_options(eng, cap=1 << 18))
    me.insert(map_xyz)
    io = orc.default_icp_options()
    io.solver = abi.SOLVER["GN"]
    io.min_number_neighbors = 10
    mm = orc.default_odometry_options().default_motion_model
    _fill_world(orc, kp, frame)
    A, b, n = me.gn_normal_equations(io, kp.copy(), frame, prev, mm)
    assert n > 100
    return np.array(A, dtype=np.float64).reshape(12, 12), np.array(b, dtype=np.float64).reshape(12)


@pytest.mark.parametrize("regime", SOLVE_REGIMES)
def test_ldlt_solve12(dm, orc, gn_tap, regime):
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + 3 * len(regime) + ord(regime[-1]))
    B = 40 if regime == "tap" else 80
    systems = _systems(regime, rng, B, gn_tap)
    A = np.array([s[0].reshape(144) for s in systems])
    b = np.array([s[1] for s in systems])
    x_reg, x_cmp = dm.solve(False, A, b), dm.solve(True, A, b)
    # (c) the register and the compact forms do the same operations on the same operands in the same order
    assert np.array_equal(x_reg, x_cmp, equal_nan=True)
    f = orc.lib.orc_ldlt_solve12
    w_truth = w_orc = 0.0
    for i, (Ai, bi, null) in enumerate(systems):
        keep = None if not null else [k for k in range(12) if k not in null]
        xt = _mp_solve(Ai, bi, keep)
        bound, d, idx = _solve_bound(Ai, xt, keep)
        if null:   # Eigen's convention: pseudo-inverse of D, zero along the null coordinates
            assert np.all(x_reg[i, null] == 0.0), (regime, x_reg[i, null])
        err = np.max(np.abs(d * (x_reg[i, idx] - np.array([float(xt[r]) for r in idx]))))
        w_truth = max(w_truth, err / bound)
        xo = np.zeros(12)
        f(P(np.ascontiguousarray(Ai)), P(np.ascontiguousarray(bi)), P(xo))
        if regime == "mid_elimination":
            # columns 0 and 1 are equal: only x0 + x1 is determined. Eliminating in natural order, the device zeroes x1;
            # the oracle's (Eigen's) diagonal pivoting may reach row 1 first and zero x0 instead
            assert xo[0] == 0.0 or xo[1] == 0.0
            xo = xo.copy()
            xo[0], xo[1] = xo[0] + xo[1], 0.0
        elif null:
            assert np.all(xo[null] == 0.0)
        w_orc = max(w_orc, np.max(np.abs(d * (x_reg[i, idx] - xo[idx]))) / (2 * bound))
    report("solve %s / truth" % regime, w_truth)
    report("solve %s / oracle" % regime, w_orc)


# ------------------------------------------------------------------------------------------------ Gauss-Newton step
def _acc_from(A, b, n):
    acc = np.zeros(96)
    for e, (i, j) in enumerate(PAIRS):
        acc[e] = A[i, j] * n
    acc[78:90] = b * n
    acc[90] = n
    return acc


def _mp_quat_from_R(R):
    """Quaternion of a rotation matrix (any branch: the exact value is branch independent up to sign)."""
    t = R[0, 0] + R[1, 1] + R[2, 2]
    cands = [(t, 3), (R[0, 0], 0), (R[1, 1], 1), (R[2, 2], 2)]
    _, k = max(cands, key=lambda c: c[0])
    q = [None] * 4
    if k == 3:
        s = mpmath.sqrt(t + 1) * 2
        q = [(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, s / 4]
    else:
        i, j, kk = k, (k + 1) % 3, (k + 2) % 3
        s = mpmath.sqrt(R[i, i] - R[j, j] - R[kk, kk] + 1) * 2
        c = [None] * 3
        c[i] = s / 4
        c[j] = (R[j, i] + R[i, j]) / s
        c[kk] = (R[kk, i] + R[i, kk]) / s
        q = [c[0], c[1], c[2], (R[kk, j] - R[j, kk]) / s]
    nq = mpmath.sqrt(sum(v * v for v in q))
    return [v / nq for v in q]


def _mp_qtoR(q):
    x, y, z, w = q
    return mpmath.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                          [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                          [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _mp_euler(a, b, g):
    ca, sa, cb, sb, cg, sg = mpmath.cos(a), mpmath.sin(a), mpmath.cos(b), mpmath.sin(b), mpmath.cos(g), mpmath.sin(g)
    return mpmath.matrix([[cg * cb, -sg * ca + cg * sb * sa, sg * sa + cg * sb * ca],
                          [sg * cb, cg * ca + sg * sb * sa, -cg * sa + sg * sb * ca],
                          [-sb, cb * sa, cb * ca]])


def _gn_case(regime, rng):
    """(acc, state, x_target): a well-conditioned system whose solution is x_target, and the pose it updates."""
    J = rng.normal(size=(40, 12))
    A = J.T @ J / 40.0 + np.eye(12)
    A = 0.5 * (A + A.T)
    x = rng.normal(size=12) * 1e-3
    qb, qe = Rotation.from_rotvec(rng.normal(size=3) * 0.3).as_quat(), Rotation.from_rotvec(rng.normal(size=3) * 0.3).as_quat()
    n = 150
    if regime == "angles_at_switch":
        for k in (0, 1, 2, 6, 7, 8):
            x[k] = 0.5 + rng.choice([-1, 1]) * 10.0 ** rng.uniform(-15, -3)
    elif regime == "pitch_pm_half_pi":
        x[1] = rng.choice([-1, 1]) * math.pi / 2
        x[7] = rng.choice([-1, 1]) * math.pi / 2
    elif regime == "qfromR_branches":   # orientations beyond 120 deg about each axis: trace(R) <= 0 after the step
        ax = np.zeros(3)
        ax[rng.integers(3)] = 1.0
        ax += rng.normal(size=3) * 0.1
        qb = Rotation.from_rotvec(ax / np.linalg.norm(ax) * rng.uniform(2.2, math.pi)).as_quat()
        qe = Rotation.from_rotvec(ax / np.linalg.norm(ax) * rng.uniform(2.2, math.pi)).as_quat()
    elif regime == "n_used_99":
        n = 99
    elif regime == "n_used_100":
        n = 100
    b = A @ x
    state = np.zeros(24)
    state[0:4], state[4:7], state[7:11], state[11:14] = qb, rng.normal(size=3), qe, rng.normal(size=3)
    state[14:17], state[17:20] = rng.normal(size=3), rng.normal(size=3)
    if rng.uniform() < 0.5:
        state[20], state[21], state[22] = 1.0, 0.001, 0.001
    return A, b, n, state


GN_REGIMES = ["random", "angles_at_switch", "pitch_pm_half_pi", "qfromR_branches", "n_used_99", "n_used_100"]


@pytest.mark.parametrize("regime", GN_REGIMES)
def test_gn_step_regimes(dm, orc, regime):
    """warp_gn_solve against an mpmath restatement of ct_icp.cpp:877-980: 1/n, regularisers, solve, Euler-ZYX
    update R * R(q), Quaternion(Matrix3), normalisation, x_norm, slerp constants."""
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + 11 * len(regime) + ord(regime[0]))
    cases = [_gn_case(regime, rng) for _ in range(60)]
    acc = np.array([_acc_from(A, b, n) for A, b, n, _ in cases])
    st = np.array([c[3] for c in cases])
    out1, sys1 = dm.gn(1, acc, st, 0.0)
    out0, sys0 = dm.gn(0, acc, st, 1e-300)
    fq = orc.lib.orc_quat_from_matrix
    w_sys = w_x = w_pose = w_orc = 0.0
    for i, (A, b, n, s) in enumerate(cases):
        if n < 100:   # ct_icp.cpp:860-871: not enough residuals: failed, pose untouched
            assert out0[i, 27] == 1 and out0[i, 28] == 1 and out0[i, 29] == 0
            assert np.array_equal(out0[i, 0:14], s[0:14])
            continue
        # mode 1: the system the solve sees
        inv = 1.0 / n
        At = np.zeros((12, 12))
        for e, (p, q) in enumerate(PAIRS):
            At[p, q] = At[q, p] = acc[i, e] * inv
        bt = acc[i, 78:90] * inv
        if s[20]:
            for d in range(3):
                At[3 + d, 3 + d] += s[21]
                bt[3 + d] -= s[21] * (s[4 + d] - s[11 + d])
                At[9 + d, 9 + d] += s[22]
                bt[9 + d] -= s[22] * (s[11 + d] - s[4 + d] - s[17 + d] + s[14 + d])
        sysA, sysb = sys1[i, :144].reshape(12, 12), sys1[i, 144:156]
        w_sys = max(w_sys, np.max(np.abs(sysA - At) / (2 * U * np.maximum(np.abs(At), 1e-300))))
        scale_b = np.abs(acc[i, 78:90] * inv) + (np.abs(s[21]) + np.abs(s[22])) * 4 * (np.abs(s[4:20]).max())
        w_sys = max(w_sys, np.max(np.abs(sysb - bt) / (4 * U * np.maximum(scale_b, 1e-300))))
        assert sys1[i, 156] == n
        # mode 0: step and pose against the restatement on the device's own system
        xt = _mp_solve(sysA, sysb)
        bound, d, _ = _solve_bound(sysA, xt)
        xd = out0[i, 14:26]
        w_x = max(w_x, np.max(np.abs(d * (xd - np.array([float(v) for v in xt])))) / bound)
        xb = bound / d.min()   # absolute bound on each step component
        for lane, (qo, to, xo) in enumerate(((0, 4, 0), (7, 11, 6))):
            q = [mpf(v) for v in s[qo:qo + 4]]
            R = _mp_euler(xt[xo], xt[xo + 1], xt[xo + 2]) * _mp_qtoR(q)
            qt = _mp_quat_from_R(R)
            qd = out0[i, qo:qo + 4]
            qtf = np.array([float(v) for v in qt])
            err = min(np.abs(qd - qtf).max(), np.abs(qd + qtf).max())
            w_pose = max(w_pose, err / (8 * xb + CC * U))
            tt = s[to:to + 3] + np.array([float(v) for v in xt[xo + 3:xo + 6]])
            w_pose = max(w_pose, np.abs(out0[i, to:to + 3] - tt).max() / (xb + 4 * U * np.abs(tt).max()))
            # (b) the oracle's Quaternion(Matrix3) on the same rotation: same branch, same sign
            Rd = np.array([[float(R[r, c]) for c in range(3)] for r in range(3)])
            qo_ = np.zeros(4)
            fq(P(np.ascontiguousarray(Rd)), P(qo_))
            qo_ /= np.linalg.norm(qo_)
            w_orc = max(w_orc, np.abs(qd - qo_).max() / (8 * xb + 2 * CC * U))
        xn = float(mpmath.sqrt(sum(v * v for v in xt)))
        assert abs(out0[i, 26] - xn) <= 2 * xb * math.sqrt(12) + CC * U * xn
        assert out0[i, 27] == 0 and out0[i, 29] == 1
    report("gn %s / system" % regime, w_sys)
    report("gn %s / step" % regime, w_x)
    report("gn %s / pose" % regime, w_pose)
    report("gn %s / oracle quat_from_matrix" % regime, w_orc)


def test_gn_step_nonfinite_and_stop_test(dm):
    """A NaN in the accumulator (a coincident-point row) or a step that overflows: failed = 4, pose untouched. The stop
    test is x_norm < threshold_orientation_norm, strict (ct_icp.cpp:978)."""
    rng = np.random.default_rng(RNG_SEED + 99)
    A, b, n, s = _gn_case("random", rng)
    acc = _acc_from(A, b, n)
    bad_nan = acc.copy()
    bad_nan[5] = np.nan
    tiny = np.zeros(96)   # a pivot just above DBL_MIN: 1 / pivot overflows
    for e, (i, j) in enumerate(PAIRS):
        if i == j:
            tiny[e] = 1.0 * n
    tiny[0] = 1e-307 * n
    tiny[78] = 1e10 * n
    tiny[90] = n
    out, _ = dm.gn(0, np.array([bad_nan, tiny]), np.array([s, s]), 1e-4)
    for k in range(2):
        assert out[k, 27] == 4 and out[k, 28] == 1, out[k, 27:31]
        assert np.array_equal(out[k, 0:14], s[0:14])
    out, _ = dm.gn(0, acc[None], s[None], 1e-300)
    xn = out[0, 26]
    at, above = dm.gn(0, acc[None], s[None], float(xn))[0], dm.gn(0, acc[None], s[None], float(np.nextafter(xn, np.inf)))[0]
    assert at[0, 26] == xn and above[0, 26] == xn
    assert at[0, 28] == 0 and above[0, 28] == 1
    print("[device-math] gn stop test: x_norm %.17g: done at threshold = x_norm: %d, one ulp above: %d"
          % (xn, at[0, 28], above[0, 28]))


# ------------------------------------------------------------------------------------------------ CT functor
def _mp_normalized(q):
    n = mpmath.sqrt(sum(v * v for v in q))
    return [v / n for v in q]


def _mp_functor(x, blk, kind, simple, branch):
    """CTFunctor<...>::operator() (cost_functions.h:186-222 -> :32-67, :121-129, :163-171) on mpmath (complex) numbers.
    `branch` fixes Eigen's slerp branch (linear or acos) at the base point, as the duals and Jets take it."""
    ref, nrm, weight, alpha, raw, info = blk[0:3], blk[3:6], blk[6], blk[7], blk[8:11], blk[11:17]
    qb, qe, tb, te = x[0:4], x[4:8], x[8:11], x[11:14]
    if simple:
        qi, tr = qe, te
    else:
        a, b = _mp_normalized(qb), _mp_normalized(qe)
        d = sum(a[k] * b[k] for k in range(4))
        neg = mpmath.re(d) < 0
        ad = -d if neg else d
        if branch:
            s0, s1 = 1 - alpha, alpha
        else:
            th = mpmath.acos(ad)
            s0, s1 = mpmath.sin((1 - alpha) * th) / mpmath.sin(th), mpmath.sin(alpha * th) / mpmath.sin(th)
        if neg:
            s1 = -s1
        qi = _mp_normalized([s0 * a[k] + s1 * b[k] for k in range(4)])
        tr = [(1 - alpha) * tb[k] + alpha * te[k] for k in range(3)]
    q = qi if kind == 1 else _mp_normalized(qi)
    qv, w = q[0:3], q[3]
    v = [mpf(t) for t in raw]
    uv = [2 * (qv[1] * v[2] - qv[2] * v[1]), 2 * (qv[2] * v[0] - qv[0] * v[2]), 2 * (qv[0] * v[1] - qv[1] * v[0])]
    cr = [qv[1] * uv[2] - qv[2] * uv[1], qv[2] * uv[0] - qv[0] * uv[2], qv[0] * uv[1] - qv[1] * uv[0]]
    p = [v[k] + w * uv[k] + cr[k] + tr[k] for k in range(3)]
    dd = [p[k] - mpf(ref[k]) for k in range(3)]
    if kind == 1:
        u = [mpf(t) for t in nrm]
        z = sum(t * t for t in u)
        if z > 0:
            u = [t / mpmath.sqrt(z) for t in u]
        c = [u[1] * dd[2] - u[2] * dd[1], u[2] * dd[0] - u[0] * dd[2], u[0] * dd[1] - u[1] * dd[0]]
        return mpf(weight) * mpmath.sqrt(sum(t * t for t in c))
    if kind == 2:
        I = [[info[0], info[1], info[2]], [info[1], info[3], info[4]], [info[2], info[4], info[5]]]
        return mpf(weight) * sum(dd[r] * mpf(I[r][c]) * dd[c] for r in range(3) for c in range(3))
    return mpf(weight) * sum(mpf(nrm[k]) * (mpf(ref[k]) - p[k]) for k in range(3))


def _plus_cols(q):
    x, y, z, w = q
    return [[w, -z, y, -x], [z, w, -x, -y], [-y, x, w, -z]]


def _mp_functor_jac(xv, blk, kind, simple, branch):
    """value and the 12 tangent partials by complex steps (h = 1e-40 at 50 digits: truncation h^2, no cancellation).
    branch: the slerp branch the device took (its own fp64 dot product, harness entry dq_dot)."""
    xm = [mpf(t) for t in xv]
    qb, qe = _mp_normalized(xm[0:4]), _mp_normalized(xm[4:8])
    d = abs(sum(qb[k] * qe[k] for k in range(4)))
    val = _mp_functor(xm, blk, kind, simple, branch)
    h = mpmath.mpf(10) ** -40
    jac = []
    for j in range(12):
        t = [mpmath.mpf(0)] * 14
        if j < 3:
            col = _plus_cols(xv[0:4])[j]
            for k in range(4):
                t[k] = mpf(col[k])
        elif j < 6:
            col = _plus_cols(xv[4:8])[j - 3]
            for k in range(4):
                t[4 + k] = mpf(col[k])
        elif j < 9:
            t[8 + j - 6] = mpmath.mpf(1)
        else:
            t[11 + j - 9] = mpmath.mpf(1)
        xc = [mpmath.mpc(xm[k], h * t[k]) for k in range(14)]
        jac.append(mpmath.im(_mp_functor(xc, blk, kind, simple, branch)) / h)
    theta = float(mpmath.acos(min(d, mpmath.mpf(1))))
    return float(val), np.array([float(v) for v in jac]), theta


def _functor_cases(regime, rng, B, dm):
    blks, kinds, xs = [], [], []
    for i in range(B):
        kind = i % 3
        ref = rng.normal(size=3) * 5
        nrm = rng.normal(size=3)
        nrm /= np.linalg.norm(nrm)
        raw = rng.normal(size=3) * 5
        M = rng.normal(size=(3, 3))
        info = np.linalg.inv(M @ M.T * 0.01 + 0.05 * np.eye(3))
        weight = rng.uniform(0.3, 1.0)
        alpha = rng.uniform()
        qb = Rotation.from_rotvec(rng.normal(size=3) * 0.2).as_quat()
        qe = (Rotation.from_rotvec(rng.normal(size=3) * 0.02) * Rotation.from_quat(qb)).as_quat()
        if regime.startswith("alpha_"):
            alpha = {"alpha_0": 0.0, "alpha_1": 1.0, "alpha_half": 0.5, "alpha_1e-9": 1e-9, "alpha_1-1e-9": 1 - 1e-9}[regime]
        elif regime == "negative_dot":
            qe = -qe
        elif regime.startswith("sweep"):   # slerp angle theta = acos|d| just below / above the 0.5 rad switch
            th = 0.5 + (-1 if regime.endswith("below") else 1) * 10.0 ** rng.uniform(-12, -4)
            ax = rng.normal(size=3)
            qe = (Rotation.from_rotvec(ax / np.linalg.norm(ax) * 2 * th) * Rotation.from_quat(qb)).as_quat()
        elif regime == "non_unit":
            qb = qb * (1 + rng.choice([-1, 1]) * 1e-8)
            qe = qe * (1 + rng.choice([-1, 1]) * 1e-8)
        elif regime == "line_distance_0":
            kind, raw, alpha = 1, np.zeros(3), 0.0
        elif regime == "weight_0":
            weight = 0.0
        elif regime == "simple":
            kind |= 16
        elif regime.startswith("dot_"):
            qe = _dot_target(regime, qb, rng, dm)
        blks.append(np.concatenate([ref, nrm, [weight, alpha], raw, [info[0, 0], info[0, 1], info[0, 2], info[1, 1],
                                                                      info[1, 2], info[2, 2]]]))
        kinds.append(kind)
        x = np.concatenate([qb, qe, rng.normal(size=3), rng.normal(size=3)])
        if regime == "line_distance_0":
            blks[-1][0:3] = x[8:11]   # ref = the begin translation = the transformed point (raw = 0, alpha = 0)
        xs.append(x)
    return np.array(blks), np.array(kinds), np.array(xs)


_ONE = 1.0 - 2.220446049250313e-16


def _dot_target(regime, qb, rng, dm):
    """q_e whose device dot product dq_dot(normalized q_b, normalized q_e) is exactly the regime's value: a small search
    over q_e's last bits with the device's own dq_dot (FMA contraction moves the last bit)."""
    target = {"dot_1": 1.0, "dot_one": _ONE, "dot_one_minus_ulp": np.nextafter(_ONE, 0.0),
              "dot_1-1e-8": 1 - 1e-8, "dot_1-1e-4": 1 - 1e-4}[regime]
    th = math.acos(target) if target < 1 else 0.0
    ax = rng.normal(size=3)
    qe0 = (Rotation.from_rotvec(ax / np.linalg.norm(ax) * 2 * th) * Rotation.from_quat(qb)).as_quat()
    if target == 1.0:
        return qb.copy()
    if target > 1 - 1e-12:   # exactly on a representable value next to 1: scan a few ulps of w
        cands = []
        base = qb.copy()
        for k in range(-40, 41):
            q = base.copy()
            q[0] = base[0] + k * 1e-9
            q[1] = base[1] - k * 1e-9
            cands.append(q)
        cands = np.array(cands)
        x = np.zeros((len(cands), 14))
        x[:, 0:4] = qb
        x[:, 4:8] = cands
        d = np.abs(dm.dq_dot(x))
        hit = np.flatnonzero(d == target)
        return cands[hit[0]] if len(hit) else cands[np.argmin(np.abs(d - target))]
    return qe0


FUNCTOR_REGIMES = ["random", "alpha_0", "alpha_1", "alpha_half", "alpha_1e-9", "alpha_1-1e-9", "negative_dot",
                   "sweep_below", "sweep_above", "non_unit", "line_distance_0", "weight_0", "simple",
                   "dot_1", "dot_one", "dot_one_minus_ulp", "dot_1-1e-8", "dot_1-1e-4"]


@pytest.mark.parametrize("regime", FUNCTOR_REGIMES)
def test_ct_residual(dm, orc, regime):
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + 5 * len(regime) + ord(regime[-1]))
    B = 48
    blk, kind, x = _functor_cases(regime, rng, B, dm)
    outs = {robust: dm.residual(robust, blk, kind, x) for robust in (True, False)}
    linear = np.abs(dm.dq_dot(x)) >= _ONE
    f = orc.lib.orc_ct_residual
    f.restype = C.c_double
    w_truth = w_orc = 0.0
    for i in range(B):
        k, simple = kind[i] & 15, bool(kind[i] & 16)
        out = outs[True][i]
        if k == 0:   # the CERES instantiation of the plane functor: same source, but compiled into another function the
            # compiler contracts differently (observed: last-bit differences), so it is held to the truth bound below
            w_truth = max(w_truth, np.abs(outs[False][i] - out).max() / (2 * CC * U * max(1.0, np.abs(out).max())))
        if simple:   # the begin pose is not a parameter of the SIMPLE functor
            assert np.all(out[[0, 1, 2, 6, 7, 8]] == 0.0)
        if regime == "weight_0":
            assert np.all(out == 0.0)
        val, jac, theta = _mp_functor_jac(x[i], blk[i], k, simple, bool(linear[i]))
        S = max(abs(val), np.abs(jac).max(), blk[i, 6] * (1 + np.abs(blk[i, 8:11]).max()) *
                (1 + np.abs(blk[i, 0:3]).max() + np.abs(x[i, 8:14]).max()) * (1 + np.abs(blk[i, 11:17]).max()))
        S = max(S, 1e-300)   # weight 0: every term is 0 (asserted exactly above)
        amp = 1.0 + (1.0 / theta ** 2 if theta > 0 and not linear[i] and not simple else 0.0)
        bound = CC * U * S * amp
        if regime == "line_distance_0":
            # |c| = 0: the sqrt has no derivative there; duals and Jets both divide 0 by 2 sqrt(0)
            assert out[12] == 0.0 and np.all(np.isnan(out[:12]))
        else:
            w_truth = max(w_truth, max(abs(out[12] - val), np.abs(out[:12] - jac).max()) / bound)
        if simple:
            continue   # the oracle's tap has no SIMPLE block
        okind = {0: abi_dist("PLANE"), 1: abi_dist("LINE"), 2: abi_dist("DIST")}[k]
        cov = None
        if k == 2:   # the tap takes the covariance and forms information = (cov + 0.05 I)^-1 itself
            info = blk[i, 11:17]
            I = np.array([[info[0], info[1], info[2]], [info[1], info[3], info[4]], [info[2], info[4], info[5]]])
            cov = np.ascontiguousarray(np.linalg.inv(I) - 0.05 * np.eye(3))
        jo = np.zeros(12)
        xi = x[i]
        ov = f(okind, C.c_double(blk[i, 7]), P(np.ascontiguousarray(blk[i, 0:3])), P(np.ascontiguousarray(blk[i, 8:11])),
               P(np.ascontiguousarray(blk[i, 3:6])), P(cov) if cov is not None else None, C.c_double(blk[i, 6]),
               P(np.ascontiguousarray(xi[0:4])), P(np.ascontiguousarray(xi[8:11])), P(np.ascontiguousarray(xi[4:8])),
               P(np.ascontiguousarray(xi[11:14])), P(jo))
        if regime == "line_distance_0":
            assert ov == 0.0 and np.all(np.isnan(jo))
            continue
        if k == 2:   # the information matrix went through an inverse on both sides: its own rounding, relative 1e3 u
            bound = bound + 1e3 * U * S
        w_orc = max(w_orc, max(abs(ov - out[12]), np.abs(jo - out[:12]).max()) / (2 * bound))
    report("functor %s / truth" % regime, w_truth)
    report("functor %s / oracle" % regime, w_orc)


def abi_dist(name):
    return {"PLANE": 0, "LINE": 2, "DIST": 3}[name]


# ------------------------------------------------------------------------------------------------ quat_plus, losses
def test_quat_plus(dm, orc):
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + 13)
    norms = [0.0, 1e-12, 0.5, float(np.nextafter(0.5, 0)), float(np.nextafter(0.5, 1)), 1.0, 3.0]
    q, d = [], []
    for nn in norms:
        for _ in range(40):
            qq = rng.normal(size=4)
            q.append(qq / np.linalg.norm(qq))
            v = rng.normal(size=3)
            d.append(v / np.linalg.norm(v) * nn)
    q, d = np.array(q), np.array(d)
    out = dm.simple("quat_plus", 4, q, d)
    f = orc.lib.orc_quat_plus
    worst = worst_o = 0.0
    for i in range(len(q)):
        dm_ = [mpf(t) for t in d[i]]
        n = mpmath.sqrt(sum(t * t for t in dm_))
        if n == 0:
            assert np.array_equal(out[i], q[i])
            continue
        s, c = mpmath.sin(n) / n, mpmath.cos(n)
        a = [s * dm_[0], s * dm_[1], s * dm_[2], c]
        b = [mpf(t) for t in q[i]]
        r = [a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1], a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
             a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0], a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]]
        worst = max(worst, max(abs(out[i, k] - float(r[k])) for k in range(4)) / (CC * U))
        o = np.zeros(4)
        f(P(np.ascontiguousarray(q[i])), P(np.ascontiguousarray(d[i])), P(o))
        worst_o = max(worst_o, np.abs(o - out[i]).max() / (2 * CC * U))
    report("quat_plus / truth", worst)
    report("quat_plus / oracle", worst_o)


LOSSES = {"STANDARD": 0, "CAUCHY": 1, "HUBER": 2, "TOLERANT": 3, "TRUNCATED": 4}


def _mp_rho(loss, s, sigma, tol):
    """the published rho, rho', rho'' in 50 digits, with the loss's fp64 constants as ceres forms them (b = sigma * sigma
    rounded, c = 1 / b rounded): the branch thresholds are those fp64 numbers"""
    s = mpf(s)
    one, zero = mpmath.mpf(1), mpmath.mpf(0)
    if loss == "STANDARD":
        return [s, one, zero]
    if loss == "CAUCHY":
        b = sigma * sigma
        c = mpf(1.0 / b)
        return [mpf(b) * mpmath.log(1 + s * c), 1 / (1 + s * c), -c / (1 + s * c) ** 2]
    if loss == "HUBER":   # the quadratic piece up to and including s = a^2
        a, b = mpf(sigma), mpf(sigma * sigma)
        if s > b:
            r = mpmath.sqrt(s)
            return [2 * a * r - b, a / r, -(a / r) / (2 * s)]
        return [s, one, zero]
    if loss == "TOLERANT":
        a, b = mpf(tol), mpf(sigma)
        x = (s - a) / b
        c = b * mpmath.log(1 + mpmath.exp(-a / b))
        e = mpmath.exp(x)
        return [b * mpmath.log(1 + e) - c, e / (1 + e), e / (b * (1 + e) ** 2)]
    b = mpf(sigma * sigma)   # TruncatedLoss: quadratic below sigma^2, constant from sigma^2 on
    return [s, one, zero] if s < b else [b, zero, zero]


@pytest.mark.parametrize("loss", list(LOSSES))
def test_loss_evaluate(dm, orc, loss):
    mpmath.mp.dps = DPS
    sigma, tol = 0.1, 0.05
    s2 = sigma * sigma
    ss = [0.0, 1e-12, s2, float(np.nextafter(s2, 0)), float(np.nextafter(s2, 1))] + list(np.logspace(-6, 1, 60))
    # Tolerant: x = (s - a) / b on both sides of the 36.7 switch (a = tol, b = sigma)
    for xx in (36.7, 36.69999999, 36.70000001, 30.0, 40.0):
        ss.append(tol + sigma * xx)
    ss = np.array(ss)
    L = np.tile([LOSSES[loss], sigma, tol], (len(ss), 1)).astype(np.float64)
    rho = dm.simple("loss_evaluate", 3, L, ss)
    o = orc.default_icp_options()
    o.loss_function, o.ls_sigma, o.ls_tolerant_min_threshold = abi.LOSS[loss], sigma, tol
    f = orc.lib.orc_loss_evaluate
    worst = worst_o = 0.0
    for i, s in enumerate(ss):
        t = [float(v) for v in _mp_rho(loss, s, sigma, tol)]
        ro = np.zeros(3)
        f(C.byref(o), C.c_double(s), P(ro))
        # magnitudes of the terms each formula adds or subtracts: rho0 = b log(1 + s c) and b log(1 + e^x) - c lose the
        # absolute error u (b + s + c) to the rounding of their arguments; rho' is O(1); rho'' is O(1 / sigma^2).
        # Tolerant beyond the x > 36.7 switch: rho' = 1, rho'' = 0 exactly where the truth is 1 - e^-x, e^-x / b
        # (< 1.2e-15): inside c u / sigma^2.
        T = [s2 + s + tol, 1.0, 1.0 / s2]
        for k in range(3):
            b = CC * U * (abs(t[k]) + T[k])
            worst = max(worst, abs(rho[i, k] - t[k]) / b if (rho[i, k] != t[k]) else 0.0)
            worst_o = max(worst_o, abs(rho[i, k] - ro[k]) / (2 * b) if rho[i, k] != ro[k] else 0.0)
    report("loss %s / truth" % loss, worst)
    report("loss %s / oracle" % loss, worst_o)


def test_corrector(dm, orc):
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + 17)
    s, rho = [], []
    for sign in (1, 0, -1):
        for _ in range(50):
            si = float(10 ** rng.uniform(-6, 0))
            r1 = float(rng.uniform(0.05, 1.0))
            # rho'' positive (tolerant-like, small enough that D > 0), zero, negative (Cauchy / Huber)
            r2 = sign * r1 / (4 * si) * float(rng.uniform(0.01, 0.4)) if sign else 0.0
            s.append(si); rho.append([0.0, r1, r2])
    s.append(0.0); rho.append([0.0, 0.5, 0.3])
    s, rho = np.array(s), np.array(rho)
    out = dm.simple("corrector", 2, s, rho)
    f = orc.lib.orc_corrector
    worst = worst_o = 0.0
    for i in range(len(s)):
        r1 = mpf(rho[i, 1])
        sq = mpmath.sqrt(r1)
        if s[i] == 0 or rho[i, 2] <= 0:
            t = [sq, sq]
        else:
            D = 1 + 2 * mpf(s[i]) * mpf(rho[i, 2]) / r1
            a = 1 - mpmath.sqrt(D)
            t = [sq / (1 - a), sq * (1 - a)]
        worst = max(worst, max(abs(out[i, k] - float(t[k])) / (CC * U * float(abs(t[k]))) for k in range(2)))
        rs, js = C.c_double(), C.c_double()
        f(C.c_double(s[i]), P(np.ascontiguousarray(rho[i])), C.byref(rs), C.byref(js))
        worst_o = max(worst_o, abs(rs.value - out[i, 0]) / (2 * CC * U * abs(rs.value)),
                      abs(js.value - out[i, 1]) / (2 * CC * U * abs(js.value)))
    report("corrector / truth", worst)
    report("corrector / oracle", worst_o)


# ------------------------------------------------------------------------------------------------ pose helpers
def test_slerp_transform_qfromR_voxel(dm, orc):
    """ct_transform_c with slerp_consts (the GN gather's world point), qfromR / qtoR, voxel_coord_rcp."""
    mpmath.mp.dps = DPS
    rng = np.random.default_rng(RNG_SEED + 19)
    rows = []
    for i in range(300):
        qb = Rotation.from_rotvec(rng.normal(size=3) * 0.5).as_quat()
        ang = [1e-9, 1e-4, 0.01, 0.4, 0.9999, 1.0001, 2.0][i % 7]   # 2 theta: around the 0.5 rad switch of qslerp_c
        ax = rng.normal(size=3)
        qe = (Rotation.from_rotvec(ax / np.linalg.norm(ax) * ang) * Rotation.from_quat(qb)).as_quat()
        if i % 5 == 0:
            qe = -qe
        rows.append(np.concatenate([qb, rng.normal(size=3), qe, rng.normal(size=3), rng.normal(size=3) * 30,
                                    [rng.uniform()]]))
    rows = np.array(rows)
    out = dm.simple("ct_transform", 12, rows)
    worst = 0.0
    for i, r in enumerate(rows):
        a, b = [mpf(t) for t in r[0:4]], [mpf(t) for t in r[7:11]]
        d = sum(a[k] * b[k] for k in range(4))
        ad = abs(d)
        t = mpf(r[17])
        if ad >= _ONE:
            s0, s1 = 1 - t, t
        else:
            th = mpmath.acos(ad)
            s0, s1 = mpmath.sin((1 - t) * th) / mpmath.sin(th), mpmath.sin(t * th) / mpmath.sin(th)
        if d < 0:
            s1 = -s1
        q = _mp_normalized([s0 * a[k] + s1 * b[k] for k in range(4)])
        R = _mp_qtoR(q)
        v = [mpf(x) for x in r[14:17]]
        tr = [(1 - t) * mpf(r[4 + k]) + t * mpf(r[11 + k]) for k in range(3)]
        w = [sum(R[k, c] * v[c] for c in range(3)) + tr[k] for k in range(3)]
        th = float(mpmath.acos(min(ad, 1)))
        # inv_sin = 1 / sqrt((1 - d)(1 + d)): 1 - d carries the absolute error u of d, relative u / theta^2
        amp = 1 + (1 / th ** 2 if th > 0 and ad < _ONE else 0)
        scale = 1 + np.abs(r[4:17]).max()
        worst = max(worst, max(abs(out[i, k] - float(w[k])) for k in range(3)) / (CC * U * scale * amp))
    report("ct_transform_c / truth", worst)
    # qfromR on every branch (trace > 0, and i = 0, 1, 2), against the oracle's Quaternion(Matrix3) and the truth
    rots = [Rotation.from_rotvec(v) for v in rng.normal(size=(100, 3)) * 0.5]
    for axis in range(3):
        for _ in range(60):
            v = rng.normal(size=3) * 0.2
            v[axis] = rng.choice([-1, 1]) * rng.uniform(2.2, math.pi)
            rots.append(Rotation.from_rotvec(v))
    rots += [Rotation.from_euler("y", s * math.pi / 2) for s in (-1, 1)] + [Rotation.from_euler(a, math.pi) for a in "xyz"]
    Rm = np.array([r.as_matrix().reshape(9) for r in rots])
    qd = dm.simple("qfromR", 4, Rm)
    Rd = dm.simple("qtoR", 9, qd)
    fq = orc.lib.orc_quat_from_matrix
    w_q = w_o = w_r = 0.0
    for i in range(len(Rm)):
        qo = np.zeros(4)
        fq(P(np.ascontiguousarray(Rm[i])), P(qo))
        w_o = max(w_o, np.abs(qo - qd[i]).max() / (CC * U))
        qt = _mp_quat_from_R(mpmath.matrix(Rm[i].reshape(3, 3).tolist()))
        qtf = np.array([float(v) for v in qt])
        w_q = max(w_q, min(np.abs(qd[i] - qtf).max(), np.abs(qd[i] + qtf).max()) / (CC * U))
        w_r = max(w_r, np.abs(Rd[i] - Rm[i]).max() / (CC * U))
    report("qfromR / truth", w_q)
    report("qfromR / oracle", w_o)
    report("qtoR(qfromR(R)) / R", w_r)
    # voxel_coord_rcp: C truncation of p / res, including quotients within ulps of an integer
    res = 0.1
    base = rng.integers(-5000, 5000, size=400) * res
    p = np.concatenate([base, np.nextafter(base, np.inf), np.nextafter(base, -np.inf), rng.uniform(-500, 500, 400)])
    vc = dm.simple("voxel_coord_rcp", 1, p, extra=(float(res),))
    want = np.array([int(x / res) for x in p])
    assert np.array_equal(vc, want)


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("solver", ["GN", "CERES"])
def test_constant_timestamps_sequence(orc, eng, seq_small, solver):
    """A scan whose points all carry the same time (a driver without per-point time): every alpha is 1, the begin-pose
    columns of the GN system are exactly zero and the solve's zero-pivot rule (pseudo-inverse of D, like Eigen's LDLT)
    decides the step; solver CERES sees the same zero columns through its LM damping. Engine against the oracle."""
    from test_gpu_parity import _run_sequence
    from test_gpu_parity_r2 import _compare
    seq = []
    for s in seq_small:
        s = dict(s)
        s["t"] = np.full_like(s["t"], float(s["t"].max()))
        seq.append(s)
    _, ro = _run_sequence(orc, seq, solver, init_num_frames=4)
    _, re_ = _run_sequence(eng, seq, solver, init_num_frames=4)
    wt, wr = _compare(ro, re_)
    print("[device-math] constant timestamps / %s: worst per-frame pose difference %.3e m, %.3e rad" % (solver, wt, wr))
