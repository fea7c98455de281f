"""Dense high-precision reference of the damped normal-equation solve (icc_solve_normal_equations) and the cases the solver tests run.

The solve: A = S H S + D, b = -S g, y = A^-1 b, delta = S y, with S = diag(1 / (1 + sqrt(H_ii))) (I without Jacobi scaling) and
D = diag(clamp(H_ii s_i^2, min_lm_diagonal, max_lm_diagonal) / radius)  (Ceres' LevenbergMarquardtStrategy).

Bars (u = 2^-53):
  * backward error.  A blocked LDL^T in any summation order (tensor-core tiles, atomics into the reduced systems) is backward
    stable: the computed y solves (A + dA) y = b with |dA| <= g_m |L||D||L^T|, m the longest inner product (the border rows:
    m ~ n).  The probabilistic form of that bound (Higham & Mary 2019) replaces g_m by lambda sqrt(m) u, so the normwise backward
    error eta = ||A y - b|| / (||A|| ||y|| + ||b||) (infinity norms) is bounded by ETA_LAMBDA sqrt(n) u rho, with the growth factor
    rho = || |L||L^T| || / ||A|| of the reference Cholesky factor.  The same bound row by row gives the componentwise (Oettli-Prager)
    backward error omega = max_i |A y - b|_i / (|A||y| + |b|)_i <= ETA_LAMBDA sqrt(n) u rho_c, rho_c = max_i (|L||L^T||y|)_i / (|A||y|)_i.
    omega is the sharper test: an error in one coupling entry shows in its own row instead of being divided by ||A|| ||y||.
  * forward error (in the scaled unknowns y): ||y - y_ref|| / ||y_ref|| <= 2 kappa eta / (1 - kappa eta) plus the reference's own
    error; checked against 4 kappa eta_bar, and skipped where kappa eps > 1e-2 (nothing meaningful is left to compare).
  * model change -(g^T delta + delta^T H delta / 2): the solver forms it as (y^T D y - y^T S g) / 2, which equals the expression only
    for an exact solve; the two differ by y^T r / 2 (r = A y - b) plus the rounding of an n-term sum.
"""
from __future__ import annotations

import dataclasses
import functools

import numpy as np
import scipy.linalg as sla
from scipy.sparse.linalg import LinearOperator, onenormest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import synthetic as syn

U = np.finfo(np.float64).eps / 2
EPS = np.finfo(np.float64).eps
ETA_LAMBDA = 8.0
F_STAGE1 = capi.FLAG_SPLINE | capi.FLAG_T_I_C
F_STAGE2 = capi.FLAG_CAM_LINE_DELAY
F_ALL = F_STAGE1 | capi.FLAG_GRAVITY_DIR | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_IMU_BIASES
F_POINTS = F_STAGE1 | capi.FLAG_POINTS
F_WIDE = F_STAGE1 | capi.FLAG_IMU_BIASES | capi.FLAG_GRAVITY_DIR


# ---- datasets and cases ---------------------------------------------------------------------------------------------------
DATA = {
    "tiny": {},
    "tiny20": dict(n_frames=20),                                    # with the most chunks, every leaf has exactly kd + 1 columns
    "tiny_gs": dict(line_delay_truth=0.0),                           # global shutter: vision has zero weight
    "dt_04_07": dict(dt_so3_s=0.04, dt_r3_s=0.07),                   # kd 47
    "dt_09_05": dict(dt_so3_s=0.09, dt_r3_s=0.05),                   # kd 47
    "kd62": dict(n_frames=60, dt_so3_s=0.06, dt_r3_s=0.02),          # the widest band measured that still takes P = 2
    "kd110": dict(n_frames=60, dt_so3_s=0.1175, dt_r3_s=0.02),       # the widest band any plan takes (P = 1, a 378-column leaf)
    "kd110_long": dict(n_frames=400, dt_so3_s=0.1175, dt_r3_s=0.02),  # the same band over 2400 knot columns: no plan
    "kd113": dict(n_frames=60, dt_so3_s=0.125, dt_r3_s=0.02),        # no plan at any length
    "kd68_100s": dict(n_frames=3000, dt_so3_s=0.0625, dt_r3_s=0.02),  # kd 68 over 19 827 knot columns: one chunk takes at most 15 076
    "tiny1150": dict(n_frames=1150),                                 # 4632 knot columns: the planner takes 64 chunks (dense n = 4638)
    "wide200": dict(n_frames=400, fps=2.0, dt_so3_s=0.5, dt_r3_s=0.5, imu_rate_hz=50.0, seed=41),   # 200 s, 2 x 23 bias knots
    "points396": dict(grid=(13, 10)),                                # 130 board points: 396 border columns, the widest that fits
    "points402": dict(grid=(12, 11)),                                # 132 board points: 402 border columns, no plan
    "cfg2": 2,
    "cfg4": 4,
}


@functools.lru_cache(maxsize=None)
def dataset(name):
    spec = DATA[name]
    return syn.make_dataset(syn.CONFIGS[spec] if isinstance(spec, int) else syn.tiny_config(**spec))


def load(api, name, known_gravity=True):
    capi.load_dataset(api, dataset(name), known_gravity=known_gravity)
    return api


@dataclasses.dataclass(frozen=True)
class Case:
    id: str
    data: str
    flags: int
    chunks: int = 0
    radius: float = 1e4
    jacobi: int = 1
    known_gravity: bool = True


MAX_CHUNKS = 1 << 11    # clamped by the planner to the most chunks whose leaves keep kd + 1 columns


def _plan_cases():
    out = [Case(f"cfg2-chunks{c if c else 'auto'}", "cfg2", F_STAGE1, c) for c in (0, 1, 2, 3, 4, 5, 7, 8, 16, 31)]
    return out + [Case("cfg2-chunks-max", "cfg2", F_STAGE1, MAX_CHUNKS)]


CASES = _plan_cases() + [
    # borders
    Case("nb0-spline", "tiny", capi.FLAG_SPLINE),
    Case("nb1-spline-line-delay", "tiny", capi.FLAG_SPLINE | capi.FLAG_CAM_LINE_DELAY),
    Case("stage1", "tiny", F_STAGE1),
    Case("all-biases", "tiny", F_ALL, known_gravity=False),
    Case("wide200-hbm-borders", "wide200", F_WIDE, known_gravity=False),
    Case("P64-dense", "tiny1150", F_STAGE1),
    Case("points396-unstaged", "points396", F_POINTS),
    # border only (no knot columns)
    Case("nk0-T_i_c", "tiny", capi.FLAG_T_I_C),
    Case("nk0-line-delay", "tiny", F_STAGE2),
    Case("nk0-gravity-acc-bias", "tiny", capi.FLAG_GRAVITY_DIR | capi.FLAG_ACC_BIAS, known_gravity=False),
    # band widths
    Case("kd47-dt-04-07", "dt_04_07", F_STAGE1),
    Case("kd47-dt-09-05", "dt_09_05", F_STAGE1),
    Case("kd62-two-chunks", "kd62", F_STAGE1),
    Case("kd110-one-chunk", "kd110", F_STAGE1),
    Case("smallest-leaf", "tiny20", F_STAGE1, MAX_CHUNKS),
    # damping
    Case("radius-1e-3", "tiny", F_STAGE1, radius=1e-3),
    Case("radius-1e16", "tiny", F_STAGE1, radius=1e16),
    Case("no-jacobi-scaling", "tiny", F_STAGE1, jacobi=0),
    Case("global-shutter-radius-1e16", "tiny_gs", F_STAGE1, radius=1e16),
]

# config 4 at full size (checked through J^T J products: a dense H would be 1.2 GB)
FULLSIZE_CHUNKS = (0, 64, 127)
# shapes no plan fits: (data, flags, where the refusal comes from)
UNFIT = [("points402", F_POINTS, "solve"), ("kd110_long", F_STAGE1, "configure"), ("kd113", F_STAGE1, "configure"),
         ("kd68_100s", F_STAGE1, "configure")]


def single_chunk_max_columns(kd):
    """Longest knot band one chunk takes (no border): the level-0 back-substitution holds (nbl + 4) + 4 + (nk + 1 + 4) + (128 + kd)(kd + 1)
    + 128 doubles (+ 64 B) in shared memory, within 230 000 B, i.e. nk <= 28 600 - (128 + kd)(kd + 1)."""
    return 28600 - (128 + kd) * (kd + 1)


# ---- the reference ----------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class System:
    A: np.ndarray          # float64, as the solver forms it
    b: np.ndarray
    s: np.ndarray
    dlm: np.ndarray        # LM diagonal D
    A_ld: np.ndarray       # long double
    b_ld: np.ndarray


def lm_system(H, g, radius, jacobi=1, min_diag=1e-6, max_diag=1e32) -> System:
    d = np.diag(H).copy()
    s = 1.0 / (1.0 + np.sqrt(d)) if jacobi else np.ones_like(d)
    dlm = np.clip(d * s * s, min_diag, max_diag) / radius
    A = s[:, None] * H * s[None, :]
    A[np.diag_indices_from(A)] += dlm
    b = -s * g
    sl = s.astype(np.longdouble)
    A_ld = sl[:, None] * H.astype(np.longdouble) * sl[None, :]
    A_ld[np.diag_indices_from(A_ld)] += dlm.astype(np.longdouble)
    return System(A, b, s, dlm, A_ld, b.astype(np.longdouble))


def residual(sys_: System, y) -> np.ndarray:
    return (sys_.A_ld @ np.asarray(y, dtype=np.longdouble)) - sys_.b_ld


def componentwise_error(sys_: System, y) -> float:
    """Oettli-Prager componentwise backward error max_i |A y - b|_i / (|A||y| + |b|)_i (0/0 = 0: a knot no residual touches has
    H_ii = g_i = 0, so its row of A is the LM diagonal alone and y_i = 0 solves it exactly)."""
    r = np.abs(residual(sys_, y))
    den = np.abs(sys_.A_ld) @ np.abs(np.asarray(y, dtype=np.longdouble)) + np.abs(sys_.b_ld)
    zero = den == 0
    assert not np.any(r[zero] != 0), "a nonzero residual in a row with |A||y| + |b| = 0"
    return float((r[~zero] / den[~zero]).max()) if np.any(~zero) else 0.0


def backward_error(sys_: System, y) -> float:
    r = residual(sys_, y)
    nA = float(np.abs(sys_.A_ld).sum(axis=1).max())
    return float(np.abs(r).max()) / (nA * float(np.abs(y).max()) + float(np.abs(sys_.b).max()))


@dataclasses.dataclass
class Reference:
    y: np.ndarray
    delta: np.ndarray
    kappa: float           # infinity-norm condition number of A (estimated)
    rho: float             # || |L||L^T| || / ||A||
    eta_bar: float
    rho_c: float           # max_i (|L||L^T||y|)_i / (|A||y|)_i
    omega_bar: float
    factor: tuple


def reference(sys_: System, refine=3) -> Reference:
    """float64 Cholesky + iterative refinement with the residual in long double."""
    c = sla.cho_factor(sys_.A, lower=True)
    y = sla.cho_solve(c, sys_.b)
    for _ in range(refine):
        y = y - sla.cho_solve(c, residual(sys_, y).astype(np.float64))
    L = np.tril(c[0])
    absL = np.abs(L)
    nA = float(np.abs(sys_.A).sum(axis=1).max())
    rho = float((absL @ (absL.T @ np.ones(len(y)))).max()) / nA
    n = len(y)
    inv = LinearOperator((n, n), matvec=lambda v: sla.cho_solve(c, np.ravel(v)), rmatvec=lambda v: sla.cho_solve(c, np.ravel(v)), dtype=np.float64)
    kappa = nA * float(onenormest(inv)) if n > 1 else 1.0     # A symmetric: ||A^-1||_inf = ||A^-1||_1
    rho_c = float(((absL @ (absL.T @ np.abs(y))) / np.maximum(np.abs(sys_.A) @ np.abs(y), np.finfo(float).tiny)).max())
    return Reference(y, sys_.s * y, kappa, rho, eta_bar(n, rho), rho_c, eta_bar(n, rho_c), c)


def eta_bar(n, rho=1.0) -> float:
    return ETA_LAMBDA * np.sqrt(max(n, 1)) * U * max(rho, 1.0)


def model_change(H, g, delta) -> float:
    """-(g^T delta + delta^T H delta / 2) in long double."""
    d = np.asarray(delta, dtype=np.longdouble)
    return float(-(np.asarray(g, dtype=np.longdouble) @ d + 0.5 * (d @ (np.asarray(H, dtype=np.longdouble) @ d))))


def model_change_bar(sys_: System, y, eta_b) -> float:
    """|solver's (y^T D y - y^T S g) / 2  -  model_change(delta)| <= ||y||_1 ||r|| / 2 + n u sum |terms|, with ||r|| at the bar."""
    nA = float(np.abs(sys_.A).sum(axis=1).max())
    r_bar = eta_b * (nA * float(np.abs(y).max()) + float(np.abs(sys_.b).max()))
    terms = float(np.sum(sys_.dlm * y * y + np.abs(y * sys_.b)))
    n = len(y)
    return 0.5 * float(np.abs(y).sum()) * r_bar + 2 * (n + 4) * U * terms


def cholesky_solve(sys_: System) -> np.ndarray:
    """Plain float64 Cholesky solve, no refinement."""
    return sla.cho_solve(sla.cho_factor(sys_.A, lower=True), sys_.b)


def perturbed_solution(sys_: System, i, j, rel=1e-9):
    """Solution of the system with the coupling entry (i, j) (and its mirror) scaled by 1 + rel: a subtly wrong solve."""
    A = sys_.A.copy()
    A[i, j] *= 1.0 + rel
    A[j, i] = A[i, j]
    return sla.cho_solve(sla.cho_factor(A, lower=True), sys_.b)


def strongest_coupling(sys_: System, y, rows, cols):
    """(i, j) with i in rows, j in cols, i != j, maximising |A_ij y_j| / (|A||y|)_i: the entry whose error moves row i's residual most."""
    rows, cols = np.asarray(rows), np.asarray(cols)
    W = np.abs(sys_.A[np.ix_(rows, cols)] * y[cols][None, :]) / (np.abs(sys_.A[rows]) @ np.abs(y))[:, None]
    W[rows[:, None] == cols[None, :]] = 0.0
    a, b = np.unravel_index(int(np.argmax(W)), W.shape)
    return int(rows[a]), int(cols[b])


def banded_bordered_hessian(nk, kd, nb, rows=None, seed=0):
    """A J^T J with the solver's structure: every row touches a window of kd + 1 consecutive knot columns and a few border
    columns, with column norms spread over six decades (as the spline knots, T_i_c and the biases are)."""
    rng = np.random.default_rng(seed)
    n = nk + nb
    rows = rows or 4 * n
    J = np.zeros((rows, n))
    for r in range(rows):
        a = rng.integers(0, max(1, nk - kd))
        J[r, a:a + kd + 1] = rng.normal(size=min(kd + 1, nk - a))
        if nb:
            k = rng.integers(0, nb, size=min(nb, 3))
            J[r, nk + k] = rng.normal(size=k.size)
    J *= 10.0 ** rng.uniform(-1, 1, size=n)[None, :]
    return J.T @ J, J.T @ rng.normal(size=rows)


# ---- the update statement (update_kernel's Plus) ----------------------------------------------------------------------------
def _qmul(a, b):
    ax, ay, az, aw = a; bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def so3_exp_quat(phi):
    phi = np.asarray(phi, dtype=np.float64)
    th = float(np.linalg.norm(phi))
    if th < 1e-10:
        v = 0.5 * phi
        return np.array([v[0], v[1], v[2], 1.0]) / np.sqrt(1.0 + v @ v)
    k = np.sin(0.5 * th) / th
    return np.array([k * phi[0], k * phi[1], k * phi[2], np.cos(0.5 * th)])


def se3_exp(xi):
    """Sophus SE3::exp, tangent (upsilon, omega) -> (quaternion x,y,z,w, translation)."""
    ups, om = np.asarray(xi[:3], dtype=np.float64), np.asarray(xi[3:], dtype=np.float64)
    q = so3_exp_quat(om)
    th = float(np.linalg.norm(om))
    if th < 1e-10:
        return q, syn.quat_xyzw_to_matrix(q) @ ups
    K = syn._hat(om)
    V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * (K @ K)
    return q, V @ ups


def plus(state, delta, layout, max_ba=1.0, max_bg=0.1):
    """Plus(x, delta) as update_kernel applies it: SO(3) knots q (x) exp(d) (right), R^3 knots + d, T_i_c by the SE(3) exponential on
    the right, gravity / line delay + d, bias knots + d projected onto the box [-max, max]."""
    so3, r3, ba, bg, T, grav, ld = (np.array(x, dtype=np.float64, copy=True) for x in state)
    c = 0
    if layout["spline"]:
        for k in range(len(so3)):
            q = _qmul(so3[k], so3_exp_quat(delta[c:c + 3])); so3[k] = q / np.linalg.norm(q); c += 3
        for k in range(len(r3)):
            r3[k] += delta[c:c + 3]; c += 3
    if layout["tic"]:
        dq, dt = se3_exp(delta[c:c + 6]); c += 6
        q = T[:4]
        R = syn.quat_xyzw_to_matrix(q)
        qn = _qmul(q, dq)
        T = np.concatenate([qn / np.linalg.norm(qn), T[4:] + R @ dt])
    if layout["gravity"]:
        grav = grav + delta[c:c + 3]; c += 3
    if layout["line_delay"]:
        ld = ld + delta[c]; c += 1
    if layout["acc_bias"]:
        ba = np.clip(ba + delta[c:c + 3 * len(ba)].reshape(-1, 3), -max_ba, max_ba); c += 3 * len(ba)
    if layout["gyr_bias"]:
        bg = np.clip(bg + delta[c:c + 3 * len(bg)].reshape(-1, 3), -max_bg, max_bg); c += 3 * len(bg)
    assert c == len(delta), (c, len(delta))
    return so3, r3, ba, bg, T, grav, ld
