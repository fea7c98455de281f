"""Comparison of an evaluation with the oracle's at each quantity's own scale.

The normal equations span about 13 orders of magnitude (the line-delay diagonal against the weakest bias and end-knot columns), so
one tolerance relative to the largest entry (helpers.rel) leaves whole blocks unchecked.  Here, with d = diag(H_oracle):
  * J^T J, Jacobi-scaled: |Hg_ij - Ho_ij| / sqrt(d_i d_j) <= tol, structural zeros included; a column with d_i = 0 is exactly 0;
  * J^T r: |gg_i - go_i| <= tol * |r| sqrt(d_i), the Cauchy-Schwarz bound |J_i^T r| <= |J_i| |r| (|r| without the 1e10 sentinels
    of failed projections, whose rows have no derivative);
  * residuals per kind (vision, accelerometer, gyroscope, bias prior) at each kind's own max, the 1e10 sentinels equal position for
    position and left out of the scale;
  * where dense J^T J is too big, products with probes supported on one column block (and on the first and last SO(3) / R^3 knots,
    where the weakest columns are), each output block at its own max.
A failure names the block pair and the indices within it, e.g. `acc_bias[2].y x gravity.z: 3.1e-04`."""
import numpy as np

from openimucameracalibrator_b200 import _capi as capi

TOL = 1e-9
SENTINEL = 1e10
XYZ = "xyz"


class Block:
    def __init__(self, name, start, size, width, labels=None):
        self.name, self.start, self.size, self.width, self.labels = name, start, size, width, labels

    @property
    def stop(self):
        return self.start + self.size

    def entry(self, k):
        """Name of column start + k, e.g. so3[4].y, T_i_c.rz, cam_intrinsics[3]."""
        if self.labels is not None:
            return f"{self.name}.{self.labels[k]}"
        if self.width == 3:
            return f"{self.name}[{k // 3}].{XYZ[k % 3]}" if self.size > 3 else f"{self.name}.{XYZ[k % 3]}"
        return f"{self.name}[{k}]" if self.size > 1 else self.name


def column_blocks(api, flags):
    """The column blocks of the canonical tangent order (the oracle's configure(): so3, r3, T_i_c, gravity, line delay, acc bias,
    gyr bias, acc intrinsics, gyr intrinsics, cam intrinsics, time offset, points), knot counts from get_knots()."""
    so3, r3, ba, bg = api.get_knots()
    sizes = [("so3", 3 * len(so3) if flags & capi.FLAG_SPLINE else 0, 3, None),
             ("r3", 3 * len(r3) if flags & capi.FLAG_SPLINE else 0, 3, None),
             ("T_i_c", 6 if flags & capi.FLAG_T_I_C else 0, 6, ("tx", "ty", "tz", "rx", "ry", "rz")),
             ("gravity", 3 if flags & capi.FLAG_GRAVITY_DIR else 0, 3, None),
             ("line_delay", 1 if (flags & capi.FLAG_CAM_LINE_DELAY) and api.get_line_delay() != 0.0 else 0, 1, None),
             ("acc_bias", 3 * len(ba) if flags & (capi.FLAG_IMU_BIASES | capi.FLAG_ACC_BIAS) else 0, 3, None),
             ("gyr_bias", 3 * len(bg) if flags & (capi.FLAG_IMU_BIASES | capi.FLAG_GYR_BIAS) else 0, 3, None),
             ("acc_intrinsics", 6 if flags & capi.FLAG_IMU_INTRINSICS else 0, 1, None),
             ("gyr_intrinsics", 9 if flags & capi.FLAG_IMU_INTRINSICS else 0, 1, None),
             ("cam_intrinsics", api.num_tangent(capi.FLAG_CAM_INTRINSICS) if flags & capi.FLAG_CAM_INTRINSICS else 0, 1, None),
             ("time_offset", 1 if flags & capi.FLAG_TIME_OFFSET else 0, 1, None),
             ("points", 3 * len(api.get_board_points()) if flags & capi.FLAG_POINTS else 0, 3, None)]
    blocks, off = [], 0
    for name, size, width, labels in sizes:
        if size:
            blocks.append(Block(name, off, size, width, labels))
            off += size
    n = api.num_tangent(flags)
    assert off == n, f"column blocks {[(b.name, b.size) for b in blocks]} sum to {off}, num_tangent({flags}) = {n}"
    return blocks


def _owner(blocks, n):
    own = np.empty(n, dtype=np.int64)
    for k, b in enumerate(blocks):
        own[b.start:b.stop] = k
    return own


def _name(blocks, own, i):
    b = blocks[own[i]]
    return b.entry(i - b.start)


# ---- J^T J --------------------------------------------------------------------------------------------------------------------------
def hessian_errors(H, Ho):
    """E_ij = |H_ij - Ho_ij| / sqrt(d_i d_j), d = diag(Ho); where d_i d_j = 0 the entry must be exact (E = 0 or inf)."""
    H, Ho = np.asarray(H, dtype=np.float64), np.asarray(Ho, dtype=np.float64)
    d = np.diag(Ho)
    assert np.all(d >= 0.0)
    s = np.sqrt(d)
    den = np.outer(s, s)
    diff = np.abs(H - Ho)
    with np.errstate(divide="ignore", invalid="ignore"):
        E = np.where(den > 0.0, diff / np.where(den > 0.0, den, 1.0), np.where(diff == 0.0, 0.0, np.inf))
    return E


def assert_hessian(H, Ho, blocks, tol=TOL, what="J^T J"):
    assert H.shape == Ho.shape
    assert np.array_equal(H, H.T), f"{what} is not exactly symmetric"
    E = hessian_errors(H, Ho)
    if not E.max() <= tol:
        own = _owner(blocks, H.shape[0])
        bad = np.argwhere(E > tol)
        worst = bad[np.argsort(-E[bad[:, 0], bad[:, 1]])]
        worst = [(i, j) for i, j in worst if i <= j][:6]
        lines = [f"{_name(blocks, own, i)} x {_name(blocks, own, j)}: {E[i, j]:.1e}" for i, j in worst]
        raise AssertionError(f"{what}, Jacobi-scaled, exceeds {tol:.0e} in {len(bad)} entries; worst:\n  " + "\n  ".join(lines))
    return float(E.max())


# ---- J^T r --------------------------------------------------------------------------------------------------------------------------
def residual_norm(residuals=None, cost=None):
    """|r| without the sentinels (from the residuals), or sqrt(2 cost) when only the cost is at hand."""
    if residuals is not None:
        r = np.asarray(residuals, dtype=np.float64)
        r = r[r != SENTINEL]
        return float(np.sqrt(np.dot(r, r)))
    return float(np.sqrt(2.0 * cost))


def gradient_errors(g, go, d, rnorm):
    """e_i = |g_i - go_i| / (|r| sqrt(d_i)); a column with d_i = 0 must be exact."""
    g, go = np.asarray(g, dtype=np.float64), np.asarray(go, dtype=np.float64)
    den = rnorm * np.sqrt(np.asarray(d, dtype=np.float64))
    diff = np.abs(g - go)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0.0, diff / np.where(den > 0.0, den, 1.0), np.where(diff == 0.0, 0.0, np.inf))


def assert_gradient(g, go, d, rnorm, blocks, tol=TOL):
    e = gradient_errors(g, go, d, rnorm)
    if not e.max() <= tol:
        own = _owner(blocks, len(e))
        worst = np.argsort(-e)[:6]
        lines = [f"{_name(blocks, own, i)}: {e[i]:.1e}" for i in worst if e[i] > tol]
        raise AssertionError(f"J^T r, scaled by |r| sqrt(diag(J^T J)), exceeds {tol:.0e} in {int((e > tol).sum())} entries; worst:\n  "
                             + "\n  ".join(lines))
    return float(e.max())


# ---- residuals ----------------------------------------------------------------------------------------------------------------------
def residual_kinds(api, n_total):
    """[(kind, start, stop)] in evaluate's residual order: vision, accelerometer, gyroscope, then the bias prior rows."""
    nv, na, ng = api.num_residuals()
    spans = [("vision", 0, nv), ("accelerometer", nv, nv + na), ("gyroscope", nv + na, nv + na + ng)]
    n_prior = api.num_bias_prior_residuals() if hasattr(api.lib, api.prefix + "num_bias_prior_residuals") else 0
    spans.append(("bias_prior", nv + na + ng, nv + na + ng + n_prior))
    assert spans[-1][2] == n_total, (spans, n_total)
    return spans


def residual_kind_errors(r, ro, kinds):
    """{kind: max |r - ro| / max |ro|} over the entries that are not sentinels; the sentinels must match position for position."""
    r, ro = np.asarray(r, dtype=np.float64), np.asarray(ro, dtype=np.float64)
    out = {}
    for kind, a, b in kinds:
        x, y = r[a:b], ro[a:b]
        sent = y == SENTINEL
        if not np.array_equal(sent, x == SENTINEL):
            k = int(np.flatnonzero(sent != (x == SENTINEL))[0])
            raise AssertionError(f"{kind} residual {k}: sentinel mismatch ({x[k]!r} against {y[k]!r})")
        x, y = x[~sent], y[~sent]
        if x.size == 0:
            continue
        scale = np.abs(y).max()
        diff = np.abs(x - y).max()
        out[kind] = float(diff / scale) if scale > 0.0 else (0.0 if diff == 0.0 else np.inf)
    return out


def assert_residuals(r, ro, kinds, tol=TOL):
    errs = residual_kind_errors(r, ro, kinds)
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, "residuals at each kind's own max exceed " + f"{tol:.0e}: " + ", ".join(f"{k}: {v:.1e}" for k, v in bad.items())
    return errs


# ---- one evaluation against the oracle's ---------------------------------------------------------------------------------------------
def assert_scaled_parity(api, flags, ev_o, ev_g, blocks=None, tol=TOL):
    """Residuals, J^T r and J^T J of one evaluation (ev_g) against the oracle's (ev_o), both evaluate(flags, hessian=True) tuples of
    handles loaded alike; `api` (either handle) gives the column blocks and residual counts.  Returns the measured maxima."""
    _, ro, go, Ho = ev_o
    _, rg, gg, Hg = ev_g
    blocks = blocks if blocks is not None else column_blocks(api, flags)
    out = {"residuals": assert_residuals(rg, ro, residual_kinds(api, len(ro)), tol)}
    out["hessian"] = assert_hessian(Hg, Ho, blocks, tol)
    out["gradient"] = assert_gradient(gg, go, np.diag(Ho), residual_norm(ro), blocks, tol)
    return out


# ---- products with block probes -------------------------------------------------------------------------------------------------------
def block_probes(blocks, rng, edge_knots=3):
    """(labels, V): one random probe per column block, plus one per each of the first and last `edge_knots` SO(3) and R^3 knots."""
    n = blocks[-1].stop
    labels, rows = [], []
    for b in blocks:
        v = np.zeros(n); v[b.start:b.stop] = rng.normal(size=b.size)
        labels.append(b.name); rows.append(v)
        if b.name in ("so3", "r3"):
            nk = b.size // 3
            for k in sorted(set(range(min(edge_knots, nk))) | set(range(max(nk - edge_knots, 0), nk))):
                v = np.zeros(n); v[b.start + 3 * k: b.start + 3 * k + 3] = rng.normal(size=3)
                labels.append(f"{b.name}[{k}]"); rows.append(v)
    return labels, np.stack(rows)


def probe_errors(HV, HVo, labels, blocks):
    """{(probe, output block): max |HV - HVo| / max |HVo|} over the output block; an output block that is exactly zero in the oracle's
    product must be exactly zero (0 or inf)."""
    out = {}
    for p, lab in enumerate(labels):
        for b in blocks:
            x, y = HV[p, b.start:b.stop], HVo[p, b.start:b.stop]
            scale, diff = np.abs(y).max(), np.abs(x - y).max()
            out[(lab, b.name)] = float(diff / scale) if scale > 0.0 else (0.0 if diff == 0.0 else np.inf)
    return out


def probe_reference(o, flags, rng):
    """The oracle's side of assert_block_probes (it does not depend on the other handle: reusable across GPU handles)."""
    blocks = column_blocks(o, flags)
    labels, V = block_probes(blocks, rng)
    return dict(flags=flags, blocks=blocks, labels=labels, V=V, HVo=o.normal_matvec(flags, V))


def assert_block_probes(g, ref, tol=TOL):
    """J^T J of `g` against the oracle's (probe_reference) through normal_matvec with block probes.  Returns the error per
    (probe, output block)."""
    errs = probe_errors(g.normal_matvec(ref["flags"], ref["V"]), ref["HVo"], ref["labels"], ref["blocks"])
    bad = sorted(((v, k) for k, v in errs.items() if not v <= tol), reverse=True)
    assert not bad, f"J^T J V with block probes exceeds {tol:.0e} at each output block's own max:\n  " + "\n  ".join(
        f"probe {p} -> {b}: {v:.1e}" for v, (p, b) in bad[:8])
    return errs
