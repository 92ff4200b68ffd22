"""TEST INFRASTRUCTURE ONLY -- float64 model of the first-order derivatives of a mode's effective index.

The diagonal operator A = P Q of ``restatement.assemble_diagonal`` is not symmetric, but its left eigenvectors come for free
from the right ones: with q = Q v (the transverse-H intermediate of the field recovery) and J [a; b] = [b; -a],

    w = G J q,   G = diag(sf_x dlf_x * sb_y dlb_y  (Ex sites),  sb_x dlb_x * sf_y dlf_y  (Ey sites))

is a left eigenvector, A^T w = lambda w.  G holds the complex-stretched primal / dual cell lengths (``st["slen"]``); at a PMC
wall the first dual length is halved (the row of the backward difference there is 2 / dl_b).  First-order perturbation theory
then gives every derivative of lambda = -n^2 from one solve:

    d lambda = w^T (dA) v / (w^T v),      dn = -d lambda / (2 n),      n_group = Re n + f Re(dn/df).

A is a quadratic polynomial in the 1-D difference coefficients (the quartic terms of P Q cancel because Dxb Dyb = Dyb Dxb),
so its derivative along a coefficient direction dc is exactly [A(c + dc) - A(c - dc)] / 2.  Every coefficient is
1 / (s k0 dl) with s = kappa + i sigma / (omega eps0), so s k0 = (kappa omega + i sigma / eps0) / c0 and
f dc/df = -c kappa / s exactly.  The permittivity derivatives are taken with respect to the caller's eps_cross at fixed PML
stretch (the strip-averaged PML speeds are held constant), through the bend congruence eps' = J eps J^T / det J; cells whose
input is PEC-valued report 0.  The device computes the same quantities (tidy3d_b200/csrc/derivatives.cuh).
"""
from __future__ import annotations

import numpy as np

from oracle import restatement as R


def metric(st):
    """The diagonal G of w = G J Q v, shape (2N,)."""
    (sfx, sbx), (sfy, sby) = [(np.array(a, complex), np.array(b, complex)) for a, b in st["slen"]]
    if st["pmc"][0]:
        sbx[0] *= 0.5
    if st["pmc"][1]:
        sby[0] *= 0.5
    return np.r_[(sfx[:, None] * sby[None, :]).ravel(), (sbx[:, None] * sfy[None, :]).ravel()]


def left_vector(st, Q, v):
    """Left eigenvector w = G J (Q v) belonging to the right eigenvector v (any scale)."""
    n = st["n"]
    h = Q @ v
    return metric(st) * np.r_[h[n:], -h[:n]]


def coef_direction(st, freq):
    """f dc/df of the four 1-D coefficient vectors of both axes: -c kappa / s (kappa = Re s)."""
    out = []
    for ax in range(2):
        lf, lb = st["slen"][ax]
        f0, f1, b0, bm = st["coef"][ax]
        n = f0.size
        c0 = st["new_coords"][ax]
        dl_f = c0[1:] - c0[:-1]
        dl_b = np.hstack((dl_f[0], (dl_f[:-1] + dl_f[1:]) / 2))
        s_f, s_b = lf / dl_f, lb / dl_b
        rf, rb = s_f.real / s_f, s_b.real / s_b
        out.append((-f0 * rf, -f1 * rf, -b0 * rb, -bm * rb) if n > 1 else (f0, f1, b0, bm))
    return out


def _with_coef(st, coef):
    s = dict(st)
    s["coef"] = coef
    return s


def dA_dfreq(st, freq):
    """dA/df at fixed permittivity (exact: A is quadratic in the coefficients)."""
    d = coef_direction(st, freq)
    plus = [tuple(c + e for c, e in zip(cs, ds)) for cs, ds in zip(st["coef"], d)]
    minus = [tuple(c - e for c, e in zip(cs, ds)) for cs, ds in zip(st["coef"], d)]
    Ap = R.assemble_diagonal(_with_coef(st, plus))[2]
    Am = R.assemble_diagonal(_with_coef(st, minus))[2]
    return (Ap - Am) / (2.0 * freq)


def dlam_deps_solver(st, P, v, w):
    """w^T (dA/d eps'_aa(g)) v for the solver-frame diagonal permittivity, shape (3, N) (not yet divided by w^T v)."""
    n = st["n"]
    e = st["eps"]
    dxf, dxb, dyf, dyb = R.d_matrices(st)
    r = P.T @ w
    v1, v2 = v[:n], v[n:]
    d_xx = -r[n:] * v1
    d_yy = r[:n] * v2
    z = dxf.T @ w[:n] + dyf.T @ w[n:]
    # s = Dxb q2 - Dyb q1 = -(Dxb exx v1 + Dyb eyy v2)
    s = -(dxb @ (e[0, 0] * v1) + dyb @ (e[1, 1] * v2))
    iez = 1.0 / e[2, 2]
    d_zz = -(iez**2) * z * s
    return np.stack((d_xx, d_yy, d_zz))


def derivatives(eps_cross, coords, freq, mode_spec, v, lam, symmetry=(0, 0), mu_cross=None, eps_dfreq=None):
    """Derivatives of one mode (right eigenvector v = [Ex; Ey] of the solver-frame operator, eigenvalue lam = -n^2).

    Returns dict(dlam_dfreq, dn_dfreq, n_group, dn_deps (3, nx, ny), w, residual) with n = sqrt(-lam) * knorm the reported
    effective index; eps_dfreq (nine components in the eps_cross layout, or None) adds the material dispersion."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    if st["tensorial"]:
        raise NotImplementedError("derivatives: tensorial problems are out of scope")
    P, Q, A = R.assemble_diagonal(st)
    v = np.asarray(v, complex)
    w = left_vector(st, Q, v)
    wv = w @ v
    g = dlam_deps_solver(st, P, v, w)
    # caller frame: eps'_aa = J_aa^2 eps_aa / det J (diagonal Jacobian)
    jac = st["jac_e"]
    det = jac[0, 0] * jac[1, 1] * jac[2, 2]
    for a in range(3):
        g[a] *= jac[a, a] ** 2 / det
    raw = np.stack([np.asarray(eps_cross[i], complex).ravel() for i in (0, 4, 8)])
    g[raw.real <= 0.9 * R.PEC_VAL] = 0.0
    dlam_deps = g / wv
    dlam_df = (w @ (dA_dfreq(st, freq) @ v)) / wv
    if eps_dfreq is not None:
        de = np.stack([np.asarray(eps_dfreq[i], complex).ravel() for i in (0, 4, 8)])
        dlam_df = dlam_df + np.sum(dlam_deps * de)
    nsol = np.sqrt(-lam + 0j)
    if nsol.real < 0:
        nsol = -nsol
    knorm = st["knorm"]
    dn_df = -dlam_df / (2 * nsol) * knorm
    n = nsol * knorm
    res = np.linalg.norm(A.T @ w - lam * w) / np.linalg.norm(lam * w)
    return dict(dlam_dfreq=dlam_df, dn_dfreq=dn_df, n_group=n_group(n, dn_df, freq),
                dn_deps=(-dlam_deps / (2 * nsol) * knorm).reshape(3, st["nx"], st["ny"]), w=w, residual=res)


def n_group(n, dn_dfreq, freq):
    """Group index n_g = Re n + f Re(dn/df): what ModeData._group_index_post_process approximates by finite differences."""
    return np.real(n) + freq * np.real(dn_dfreq)
