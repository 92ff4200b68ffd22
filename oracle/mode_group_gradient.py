"""TEST INFRASTRUCTURE ONLY -- float64 model of the permittivity gradient of each mode's group index.

Extends ``oracle/mode_derivatives.py`` (first order) and ``oracle/mode_dispersion.py`` (the correction x).  Work in the scaled
direction ' = f d/df of DESIGN §4; d_g is d / d eps_aa at one Yee site g of the caller's eps_cross, taken at fixed d eps / df
and fixed PML stretch.  The operator is A = P(iez, mu) Q(exx, eyy) with p = (exx, eyy, iez) the solver-frame triple, so the
gradient of lambda at g is

    d_g lambda = chi_a D_a(w, v) / w^T v,   D_a(w, e) = w^T (dA/dp_a(g)) e,   chi = (dp_a / d eps_aa) = (1/je, 1/je, -iez^2 je)

(je: bend factor, 1 without a bend).  D_a is quadratic in the 1-D coefficients c and affine in p, so its derivative D_a' at
fixed (w, e) is exactly [D_a(c + c') - D_a(c - c')]/2 + [D_a(p + p') - D_a(p - p')]/2 with unit steps.

The left eigenvector w = G J Q v holds for every f and eps (it is structural), so w' = G'J Q v + G J Q'v + G J Q v' needs no
adjoint solve.  G holds the complex-stretched lengths l = s dl with s = kappa + i sigma / (omega eps0): l' = -i Im l.  The
correction x of the dispersion pass is v' up to a multiple of v, and a multiple a v in v' (with the a w it brings into w')
drops out of

    d_g lambda' = [ chi_a (D_a(w_hat, v) + D_a(w, x) + D_a'(w, v)) + chi_a' D_a(w, v) - chi_a D_a(w, v) (w_hat^T v + w^T x) / w^T v ]
                  / w^T v,
    w_hat = G'J Q v + G J Q'v + G J Q x,   chi' = (0, 0, -2 iez iez' je),

which is (d_g lambda)' written out (the mixed partials commute because the eps step does not depend on f).  With
s = sqrt(-lambda), n = knorm s, lambda_f = lambda' / f:

    d_g n = -knorm d_g lambda / (2 s),
    d_g (dn/df) = knorm [ -d_g lambda' / (2 s f) - lambda_f d_g lambda / (4 s^3) ],
    d_g n_group = Re d_g n + f Re d_g (dn/df)   (a real change of eps).

PEC-valued cells report 0.  The device computes the same quantities (tidy3d_b200/csrc/derivatives.cuh, group_grad_kernel).
"""
from __future__ import annotations

import numpy as np

from oracle import mode_derivatives as D
from oracle import mode_dispersion as MD
from oracle import restatement as R


def assemble_at(st, cdir=None, sc=0.0, pdir=None, sp_=0.0):
    """(P, Q, A) at c + sc cdir and p + sp_ pdir (p = (exx, eyy, iez) of the solver frame)."""
    s = dict(st)
    if cdir is not None:
        s["coef"] = [tuple(c + sc * d for c, d in zip(cs, ds)) for cs, ds in zip(st["coef"], cdir)]
    if pdir is not None:
        e = np.array(st["eps"], complex, copy=True)
        e[0, 0] = e[0, 0] + sp_ * pdir[0]
        e[1, 1] = e[1, 1] + sp_ * pdir[1]
        e[2, 2] = 1.0 / (1.0 / st["eps"][2, 2] + sp_ * pdir[2])
        s["eps"] = e
    return R.assemble_diagonal(s), s


def metric_prime(st):
    """G' of w = G J Q v along ' = f d/df: every stretched length l = s dl moves as l' = -i Im l."""
    (sfx, sbx), (sfy, sby) = [(np.array(a, complex), np.array(b, complex)) for a, b in st["slen"]]
    if st["pmc"][0]:
        sbx[0] *= 0.5
    if st["pmc"][1]:
        sby[0] *= 0.5
    d = lambda l: -1j * l.imag  # noqa: E731
    return np.r_[(d(sfx)[:, None] * sby[None, :] + sfx[:, None] * d(sby)[None, :]).ravel(),
                 (d(sbx)[:, None] * sfy[None, :] + sbx[:, None] * d(sfy)[None, :]).ravel()]


def q_prime(st, freq, p1):
    """Q' (scaled): Q is quadratic in c and linear in (exx, eyy), so unit-step central differences are exact."""
    c1 = D.coef_direction(st, freq)
    Q1 = 0.5 * (assemble_at(st, c1, 1.0)[0][1] - assemble_at(st, c1, -1.0)[0][1])
    return Q1 + 0.5 * (assemble_at(st, None, 0.0, p1, 1.0)[0][1] - assemble_at(st, None, 0.0, p1, -1.0)[0][1])


def w_prime(st, Q, Q1, v, vdot):
    """G'J Q v + G J Q'v + G J Q vdot: the exact w' when vdot = v' (w_hat of the module docstring when vdot = x)."""
    n = st["n"]
    J = lambda h: np.r_[h[n:], -h[:n]]  # noqa: E731
    return metric_prime(st) * J(Q @ v) + D.metric(st) * J(Q1 @ v + Q @ vdot)


def forms(st, P, e, w):
    """D_a(w, e) = w^T (dA / dp_a(g)) e for p = (exx, eyy, iez) at every cell g, shape (3, N); P from the same st."""
    n = st["n"]
    ex, ey = st["eps"][0, 0], st["eps"][1, 1]
    dxf, dxb, dyf, dyb = R.d_matrices(st)
    r = P.T @ w
    e1, e2 = e[:n], e[n:]
    z = dxf.T @ w[:n] + dyf.T @ w[n:]
    s = -(dxb @ (ex * e1) + dyb @ (ey * e2))  # = Dxb q2 - Dyb q1
    return np.stack((-r[n:] * e1, r[:n] * e2, z * s))


def group_gradient(eps_cross, coords, freq, mode_spec, v, lam, symmetry=(0, 0), mu_cross=None, eps_dfreq=None, x=None):
    """Permittivity gradients of one mode (right eigenvector v = [Ex; Ey] of the solver-frame operator, eigenvalue lam = -n^2,
    which may be a Ritz value).  x: the scaled correction (v' up to a multiple of v), or None to solve it as the dispersion
    model does.  Returns dict(dlam_deps, d2lam_dfreq_deps (scaled: d_g lambda'), dn_deps, d2n_dfreq_deps (1/Hz), dng_deps,
    each (3, nx, ny), and w, w_hat, x, lam1 = lambda')."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    if st["tensorial"]:
        raise NotImplementedError("group-index gradient: tensorial problems are out of scope")
    nx, ny = st["nx"], st["ny"]
    (P, Q, A), _ = assemble_at(st)
    v = np.asarray(v, complex)
    w = D.left_vector(st, Q, v)
    wv = w @ v
    p1, p2 = MD.material_directions(st, eps_cross, freq, eps_dfreq, None)
    A1, _ = MD.scaled_operators(st, freq, p1, p2)
    a1v = A1 @ v
    l1 = (w @ a1v) / wv
    if x is None:
        r = -(a1v - l1 * v)
        x, _ = MD.correction(A, lam, v, w, r - v * (w @ r) / wv)
    x = np.asarray(x, complex)
    w_hat = w_prime(st, Q, q_prime(st, freq, p1), v, x)

    d0 = forms(st, P, v, w)
    c1 = D.coef_direction(st, freq)
    e = forms(st, P, v, w_hat) + forms(st, P, x, w)
    for cdir, pdir in ((c1, None), (None, p1)):
        (Pp, _, _), sp_st = assemble_at(st, cdir, 1.0, pdir, 1.0)
        (Pm, _, _), sm_st = assemble_at(st, cdir, -1.0, pdir, -1.0)
        e = e + 0.5 * (forms(sp_st, Pp, v, w) - forms(sm_st, Pm, v, w))

    jac = st["jac_e"]
    det = jac[0, 0] * jac[1, 1] * jac[2, 2]
    iez = 1.0 / st["eps"][2, 2]
    chi = np.stack((jac[0, 0] ** 2 / det, jac[1, 1] ** 2 / det, -(iez**2) * jac[2, 2] ** 2 / det)) * np.ones((3, nx * ny))
    chi1 = np.zeros((3, nx * ny), complex)
    chi1[2] = -2 * iez * p1[2] * jac[2, 2] ** 2 / det
    g0 = chi * d0
    g1 = chi * e + chi1 * d0 - g0 * (w_hat @ v + w @ x) / wv
    raw = np.stack([np.asarray(eps_cross[i], complex).ravel() for i in (0, 4, 8)])
    pec = raw.real <= 0.9 * R.PEC_VAL
    g0[pec] = 0.0
    g1[pec] = 0.0
    dlam, dlam1 = g0 / wv, g1 / wv
    out = convert(st["knorm"], freq, lam, l1, dlam, dlam1)
    shape = (3, nx, ny)
    return dict(dlam_deps=dlam.reshape(shape), d2lam_dfreq_deps=dlam1.reshape(shape), w=w, w_hat=w_hat, x=x, lam1=l1,
                **{k: val.reshape(shape) for k, val in out.items()})


def convert(knorm, freq, lam, lam1, dlam, dlam1):
    """dn_deps, d2n_dfreq_deps (1/Hz) and dng_deps from lambda, lambda' and the gradients d_g lambda, d_g lambda' (scaled)."""
    s = np.sqrt(-lam + 0j)
    if s.real < 0:
        s = -s
    dn = -knorm * dlam / (2 * s)
    d2n = knorm * (-dlam1 / (2 * s * freq) - (lam1 / freq) * dlam / (4 * s**3))
    return dict(dn_deps=dn, d2n_dfreq_deps=d2n, dng_deps=dn.real + freq * d2n.real)
