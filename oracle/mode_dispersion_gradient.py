"""TEST INFRASTRUCTURE ONLY -- float64 model of the permittivity gradient of each mode's group-velocity dispersion.

Extends ``oracle/mode_group_gradient.py`` (forms D_a, chi, w_hat) and ``oracle/mode_fourth_order.py`` (x2, w_hat2).  Work in
t = (f_new - f) / f with the Taylor coefficients c_1 = c', c_2 = c''/2, p_1 = p', p_2 = p''/2 (' = f d/df, X'' = f^2 d^2X/df^2)
of the 1-D coefficients c and of p = (exx, eyy, iez) of the solver frame.  With v(t) = v + t x + t^2 x2 and
w(t) = w + t w_hat + t^2 w_hat2, the error of N/D = w(t)^T A(t) v(t) / w(t)^T v(t) is O(t^6) and its t^0..t^2 coefficients
are stationary in all six vectors, so the gradient of lambda_2 = lambda''/2 at a Yee site g is the explicit partial at
fixed vectors:

    d_g lambda_2 = [t^2] E(t) / D(t) = E_2 / D_0 - (E_1 D_1 + E_0 D_2) / D_0^2 + E_0 D_1^2 / D_0^3,

    E(t) = chi_a(t) D_a(t)(w(t), v(t)),   D_0 = w^T v,  D_1 = w_hat^T v + w^T x,  D_2 = w_hat2^T v + w_hat^T x + w^T x2,
    E_0 = chi D(w, v),
    E_1 = chi [D(w_hat, v) + D(w, x) + D_1(w, v)] + chi_1 D(w, v),
    E_2 = chi [D(w_hat2, v) + D(w_hat, x) + D(w, x2) + D_1(w_hat, v) + D_1(w, x) + D_2(w, v)]
          + chi_1 [D(w_hat, v) + D(w, x) + D_1(w, v)] + chi_2 D(w, v).

D_k is the t^k coefficient of the form at (c(t), p(t)).  D_a is quadratic in c and affine in p, so with unit steps
D_1 = [D(c + c_1) - D(c - c_1)]/2 + [D(p + p_1) - D(p - p_1)]/2 and D_2 = D_c[c_2] + D_cc[c_1, c_1] + D_p[p_2] + D_cp[c_1, p_1]
(D_cc[c_1, c_1] = [D(c + c_1) + D(c - c_1)]/2 - D, D_cp the four-point mixed difference at (+-c_1, +-p_1)).  Only chi_zz moves
with f: chi_zz(t) = -je iez(t)^2, so chi_1 = -2 je iez iez_1 and chi_2 = -je (2 iez iez_2 + iez_1^2).  With s = sqrt(-lambda)
(scaled derivatives): d s = -d lambda / (2 s), d s' = -(d lambda' + 2 s' d s) / (2 s), d s'' = -(d lambda'' + 4 s' d s' + 2 s'' d s) / (2 s),
d_g (d^2n/df^2) = knorm d s'' / f^2.  PEC-valued cells report 0.  The device computes the same map
(tidy3d_b200/csrc/derivatives.cuh, disp_grad_kernel).
"""
from __future__ import annotations

import numpy as np

from oracle import mode_derivatives as D
from oracle import mode_dispersion as MD
from oracle import mode_fourth_order as M4
from oracle import mode_group_gradient as MG
from oracle import restatement as R

C0_UM = 2.99792458e14  # um/s, the unit of the dispersion formula (tidy3d_b200.plugin.dispersion_of)


def dispersion_gradient(eps_cross, coords, freq, mode_spec, v, lam, symmetry=(0, 0), mu_cross=None, eps_dfreq=None, eps_d2freq=None,
                        x=None, x2=None, w_hat=None, w_hat2=None):
    """Permittivity gradients of the second frequency derivative of one mode (right eigenvector v = [Ex; Ey] of the solver-frame
    operator, eigenvalue lam = -n^2, which may be a Ritz value).  x / x2: the first / second scaled corrections, or None to
    solve them (bordered systems); w_hat / w_hat2: the left corrections (None: formed from x, x2).  Returns dict(
    d2lam_dfreq2_deps (d_g d^2 lambda / df^2, 1/Hz^2), d2n_dfreq_deps (1/Hz), d2n_dfreq2_deps (1/Hz^2), dispersion_deps
    (ps/(nm km) per unit eps), each (3, nx, ny), and x, x2, w, w_hat, w_hat2, lam1, lam2)."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    if st["tensorial"]:
        raise NotImplementedError("dispersion gradient: tensorial problems are out of scope")
    nx, ny = st["nx"], st["ny"]
    (P, Q, A), _ = MG.assemble_at(st)
    v = np.asarray(v, complex)
    w = D.left_vector(st, Q, v)
    wv = w @ v
    p1, p2 = MD.material_directions(st, eps_cross, freq, eps_dfreq, eps_d2freq)
    A1, A2 = MD.scaled_operators(st, freq, p1, p2)
    a1v = A1 @ v
    l1 = (w @ a1v) / wv
    if x is None:
        r = -(a1v - l1 * v)
        x, _ = MD.correction(A, lam, v, w, r - v * (w @ r) / wv)
    x = np.asarray(x, complex)
    Q1 = MG.q_prime(st, freq, p1)
    if w_hat is None:
        w_hat = MG.w_prime(st, Q, Q1, v, x)
    w_hat = np.asarray(w_hat, complex)
    a2v, a1x = A2 @ v, A1 @ x
    l2 = (w @ a2v + 2 * (w @ a1x - l1 * (w @ x))) / wv
    if x2 is None:
        r2 = -((a1x - l1 * x) + 0.5 * (a2v - l2 * v))
        x2, _ = MD.correction(A, lam, v, w, r2 - v * (w @ r2) / wv)
    x2 = np.asarray(x2, complex)
    if w_hat2 is None:
        w_hat2 = M4.w_second(st, Q, Q1, M4.q_second(st, freq, p2), v, x, x2)
    w_hat2 = np.asarray(w_hat2, complex)

    c1, c2 = MD.coef_directions(st, freq)

    def F(W, e, cdir=None, sc=0.0, pdir=None, sp_=0.0):  # D_a(W, e) at (c + sc cdir, p + sp_ pdir)
        (Pp, _, _), s = MG.assemble_at(st, cdir, sc, pdir, sp_)
        return MG.forms(s, Pp, e, W)

    def first(W, e):  # D_1(W, e)
        return 0.5 * (F(W, e, c1, 1.0) - F(W, e, c1, -1.0)) + 0.5 * (F(W, e, None, 0.0, p1, 1.0) - F(W, e, None, 0.0, p1, -1.0))

    d0 = F(w, v)
    cp, cm = F(w, v, c1, 1.0), F(w, v, c1, -1.0)
    d1wv = 0.5 * (cp - cm) + 0.5 * (F(w, v, None, 0.0, p1, 1.0) - F(w, v, None, 0.0, p1, -1.0))
    d2wv = 0.5 * (cp + cm) - d0
    d2wv = d2wv + 0.5 * (F(w, v, c2, 0.5) - F(w, v, c2, -0.5)) + 0.5 * (F(w, v, None, 0.0, p2, 0.5) - F(w, v, None, 0.0, p2, -0.5))
    d2wv = d2wv + 0.25 * (F(w, v, c1, 1.0, p1, 1.0) - F(w, v, c1, 1.0, p1, -1.0) - F(w, v, c1, -1.0, p1, 1.0) + F(w, v, c1, -1.0, p1, -1.0))
    b1 = F(w_hat, v) + F(w, x) + d1wv
    b2 = F(w_hat2, v) + F(w_hat, x) + F(w, x2) + first(w_hat, v) + first(w, x) + d2wv

    jac = st["jac_e"]
    det = jac[0, 0] * jac[1, 1] * jac[2, 2]
    iez = 1.0 / st["eps"][2, 2]
    kz = jac[2, 2] ** 2 / det
    chi = np.stack((jac[0, 0] ** 2 / det, jac[1, 1] ** 2 / det, -(iez**2) * kz)) * np.ones((3, nx * ny))
    chi1 = np.zeros((3, nx * ny), complex)
    chi2 = np.zeros((3, nx * ny), complex)
    chi1[2] = -2 * iez * p1[2] * kz
    chi2[2] = -(2 * iez * (0.5 * p2[2]) + p1[2] ** 2) * kz
    e0 = chi * d0
    e1 = chi * b1 + chi1 * d0
    e2 = chi * b2 + chi1 * b1 + chi2 * d0
    raw = np.stack([np.asarray(eps_cross[i], complex).ravel() for i in (0, 4, 8)])
    pec = raw.real <= 0.9 * R.PEC_VAL
    for e in (e0, e1, e2):
        e[pec] = 0.0
    D1 = w_hat @ v + w @ x
    D2 = w_hat2 @ v + w_hat @ x + w @ x2
    dlam = e0 / wv
    dlam1 = e1 / wv - e0 * D1 / wv**2
    dlam2 = e2 / wv - (e1 * D1 + e0 * D2) / wv**2 + e0 * D1**2 / wv**3  # d_g lambda_2, lambda_2 = lambda'' / 2
    s = np.sqrt(-lam + 0j)
    if s.real < 0:
        s = -s
    s1 = -l1 / (2 * s)
    s2 = -(l2 + 2 * s1 * s1) / (2 * s)
    ds = -dlam / (2 * s)
    ds1 = -(dlam1 + 2 * s1 * ds) / (2 * s)
    ds2 = -(2 * dlam2 + 4 * s1 * ds1 + 2 * s2 * ds) / (2 * s)
    knorm = st["knorm"]
    d2n1 = knorm * ds1 / freq
    d2n2 = knorm * ds2 / freq**2
    disp = -1e18 * freq**2 * (2 * d2n1.real + freq * d2n2.real) / C0_UM**2
    shape = (3, nx, ny)
    return dict(d2lam_dfreq2_deps=(2 * dlam2 / freq**2).reshape(shape), d2n_dfreq_deps=d2n1.reshape(shape),
                d2n_dfreq2_deps=d2n2.reshape(shape), dispersion_deps=disp.reshape(shape), x=x, x2=x2, w=w, w_hat=w_hat,
                w_hat2=w_hat2, lam1=l1, lam2=l2)
