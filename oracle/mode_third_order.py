"""TEST INFRASTRUCTURE ONLY -- float64 model of the third frequency derivative (third-order dispersion) of a mode.

Extends ``oracle/mode_dispersion.py`` (the correction x, lambda'') and ``oracle/mode_group_gradient.py`` (the left correction
w_hat).  Work in the scaled direction ' = f d/df, so X'' means f^2 d^2X/df^2 and X''' means f^3 d^3X/df^3.  By Wigner's 2n+1 rule
the functional L(v, w) = w^T A v / w^T v is stationary in both vectors, so the first-order corrections v + t x and w + t w_hat
give lambda(t) to O(t^4).  Expanding N/D, N = (w + t w_hat)^T A(t) (v + t x), D = (w + t w_hat)^T (v + t x), to t^3:

    lambda''' w^T v = w^T A''' v + 3 w_hat^T A'' v + 3 w^T A'' x + 6 w_hat^T A' x - 6 lambda' w_hat^T x - 3 lambda'' (w_hat^T v + w^T x).

x may carry any multiple of v and w_hat the same multiple of w: the result does not change.  A has bidegree (2, 2) in the 1-D
coefficients c and the solver-frame triple p = (exx, eyy, 1/ezz), so

    A''' = A_c[c'''] + A_p[p'''] + 3 A_cc[c', c''] + 3 A_pp[p', p''] + 3 A_cp[c', p''] + 3 A_cp[c'', p'] + 3 A_ccp[c', c', p']
           + 3 A_cpp[c', p', p']

is exact from unit-step operator evaluations E(c + a, p + b) (see ``third_operator``), with c''' = 6 c'^3 / c^2 (c = K / (a f + b):
f^n d^nc/df^n = n! c (c'/c)^n) and iez''' = -ezz''' iez^2 + 6 ezz' ezz'' iez^3 - 6 ezz'^3 iez^4.  With s = sqrt(-lambda):
s''' = -(lambda''' + 6 s' s'') / (2 s), n''' = knorm s'''.  The device computes the same quantities
(tidy3d_b200/csrc/derivatives.cuh, third_scan_kernel).
"""
from __future__ import annotations

import numpy as np

from oracle import mode_derivatives as D
from oracle import mode_dispersion as MD
from oracle import mode_group_gradient as MG
from oracle import restatement as R

C0_UM = MD.C0_UM  # um/s
C0_NM = 2.99792458e17  # nm/s
C0_M = 2.99792458e8  # m/s


def material_direction3(st, eps_cross, freq, eps_dfreq=None, eps_d2freq=None, eps_d3freq=None):
    """f^3 p''' of p = (exx, eyy, iez) of the solver frame, (3, N); 0 at PEC-valued cells."""
    nx, ny = st["nx"], st["ny"]
    d = [MD._diag3(a, nx, ny) * freq**k for k, a in ((1, eps_dfreq), (2, eps_d2freq), (3, eps_d3freq))]
    jac = st["jac_e"]
    det = jac[0, 0] * jac[1, 1] * jac[2, 2]
    for a in range(3):  # caller frame -> solver frame, as material_directions
        for dk in d:
            dk[a] = dk[a] * jac[a, a] ** 2 / det
    iez = 1.0 / st["eps"][2, 2]
    e1, e2, e3 = d[0][2], d[1][2], d[2][2]
    p3 = np.stack((d[2][0], d[2][1], -e3 * iez**2 + 6 * e1 * e2 * iez**3 - 6 * e1**3 * iez**4))
    raw = MD._diag3(eps_cross, nx, ny)
    p3[raw.real <= 0.9 * R.PEC_VAL] = 0.0
    return p3


def coef_direction3(st, freq):
    """c''' = f^3 d^3c/df^3 = 6 c'^3 / c^2 per axis."""
    d1 = D.coef_direction(st, freq)
    return [tuple(6 * np.divide(d**3, c * c, out=np.zeros_like(d), where=c != 0) for c, d in zip(cs, ds)) for cs, ds in zip(st["coef"], d1)]


def _cmix(a, sa, b, sb):
    """sa a + sb b of two coefficient directions (per axis, per row)."""
    return [tuple(sa * x + sb * y for x, y in zip(ta, tb)) for ta, tb in zip(a, b)]


def third_operator(st, freq, p1, p2, p3):
    """f^3 d^3A/df^3 including the material terms, exact: with E(a, b) = A(c + a, p + b),
    A_c[a] = [E(a) - E(-a)]/2, A_cc[a, b] = [E(a+b) - E(a-b) - E(-a+b) + E(-a-b)]/4 (A_pp alike),
    A_cp[a, b] = [E(a, b) - E(a, -b) - E(-a, b) + E(-a, -b)]/4 and
    3 A_ccp[a, a, b] + 3 A_cpp[a, b, b] = 3 [E(a, b) - E(-a, -b) - E(0, b) + E(0, -b) - E(a, 0) + E(-a, 0)]."""
    c1, c2 = MD.coef_directions(st, freq)
    c3 = coef_direction3(st, freq)

    def E(cd=None, sc=0.0, pd=None, sp_=0.0):
        return MD.assemble_at(st, cd, sc, pd, sp_)

    cs, cd = _cmix(c1, 1.0, c2, 1.0), _cmix(c1, 1.0, c2, -1.0)  # c' + c'', c' - c''
    A3 = 0.5 * (E(c3, 1.0) - E(c3, -1.0))
    A3 = A3 + 0.75 * (E(cs, 1.0) - E(cd, 1.0) - E(cd, -1.0) + E(cs, -1.0))
    if p1 is not None and (np.any(p1) or np.any(p2) or np.any(p3)):
        ps, pd = p1 + p2, p1 - p2
        A3 = A3 + 0.5 * (E(None, 0.0, p3, 1.0) - E(None, 0.0, p3, -1.0))
        A3 = A3 + 0.75 * (E(None, 0.0, ps, 1.0) - E(None, 0.0, pd, 1.0) - E(None, 0.0, pd, -1.0) + E(None, 0.0, ps, -1.0))
        for ca, pb in ((c1, p2), (c2, p1)):
            A3 = A3 + 0.75 * (E(ca, 1.0, pb, 1.0) - E(ca, 1.0, pb, -1.0) - E(ca, -1.0, pb, 1.0) + E(ca, -1.0, pb, -1.0))
        A3 = A3 + 3.0 * (E(c1, 1.0, p1, 1.0) - E(c1, -1.0, p1, -1.0) - E(None, 0.0, p1, 1.0) + E(None, 0.0, p1, -1.0)
                         - E(c1, 1.0) + E(c1, -1.0))
    return A3.tocsr()


def d3A_dfreq3(st, freq, eps_cross, eps_dfreq=None, eps_d2freq=None, eps_d3freq=None):
    """d^3A/df^3 including the material dispersion (1/Hz^3)."""
    p1, p2 = MD.material_directions(st, eps_cross, freq, eps_dfreq, eps_d2freq)
    p3 = material_direction3(st, eps_cross, freq, eps_dfreq, eps_d2freq, eps_d3freq)
    return third_operator(st, freq, p1, p2, p3) / freq**3


def dispersion_slope(freq, dn_dfreq, d2n_dfreq2, d3n_dfreq3):
    """S = dD/d(wavelength) in ps/(nm^2 km): dD/df = -1e18 (4 f Re n' + 5 f^2 Re n'' + f^3 Re n''') / c0^2, S = -(f^2 / c_nm) dD/df."""
    dd = -1e18 * (4 * freq * np.real(dn_dfreq) + 5 * freq**2 * np.real(d2n_dfreq2) + freq**3 * np.real(d3n_dfreq3)) / C0_UM**2
    return -(freq**2 / C0_NM) * dd


def beta3(freq, d2n_dfreq2, d3n_dfreq3):
    """beta3 = d^3 beta / d omega^3 = (3 Re n'' + f Re n''') / (4 pi^2 c) in ps^3/km (1 s^3/m = 1e39 ps^3/km)."""
    return (3 * np.real(d2n_dfreq2) + freq * np.real(d3n_dfreq3)) / (4 * np.pi**2 * C0_M) * 1e39


def third_derivatives(eps_cross, coords, freq, mode_spec, v, lam, symmetry=(0, 0), mu_cross=None, eps_dfreq=None, eps_d2freq=None,
                      eps_d3freq=None, x=None, w_hat=None):
    """Third frequency derivative of one mode (right eigenvector v = [Ex; Ey] of the solver-frame operator, eigenvalue
    lam = -n^2, which may be a Ritz value).  x: the scaled correction (v' up to a multiple of v) or None to solve it as the
    dispersion model does; w_hat: the left correction (None: formed from x).  Returns dict(lam1, lam2, lam3 (scaled),
    d3lam_dfreq3, dn_dfreq, d2n_dfreq2, d3n_dfreq3 (1/Hz^3), dispersion_slope (ps/(nm^2 km)), beta3 (ps^3/km), A1, A2, A3
    (scaled operators), x, w, w_hat)."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    if st["tensorial"]:
        raise NotImplementedError("third derivatives: tensorial problems are out of scope")
    (_, Q, A), _ = MG.assemble_at(st)
    v = np.asarray(v, complex)
    w = D.left_vector(st, Q, v)
    wv = w @ v
    p1, p2 = MD.material_directions(st, eps_cross, freq, eps_dfreq, eps_d2freq)
    p3 = material_direction3(st, eps_cross, freq, eps_dfreq, eps_d2freq, eps_d3freq)
    A1, A2 = MD.scaled_operators(st, freq, p1, p2)
    A3 = third_operator(st, freq, p1, p2, p3)
    a1v = A1 @ v
    l1 = (w @ a1v) / wv
    if x is None:
        r = -(a1v - l1 * v)
        x, _ = MD.correction(A, lam, v, w, r - v * (w @ r) / wv)
    x = np.asarray(x, complex)
    if w_hat is None:
        w_hat = MG.w_prime(st, Q, MG.q_prime(st, freq, p1), v, x)
    w_hat = np.asarray(w_hat, complex)
    a2v, a2x, a1x = A2 @ v, A2 @ x, A1 @ x
    l2 = (w @ a2v + 2 * (w @ a1x - l1 * (w @ x))) / wv
    l3 = (w @ (A3 @ v) + 3 * (w_hat @ a2v) + 3 * (w @ a2x) + 6 * (w_hat @ a1x) - 6 * l1 * (w_hat @ x)
          - 3 * l2 * (w_hat @ v + w @ x)) / wv
    dl, d2l, d3l = l1 / freq, l2 / freq**2, l3 / freq**3
    s = np.sqrt(-lam + 0j)
    if s.real < 0:
        s = -s
    ds = -dl / (2 * s)
    d2s = -(d2l + 2 * ds * ds) / (2 * s)
    d3s = -(d3l + 6 * ds * d2s) / (2 * s)
    knorm = st["knorm"]
    dn, d2n, d3n = knorm * ds, knorm * d2s, knorm * d3s
    return dict(lam1=l1, lam2=l2, lam3=l3, d3lam_dfreq3=d3l, dn_dfreq=dn, d2n_dfreq2=d2n, d3n_dfreq3=d3n,
                dispersion_slope=dispersion_slope(freq, dn, d2n, d3n), beta3=beta3(freq, d2n, d3n),
                A1=A1, A2=A2, A3=A3, x=x, w=w, w_hat=w_hat)
