"""TEST INFRASTRUCTURE ONLY -- float64 model of the fourth frequency derivative (fourth-order dispersion) of a mode.

Extends ``oracle/mode_third_order.py`` (x, w_hat, lambda''').  Work in the scaled direction ' = f d/df (X'''' = f^4 d^4X/df^4)
and Taylor-expand in t = (f_new - f) / f.  The right eigenvector v(t) = v + t x + t^2 x2 + O(t^3) needs one more correction:

    (A - lambda) x2 = r2 = -Pi [(A' - lambda') x + 1/2 (A'' - lambda'') v],   Pi = I - v w^T / (w^T v),

(the order-t^2 part of (A(t) - lambda(t)) v(t) = 0; Pi removes nothing from a consistent right-hand side, since
w^T r2 = 0 is the formula for lambda'').  The left eigenvector w(t) = G(t) J Q(t) v(t) is structural for every t, so its
second-order coefficient is local work on v, x and x2 with the Taylor coefficients G_i, Q_j in t:

    w_hat2 = G_2 J Q v + G_1 J (Q_1 v + Q x) + G J (Q_2 v + Q_1 x + Q x2),

where every stretched length l = s dl moves as l(t) = Re l + i Im l / (1 + t) (l_1 = -i Im l, l_2 = i Im l), and Q (quadratic in
the 1-D coefficients c, affine in (exx, eyy)) has Q_2 = B(c_1, c_1) + Q_c[c_2] + Q_p[p_2] with c_2 = c''/2, p_2 = p''/2.
The functional w^T A v / w^T v is stationary in both vectors, so V = v + t x + t^2 x2 and W = w + t w_hat + t^2 w_hat2 give
lambda(t) = N(t) / D(t) + O(t^6), N = W^T A(t) V, D = W^T V, and lambda'''' = 4! [t^4] N / D:

    lambda'''' w^T v = w^T A''''v + 4 w_hat^T A'''v + 4 w^T A'''x + 12 w_hat2^T A''v + 12 w^T A''x2 + 12 w_hat^T A''x
                       + 24 w_hat2^T A'x + 24 w_hat^T A'x2 + 24 w_hat2^T (A - lambda) x2
                       - 24 lambda' D_3 - 12 lambda'' D_2 - 4 lambda''' D_1,
    D_1 = w_hat^T v + w^T x,   D_2 = w_hat2^T v + w_hat^T x + w^T x2,   D_3 = w_hat2^T x + w_hat^T x2.

x may carry any multiple a v (then x2 carries a x, and the w side the matching multiples) and x2 any multiple of v: the
result does not change.  A has bidegree (2, 2) in (c, p), so A'''' is exact from unit-step operator evaluations (see
``fourth_operator``), with c'''' = 24 c'^4 / c^3 and iez'''' = -ezz'''' iez^2 + (8 ezz' ezz''' + 6 ezz''^2) iez^3
- 36 ezz'^2 ezz'' iez^4 + 24 ezz'^4 iez^5.  With s = sqrt(-lambda): s'''' = -(lambda'''' + 8 s' s''' + 6 s''^2) / (2 s),
n'''' = knorm s''''.  The device computes the same quantities (tidy3d_b200/csrc/derivatives.cuh, fourth_rhs_kernel,
fourth_scan_kernel).
"""
from __future__ import annotations

import numpy as np

from oracle import mode_derivatives as D
from oracle import mode_dispersion as MD
from oracle import mode_group_gradient as MG
from oracle import mode_third_order as M3
from oracle import restatement as R

C0_M = M3.C0_M


def material_direction4(st, eps_cross, freq, eps_dfreq=None, eps_d2freq=None, eps_d3freq=None, eps_d4freq=None):
    """f^4 p'''' of p = (exx, eyy, iez) of the solver frame, (3, N); 0 at PEC-valued cells."""
    nx, ny = st["nx"], st["ny"]
    d = [MD._diag3(a, nx, ny) * freq**k for k, a in ((1, eps_dfreq), (2, eps_d2freq), (3, eps_d3freq), (4, eps_d4freq))]
    jac = st["jac_e"]
    det = jac[0, 0] * jac[1, 1] * jac[2, 2]
    for a in range(3):  # caller frame -> solver frame, as material_directions
        for dk in d:
            dk[a] = dk[a] * jac[a, a] ** 2 / det
    iez = 1.0 / st["eps"][2, 2]
    e1, e2, e3, e4 = d[0][2], d[1][2], d[2][2], d[3][2]
    iz4 = -e4 * iez**2 + (8 * e1 * e3 + 6 * e2 * e2) * iez**3 - 36 * e1 * e1 * e2 * iez**4 + 24 * e1**4 * iez**5
    p4 = np.stack((d[3][0], d[3][1], iz4))
    raw = MD._diag3(eps_cross, nx, ny)
    p4[raw.real <= 0.9 * R.PEC_VAL] = 0.0
    return p4


def coef_direction4(st, freq):
    """c'''' = f^4 d^4c/df^4 = 24 c'^4 / c^3 per axis."""
    d1 = D.coef_direction(st, freq)
    return [tuple(24 * np.divide(d**4, c**3, out=np.zeros_like(d), where=c != 0) for c, d in zip(cs, ds)) for cs, ds in zip(st["coef"], d1)]


def fourth_operator(st, freq, p1, p2, p3, p4):
    """f^4 d^4A/df^4 including the material terms, exact.  With c_k, p_k the Taylor coefficients in t (c_k = c^(k) / k!),
    [t^4] A(c(t), p(t)) = A_c[c_4] + A_cc[c_1, c_3] + A_cc[c_2, c_2]/2 + (the same in p) + A_cp[c_1, p_3] + A_cp[c_2, p_2]
    + A_cp[c_3, p_1] + A_ccp[c_1, c_1, p_2]/2 + A_ccp[c_1, c_2, p_1] + A_cpp[c_2, p_1, p_1]/2 + A_cpp[c_1, p_1, p_2]
    + A_ccpp[c_1, c_1, p_1, p_1]/4.  With E(a, b) = A(c + a, p + b) and the odd / even parts of the bidegree-(2, 2) polynomial:
    A_c[a] = [E(a) - E(-a)]/2, A_cc[a, b] = [E(a+b) - E(a-b) - E(-a+b) + E(-a-b)]/4, A_cc[a, a] = E(a) + E(-a) - 2 E(0),
    A_cp[a, b] = [E(a, b) - E(a, -b) - E(-a, b) + E(-a, -b)]/4,
    A_ccp[a, a, b]/2 = [E(a, b) - E(a, -b) + E(-a, b) - E(-a, -b)]/4 - A_p[b] (A_ccp[a, a', b] by polarisation over a +- a'),
    A_cpp alike, and A_ccpp[a, a, b, b]/4 = sum E(+-a, +-b)/4 - [E(a, 0) + E(-a, 0) + E(0, b) + E(0, -b)]/2 + E(0)."""
    c1, c2 = MD.coef_directions(st, freq)
    c3 = M3.coef_direction3(st, freq)
    c4 = coef_direction4(st, freq)
    mix = M3._cmix

    def E(cd=None, sc=0.0, pd=None, sp_=0.0):
        return MD.assemble_at(st, cd, sc, pd, sp_)

    E0 = E()
    s13, d13 = mix(c1, 1.0, c3, 1.0), mix(c1, 1.0, c3, -1.0)
    A4 = 0.5 * (E(c4, 1.0) - E(c4, -1.0))
    A4 = A4 + (E(s13, 1.0) - E(d13, 1.0) - E(d13, -1.0) + E(s13, -1.0))  # 4 A_cc[c', c''']
    A4 = A4 + 3.0 * (E(c2, 1.0) + E(c2, -1.0) - 2 * E0)  # 3 A_cc[c'', c'']
    if p1 is None or not (np.any(p1) or np.any(p2) or np.any(p3) or np.any(p4)):
        return A4.tocsr()

    def Ep(pd, sp_, cd=None, sc=0.0):
        return E(cd, sc, pd, sp_)

    A4 = A4 + 0.5 * (Ep(p4, 1.0) - Ep(p4, -1.0))
    s13p, d13p = p1 + p3, p1 - p3
    A4 = A4 + (Ep(s13p, 1.0) - Ep(d13p, 1.0) - Ep(d13p, -1.0) + Ep(s13p, -1.0))  # 4 A_pp[p', p''']
    A4 = A4 + 3.0 * (Ep(p2, 1.0) + Ep(p2, -1.0) - 2 * E0)  # 3 A_pp[p'', p'']

    def cp(a, b):  # 4 A_cp[a, b]
        return E(a, 1.0, b, 1.0) - E(a, 1.0, b, -1.0) - E(a, -1.0, b, 1.0) + E(a, -1.0, b, -1.0)

    A4 = A4 + cp(c1, p3) + 1.5 * cp(c2, p2) + cp(c3, p1)  # 4 A_cp[c', p'''] + 6 A_cp[c'', p''] + 4 A_cp[c''', p']

    def ccp(a, b):  # 4 (A_ccp[a, a, b]/2 + A_p[b])
        return E(a, 1.0, b, 1.0) - E(a, 1.0, b, -1.0) + E(a, -1.0, b, 1.0) - E(a, -1.0, b, -1.0)

    def cpp(a, b):  # 4 (A_cpp[a, b, b]/2 + A_c[a])
        return E(a, 1.0, b, 1.0) + E(a, 1.0, b, -1.0) - E(a, -1.0, b, 1.0) - E(a, -1.0, b, -1.0)

    # 6 A_ccp[c', c', p''] = 12 (A_ccp/2) and 12 A_ccp[c', c'', p'] = 1.5 (ccp(c' + c'') - ccp(c' - c''))
    A4 = A4 + 3.0 * ccp(c1, p2) - 6.0 * (Ep(p2, 1.0) - Ep(p2, -1.0))
    A4 = A4 + 1.5 * (ccp(mix(c1, 1.0, c2, 1.0), p1) - ccp(mix(c1, 1.0, c2, -1.0), p1))
    # 6 A_cpp[c'', p', p'] and 12 A_cpp[c', p', p''] alike
    A4 = A4 + 3.0 * cpp(c2, p1) - 6.0 * (E(c2, 1.0) - E(c2, -1.0))
    A4 = A4 + 1.5 * (cpp(c1, p1 + p2) - cpp(c1, p1 - p2))
    # 6 A_ccpp[c', c', p', p'] = 24 (A_ccpp/4)
    quad = E(c1, 1.0, p1, 1.0) + E(c1, 1.0, p1, -1.0) + E(c1, -1.0, p1, 1.0) + E(c1, -1.0, p1, -1.0)
    A4 = A4 + 6.0 * quad - 12.0 * (E(c1, 1.0) + E(c1, -1.0) + Ep(p1, 1.0) + Ep(p1, -1.0)) + 24.0 * E0
    return A4.tocsr()


def d4A_dfreq4(st, freq, eps_cross, eps_dfreq=None, eps_d2freq=None, eps_d3freq=None, eps_d4freq=None):
    """d^4A/df^4 including the material dispersion (1/Hz^4)."""
    p1, p2 = MD.material_directions(st, eps_cross, freq, eps_dfreq, eps_d2freq)
    p3 = M3.material_direction3(st, eps_cross, freq, eps_dfreq, eps_d2freq, eps_d3freq)
    p4 = material_direction4(st, eps_cross, freq, eps_dfreq, eps_d2freq, eps_d3freq, eps_d4freq)
    return fourth_operator(st, freq, p1, p2, p3, p4) / freq**4


def metric_second(st):
    """G_2, the t^2 coefficient of G(t) in w = G J Q v: l(t) = Re l + i Im l / (1 + t) has l_1 = -i Im l, l_2 = i Im l."""
    (sfx, sbx), (sfy, sby) = [(np.array(a, complex), np.array(b, complex)) for a, b in st["slen"]]
    if st["pmc"][0]:
        sbx[0] *= 0.5
    if st["pmc"][1]:
        sby[0] *= 0.5
    d1 = lambda l: -1j * l.imag  # noqa: E731
    d2 = lambda l: 1j * l.imag  # noqa: E731

    def g2(a, b):
        return (d2(a)[:, None] * b[None, :] + d1(a)[:, None] * d1(b)[None, :] + a[:, None] * d2(b)[None, :]).ravel()

    return np.r_[g2(sfx, sby), g2(sbx, sfy)]


def q_second(st, freq, p2):
    """Q_2, the t^2 coefficient of Q(t): B(c', c') + Q_c[c''/2] + Q_p[p''/2], all exact with unit steps."""
    c1, c2 = MD.coef_directions(st, freq)
    Q0 = MG.assemble_at(st)[0][1]
    Q2 = 0.5 * (MG.assemble_at(st, c1, 1.0)[0][1] + MG.assemble_at(st, c1, -1.0)[0][1]) - Q0
    Q2 = Q2 + 0.5 * (MG.assemble_at(st, c2, 0.5)[0][1] - MG.assemble_at(st, c2, -0.5)[0][1])
    return Q2 + 0.5 * (MG.assemble_at(st, None, 0.0, p2, 0.5)[0][1] - MG.assemble_at(st, None, 0.0, p2, -0.5)[0][1])


def w_second(st, Q, Q1, Q2, v, x, x2):
    """w_hat2 = G_2 J Q v + G_1 J (Q_1 v + Q x) + G J (Q_2 v + Q_1 x + Q x2)."""
    n = st["n"]
    J = lambda h: np.r_[h[n:], -h[:n]]  # noqa: E731
    return (metric_second(st) * J(Q @ v) + MG.metric_prime(st) * J(Q1 @ v + Q @ x)
            + D.metric(st) * J(Q2 @ v + Q1 @ x + Q @ x2))


def beta4(freq, d3n_dfreq3, d4n_dfreq4):
    """beta4 = d^4 beta / d omega^4 = (4 Re n''' + f Re n'''') / (8 pi^3 c) in ps^4/km (1 s^4/m = 1e51 ps^4/km)."""
    return (4 * np.real(d3n_dfreq3) + freq * np.real(d4n_dfreq4)) / (8 * np.pi**3 * C0_M) * 1e51


def fourth_derivatives(eps_cross, coords, freq, mode_spec, v, lam, symmetry=(0, 0), mu_cross=None, eps_dfreq=None, eps_d2freq=None,
                       eps_d3freq=None, eps_d4freq=None, x=None, x2=None, w_hat=None, w_hat2=None):
    """Fourth frequency derivative of one mode (right eigenvector v = [Ex; Ey] of the solver-frame operator, eigenvalue
    lam = -n^2, which may be a Ritz value).  x / x2: the first / second scaled corrections, or None to solve them (bordered
    systems, w^T x = w^T x2 = 0); w_hat / w_hat2: the left corrections (None: formed from x, x2).  Returns dict(lam1 .. lam4
    (scaled), d4lam_dfreq4, dn_dfreq, d2n_dfreq2, d3n_dfreq3, d4n_dfreq4 (1/Hz^4), beta4 (ps^4/km), A1 .. A4 (scaled operators),
    A, x, x2, r2, w, w_hat, w_hat2)."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    if st["tensorial"]:
        raise NotImplementedError("fourth derivatives: tensorial problems are out of scope")
    (_, Q, A), _ = MG.assemble_at(st)
    v = np.asarray(v, complex)
    w = D.left_vector(st, Q, v)
    wv = w @ v
    p1, p2 = MD.material_directions(st, eps_cross, freq, eps_dfreq, eps_d2freq)
    p3 = M3.material_direction3(st, eps_cross, freq, eps_dfreq, eps_d2freq, eps_d3freq)
    p4 = material_direction4(st, eps_cross, freq, eps_dfreq, eps_d2freq, eps_d3freq, eps_d4freq)
    A1, A2 = MD.scaled_operators(st, freq, p1, p2)
    A3 = M3.third_operator(st, freq, p1, p2, p3)
    A4 = fourth_operator(st, freq, p1, p2, p3, p4)
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
    l3 = (w @ (A3 @ v) + 3 * (w_hat @ a2v) + 3 * (w @ (A2 @ x)) + 6 * (w_hat @ a1x) - 6 * l1 * (w_hat @ x)
          - 3 * l2 * (w_hat @ v + w @ x)) / wv
    r2 = -((a1x - l1 * x) + 0.5 * (a2v - l2 * v))
    r2 = r2 - v * (w @ r2) / wv
    if x2 is None:
        x2, _ = MD.correction(A, lam, v, w, r2)
    x2 = np.asarray(x2, complex)
    if w_hat2 is None:
        w_hat2 = w_second(st, Q, Q1, q_second(st, freq, p2), v, x, x2)
    w_hat2 = np.asarray(w_hat2, complex)
    d1 = w_hat @ v + w @ x
    d2 = w_hat2 @ v + w_hat @ x + w @ x2
    d3 = w_hat2 @ x + w_hat @ x2
    num = (w @ (A4 @ v) + 4 * (w_hat @ (A3 @ v)) + 4 * (w @ (A3 @ x)) + 12 * (w_hat2 @ a2v) + 12 * (w @ (A2 @ x2))
           + 12 * (w_hat @ (A2 @ x)) + 24 * (w_hat2 @ a1x) + 24 * (w_hat @ (A1 @ x2)) + 24 * (w_hat2 @ (A @ x2 - lam * x2)))
    l4 = (num - 24 * l1 * d3 - 12 * l2 * d2 - 4 * l3 * d1) / wv
    dl, d2l, d3l, d4l = l1 / freq, l2 / freq**2, l3 / freq**3, l4 / freq**4
    s = np.sqrt(-lam + 0j)
    if s.real < 0:
        s = -s
    ds = -dl / (2 * s)
    d2s = -(d2l + 2 * ds * ds) / (2 * s)
    d3s = -(d3l + 6 * ds * d2s) / (2 * s)
    d4s = -(d4l + 8 * ds * d3s + 6 * d2s * d2s) / (2 * s)
    knorm = st["knorm"]
    dn, d2n, d3n, d4n = knorm * ds, knorm * d2s, knorm * d3s, knorm * d4s
    return dict(lam1=l1, lam2=l2, lam3=l3, lam4=l4, d4lam_dfreq4=d4l, dn_dfreq=dn, d2n_dfreq2=d2n, d3n_dfreq3=d3n, d4n_dfreq4=d4n,
                beta4=beta4(freq, d3n, d4n), A1=A1, A2=A2, A3=A3, A4=A4, A=A, x=x, x2=x2, r2=r2, w=w, w_hat=w_hat, w_hat2=w_hat2)
