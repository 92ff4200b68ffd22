"""TEST INFRASTRUCTURE ONLY -- float64 model of the second frequency derivative (group-velocity dispersion) of a mode.

Extends ``oracle/mode_derivatives.py`` (left eigenvector w = G J Q v, first-order theory).  Work in the scaled direction
' = f d/df.  A is a polynomial of degree <= 2 in the 1-D difference coefficients c and of degree <= 2 in the per-cell triple
p = (eps_xx, eps_yy, 1/eps_zz) of the solver frame (after the bend congruence, which does not depend on f), so with
c' = -c kappa / s, c'' = 2 c'^2 / c (c = 1 / (s k0 dl) is 1 / (a f + b)), p' and p'' from the material dispersion:

    A'v  = [A(c+c',p) - A(c-c',p)]/2 + [A(c,p+p') - A(c,p-p')]/2
    A''v = [A(c+c',p) + A(c-c',p) - 2A] + [A(c+c'',p) - A(c-c'',p)]/2 + [A(c,p+p') + A(c,p-p') - 2A] + [A(c,p+p'') - A(c,p-p'')]/2
           + [A(c+c',p+p') - A(c+c',p-p') - A(c-c',p+p') + A(c-c',p-p')]/2

are exact with unit steps (a joint difference along (c, p) would not be: c^2 eps / eps_zz has degree 4).  Then

    lambda' = w^T A' v / w^T v,   (A - lambda) x = r = -Pi (A' - lambda') v,  Pi = I - v w^T / (w^T v),  w^T x = 0,
    lambda'' = [w^T A'' v + 2 w^T (A' - lambda') x] / w^T v,

solved here as the bordered system [[A - lambda, v], [w^T, 0]] [x; mu] = [r; 0] (nonsingular for a simple eigenvalue, and
well posed for a lambda that is only a Ritz value of this A, such as the device's).  With s = sqrt(-lambda):
s' = -lambda'/(2 s), s'' = -(lambda'' + 2 s'^2)/(2 s), n'' = knorm s''.  The device computes the same quantities
(tidy3d_b200/csrc/derivatives.cuh, dispersion pass).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from oracle import mode_derivatives as D
from oracle import restatement as R

C0_UM = 2.99792458e14  # um/s


def _diag3(a, nx, ny):
    """The diagonal (xx, yy, zz) of a nine-component eps-layout input, shape (3, N)."""
    if a is None:
        return np.zeros((3, nx * ny), complex)
    return np.stack([np.asarray(a[i], complex).ravel() for i in (0, 4, 8)])


def material_directions(st, eps_cross, freq, eps_dfreq=None, eps_d2freq=None):
    """Scaled directions (f p', f^2 p'') of p = (exx, eyy, iez) of the solver frame, each (3, N); 0 at PEC-valued cells."""
    nx, ny = st["nx"], st["ny"]
    d1, d2 = _diag3(eps_dfreq, nx, ny) * freq, _diag3(eps_d2freq, nx, ny) * freq**2
    jac = st["jac_e"]
    det = jac[0, 0] * jac[1, 1] * jac[2, 2]
    for a in range(3):  # caller frame -> solver frame: eps'_aa = J_aa^2 eps_aa / det J
        d1[a] = d1[a] * jac[a, a] ** 2 / det
        d2[a] = d2[a] * jac[a, a] ** 2 / det
    iez = 1.0 / st["eps"][2, 2]
    p1 = np.stack((d1[0], d1[1], -d1[2] * iez**2))
    p2 = np.stack((d2[0], d2[1], 2 * d1[2] ** 2 * iez**3 - d2[2] * iez**2))
    raw = _diag3(eps_cross, nx, ny)
    pec = raw.real <= 0.9 * R.PEC_VAL
    p1[pec] = 0.0
    p2[pec] = 0.0
    return p1, p2


def coef_directions(st, freq):
    """(c', c'') per axis: f dc/df = -c kappa / s and f^2 d^2c/df^2 = 2 c'^2 / c."""
    d1 = D.coef_direction(st, freq)
    d2 = []
    for cs, ds in zip(st["coef"], d1):
        d2.append(tuple(2 * np.divide(d * d, c, out=np.zeros_like(d), where=c != 0) for c, d in zip(cs, ds)))
    return d1, d2


def assemble_at(st, cdir=None, sc=0.0, pdir=None, sp_=0.0):
    """A at c + sc cdir and p + sp_ pdir (sparse)."""
    s = dict(st)
    if cdir is not None:
        s["coef"] = [tuple(c + sc * d for c, d in zip(cs, ds)) for cs, ds in zip(st["coef"], cdir)]
    if pdir is not None:
        e = np.array(st["eps"], complex, copy=True)
        e[0, 0] = e[0, 0] + sp_ * pdir[0]
        e[1, 1] = e[1, 1] + sp_ * pdir[1]
        e[2, 2] = 1.0 / (1.0 / st["eps"][2, 2] + sp_ * pdir[2])
        s["eps"] = e
    return R.assemble_diagonal(s)[2]


def scaled_operators(st, freq, p1, p2):
    """(f dA/df, f^2 d^2A/df^2) including the material terms, exact (see the module docstring)."""
    c1, c2 = coef_directions(st, freq)
    A0 = assemble_at(st)
    Acp, Acm = assemble_at(st, c1, 1.0), assemble_at(st, c1, -1.0)
    App, Apm = assemble_at(st, None, 0.0, p1, 1.0), assemble_at(st, None, 0.0, p1, -1.0)
    A1 = 0.5 * (Acp - Acm) + 0.5 * (App - Apm)
    A2 = (Acp + Acm - 2 * A0) + 0.5 * (assemble_at(st, c2, 1.0) - assemble_at(st, c2, -1.0))
    A2 = A2 + (App + Apm - 2 * A0) + 0.5 * (assemble_at(st, None, 0.0, p2, 1.0) - assemble_at(st, None, 0.0, p2, -1.0))
    mixed = assemble_at(st, c1, 1.0, p1, 1.0) - assemble_at(st, c1, 1.0, p1, -1.0) - assemble_at(st, c1, -1.0, p1, 1.0)
    A2 = A2 + 0.5 * (mixed + assemble_at(st, c1, -1.0, p1, -1.0))
    return A1.tocsr(), A2.tocsr()


def dA_dfreq_total(st, freq, eps_cross, eps_dfreq=None):
    """dA/df including the material dispersion (1/Hz)."""
    p1, p2 = material_directions(st, eps_cross, freq, eps_dfreq, None)
    return scaled_operators(st, freq, p1, p2)[0] / freq


def d2A_dfreq2(st, freq, eps_cross, eps_dfreq=None, eps_d2freq=None):
    """d^2A/df^2 including the material dispersion (1/Hz^2)."""
    p1, p2 = material_directions(st, eps_cross, freq, eps_dfreq, eps_d2freq)
    return scaled_operators(st, freq, p1, p2)[1] / freq**2


def correction(A, lam, v, w, r):
    """x with (A - lam) x + mu v = r and w^T x = 0: the bordered system, sparse LU."""
    n = A.shape[0]
    K = sp.bmat([[A - lam * sp.eye(n, format="csr"), sp.csr_matrix(v.reshape(-1, 1))], [sp.csr_matrix(w.reshape(1, -1)), None]], format="csc")
    sol = spl.splu(K).solve(np.r_[r, 0.0].astype(complex))
    return sol[:n], sol[n]


def dispersion(freq, dn_dfreq, d2n_dfreq2):
    """D = -1e18 f^2 (2 Re n' + f Re n'') / c0^2 in ps/(nm km)."""
    return -1e18 * freq**2 * (2 * np.real(dn_dfreq) + freq * np.real(d2n_dfreq2)) / C0_UM**2


def second_derivatives(eps_cross, coords, freq, mode_spec, v, lam, symmetry=(0, 0), mu_cross=None, eps_dfreq=None, eps_d2freq=None):
    """Second frequency derivative of one mode (right eigenvector v = [Ex; Ey] of the solver-frame operator, eigenvalue
    lam = -n^2, which may be a Ritz value).  Returns dict(dlam_dfreq, d2lam_dfreq2, dn_dfreq, d2n_dfreq2 (1/Hz^2), dispersion
    (ps/(nm km)), x and r (the scaled correction and its right-hand side), A (the operator), w, mu)."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    if st["tensorial"]:
        raise NotImplementedError("second derivatives: tensorial problems are out of scope")
    _, Q, A = R.assemble_diagonal(st)
    v = np.asarray(v, complex)
    w = D.left_vector(st, Q, v)
    wv = w @ v
    p1, p2 = material_directions(st, eps_cross, freq, eps_dfreq, eps_d2freq)
    A1, A2 = scaled_operators(st, freq, p1, p2)
    a1v = A1 @ v
    l1 = (w @ a1v) / wv
    r = -(a1v - l1 * v)
    r = r - v * (w @ r) / wv
    x, mu = correction(A, lam, v, w, r)
    l2 = (w @ (A2 @ v) + 2 * (w @ (A1 @ x) - l1 * (w @ x))) / wv
    dl, d2l = l1 / freq, l2 / freq**2
    s = np.sqrt(-lam + 0j)
    if s.real < 0:
        s = -s
    ds = -dl / (2 * s)
    d2s = -(d2l + 2 * ds * ds) / (2 * s)
    knorm = st["knorm"]
    dn, d2n = knorm * ds, knorm * d2s
    return dict(dlam_dfreq=dl, d2lam_dfreq2=d2l, dn_dfreq=dn, d2n_dfreq2=d2n, dispersion=dispersion(freq, dn, d2n),
                x=x, r=r, A=A, w=w, mu=mu)
