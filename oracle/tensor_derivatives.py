"""TEST INFRASTRUCTURE ONLY -- float64 model of the adjoint (left-eigenvector) side of the tensorial first-order operator.

The tensorial operator is the 4N first-order M of ``restatement.assemble_tensorial`` (eigenvalue n, the solver works with
mat = msign (-i) M).  Unlike the diagonal A = P Q of ``mode_derivatives``, M has no structural left eigenvector: reciprocity
(-n in the spectrum, the backward mode as left eigenvector) fails once PML, a non-uniform grid or a PMC wall meets a z-coupled
permittivity.  What does hold is a local pairing of its diagonal-tensor part mat_d = [[0, P], [Q, 0]]:

    K mat_d = -mat_d^T K,   K [Ex; Ey; Hx; Hy] = [gx Hy; -gy Hx; gy Ey; -gx Ex],

with gx = sf_x dlf_x * sb_y dlb_y (Ex sites) and gy = sb_x dlb_x * sf_y dlf_y (Ey sites) the complex-stretched primal / dual cell
lengths of ``mode_derivatives.metric`` (first dual length halved at a PMC wall; the bend enters through eps', not K).  So

    (mat_d^T - sigma)^-1 = -K (mat_d + sigma)^-1 K^-1,

and the preconditioner of the forward solve, with its shift negated, preconditions a solve with mat^T.  The device's transposed
operator and preconditioner (tensor_apply_kernel<C, true>, BatchSolver::precondition_tensor_T) are pinned against this model.

Left eigenvectors come from an eigen-solve of M^T at the forward shift, independently of K, and first-order perturbation theory
gives dn = w^T (d mat) u / (w^T u).  M has degree <= 2 in the 1-D difference coefficients c (the Dxf iez Dyb blocks) and no
frequency dependence elsewhere at fixed permittivity, so f dM/df = [M(c + c') - M(c - c')] / 2 exactly with the f dc/df = -c
kappa / s directions of ``mode_derivatives.coef_direction``.  M is affine in the per-site derived fields q of eps' (the
order of the device's coefficient fields), so the permittivity gradient is a per-site sum of products (A^T w)(B u) over the
blocks A diag(q) B, chained through dq/deps', the congruence eps' = J eps J^T / det J and the PEC model; a nine-component
eps_dfreq adds the material dispersion to dn/df.  On uniform grids without z-coupled PML, w is parallel to K u(-n).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from oracle import mode_derivatives as D
from oracle import restatement as R


def diagonal_part(st):
    """mat_d = [[0, P], [Q, 0]]: the diagonal-tensor part of M (solver.py:479-489), 4N x 4N."""
    P, Q, _ = R.assemble_diagonal(st)
    return sp.bmat([[None, P], [Q, None]], format="csr")


def pairing(st):
    """The local pairing K of K mat_d = -mat_d^T K, 4N x 4N (four scaled identity blocks)."""
    g = D.metric(st)
    n = st["n"]
    gx, gy = R._dg(g[:n]), R._dg(g[n:])
    return sp.bmat([[None, None, None, gx], [None, None, -gy, None], [None, gy, None, None], [-gx, None, None, None]], format="csr")


def operator(st, msign=1.0):
    """mat = msign (-i) M, the operator the solver iterates with (solver.py:655-670)."""
    return (msign * -1j) * R.assemble_tensorial(st)


def _with_coef(st, coef):
    s = dict(st)
    s["coef"] = coef
    return s


def dM_dfreq(st, freq):
    """dM/df at fixed permittivity (exact: M has degree <= 2 in the coefficients)."""
    d = D.coef_direction(st, freq)
    plus = [tuple(c + e for c, e in zip(cs, ds)) for cs, ds in zip(st["coef"], d)]
    minus = [tuple(c - e for c, e in zip(cs, ds)) for cs, ds in zip(st["coef"], d)]
    return (R.assemble_tensorial(_with_coef(st, plus)) - R.assemble_tensorial(_with_coef(st, minus))) / (2.0 * freq)


def eigenpairs(st, k, sigma=None, tol=1e-13, msign=1.0):
    """Right and left eigenpairs of mat = msign (-i) M nearest sigma (default: the solver's target), largest Re n first.

    Returns (n, u, n_left, w): n_left[q] is the eigenvalue of mat^T nearest n[q] and w[:, q] its eigenvector."""
    M = operator(st, msign).tocsc()
    sigma = st["target"] if sigma is None else sigma
    vals, vecs = spl.eigs(M, k=k, sigma=sigma, tol=tol)
    order = np.argsort(vals.real)[::-1]
    vals, vecs = vals[order], vecs[:, order]
    lvals, lvecs = spl.eigs(M.T.tocsc(), k=k, sigma=sigma, tol=tol)
    pick = [int(np.argmin(np.abs(lvals - v))) for v in vals]
    return vals, vecs, lvals[pick], lvecs[:, pick]


def dn_dfreq(st, freq, u, w, msign=1.0):
    """dn/df at fixed permittivity of the eigenvalue n of mat = msign (-i) M (solver units, before knorm) from the right / left
    eigenvectors u, w."""
    return (msign * -1j) * (w @ (dM_dfreq(st, freq) @ u)) / (w @ u)


# --------------------------------------------------------------------------------------------
# permittivity gradient: M is affine in the per-site derived fields q of eps (and of mu, held fixed here)
# --------------------------------------------------------------------------------------------
# q_e = [t_zx/t_zz, t_zy/t_zz, 1/t_zz, t_yz/t_zz, t_xz/t_zz, S_xx, S_xy, S_yx, S_yy] of the solver-frame eps' (the order of the
# device's coefficient fields), S_ab = t_ab - t_az t_zb / t_zz.  Each entry is (row block, column block, sign, left factor,
# q index, right factor): the block holds sign * left diag(q) right.
def _eps_terms(st):
    dxf, dxb, dyf, dyb = R.d_matrices(st)
    return [
        (0, 0, -1, dxf, 0, None), (0, 1, -1, dxf, 1, None), (0, 2, -1, dxf, 2, dyb), (0, 3, 1, dxf, 2, dxb),
        (1, 0, -1, dyf, 0, None), (1, 1, -1, dyf, 1, None), (1, 2, -1, dyf, 2, dyb), (1, 3, 1, dyf, 2, dxb),
        (2, 0, 1, None, 7, None), (2, 1, 1, None, 8, None), (2, 2, -1, None, 3, dyb), (2, 3, 1, None, 3, dxb),
        (3, 0, -1, None, 5, None), (3, 1, -1, None, 6, None), (3, 2, 1, None, 4, dyb), (3, 3, -1, None, 4, dxb),
    ]


def _dq_dt(t):
    """d q_e / d t'_ab, shape (9 q, 3, 3, N), for the solver-frame tensor t (3, 3, N)."""
    n = t.shape[-1]
    z = t[2, 2]
    out = np.zeros((9, 3, 3, n), complex)
    for j, (a, b) in enumerate(((2, 0), (2, 1))):
        out[j, a, b] = 1 / z
        out[j, 2, 2] = -t[a, b] / z**2
    out[2, 2, 2] = -1 / z**2
    for j, (a, b) in zip((3, 4), ((1, 2), (0, 2))):
        out[j, a, b] = 1 / z
        out[j, 2, 2] = -t[a, b] / z**2
    for j, (a, b) in zip((5, 6, 7, 8), ((0, 0), (0, 1), (1, 0), (1, 1))):
        out[j, a, b] = 1.0
        out[j, a, 2] = -t[2, b] / z
        out[j, 2, b] = -t[a, 2] / z
        out[j, 2, 2] = t[a, 2] * t[2, b] / z**2
    return out


def dmat_dq(st, u, w, msign=1.0):
    """w^T (d mat / d q_e[j](g)) u, shape (9, N) (not yet divided by w^T u)."""
    n = st["n"]
    ub = [u[i * n:(i + 1) * n] for i in range(4)]
    wb = [w[i * n:(i + 1) * n] for i in range(4)]
    out = np.zeros((9, n), complex)
    for r, c, sgn, left, j, right in _eps_terms(st):
        lw = wb[r] if left is None else left.T @ wb[r]
        ru = ub[c] if right is None else right @ ub[c]
        out[j] += sgn * lw * ru
    return (msign * -1j) * out


def dn_deps_tensor(eps_cross, coords, freq, mode_spec, u, w, symmetry=(0, 0), mu_cross=None, msign=1.0):
    """dn / d eps_cross[k] at every site, shape (9, nx, ny), k in the eps_cross order (row-major xx, xy, ..., zz), in the
    solver's units (multiply by knorm for the reported index).  Taken at fixed PML stretch, through the angle / bend congruence
    eps' = J eps J^T / det J; entries of eps' that the PEC model replaces report 0."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    u, w = np.asarray(u, complex), np.asarray(w, complex)
    cq = dmat_dq(st, u, w, msign) / (w @ u)
    jac = st["jac_e"]
    det = np.linalg.det(np.moveaxis(jac, [0, 1], [-2, -1]))
    raw = np.array([np.asarray(eps_cross[i], complex).ravel() for i in range(9)]).reshape(3, 3, -1)
    t = np.einsum("acn,cdn,bdn->abn", jac, raw, jac) / det
    gt = np.einsum("jn,jabn->abn", cq, _dq_dt(st["eps"]))
    gt[t <= 0.9 * R.PEC_VAL] = 0.0
    g = np.einsum("abn,acn,bdn->cdn", gt, jac, jac) / det
    return g.reshape(9, st["nx"], st["ny"])


def derivatives(eps_cross, coords, freq, mode_spec, u, w, symmetry=(0, 0), mu_cross=None, eps_dfreq=None, msign=1.0):
    """dn/df (with the material dispersion of the nine-component eps_dfreq when given), n_group and the (9, nx, ny)
    permittivity gradient of one mode, in the reported units (times knorm)."""
    st = R.setup(eps_cross, coords, freq, mode_spec, symmetry, mu_cross)
    u, w = np.asarray(u, complex), np.asarray(w, complex)
    dn_df = dn_dfreq(st, freq, u, w, msign)
    geps = dn_deps_tensor(eps_cross, coords, freq, mode_spec, u, w, symmetry, mu_cross, msign)
    if eps_dfreq is not None:
        dn_df = dn_df + np.sum(geps * np.array([np.asarray(e, complex) for e in eps_dfreq]))
    n = (w @ (operator(st, msign) @ u)) / (w @ u) * st["knorm"]
    dn_df = dn_df * st["knorm"]
    return dict(n=n, dn_dfreq=dn_df, n_group=D.n_group(n, dn_df, freq), dn_deps_tensor=geps * st["knorm"])
