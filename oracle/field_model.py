"""Float64 model of the device field recovery (the epilogue, test-only).

Maps the eigenvectors of one problem, as ``oracle.mg_model.Problem`` sees it, to the six field components the caller receives,
written in the expression form of ``epilogue_kernel`` / ``tensor_epilogue_kernel`` (``csrc/kernels.cuh``):

- diagonal problems, v = [Ex; Ey] (``DiagSite``):  t = imz (Dxf v2 - Dyf v1),  q1 = Dxb t + eyy v2,  q2 = Dyb t - exx v1,
  u = -iez (Dxb exx v1 + Dyb eyy v2);  E = (Ex, Ey, u / (i n)),  H = (-i / eta0) (q1 / (i n), q2 / (i n), t).  The restatement's
  Ez = iez (Dxb Hy - Dyb Hx) is the same value in exact arithmetic but cancels badly next to a PEC-model eps of about 1e8.
  Direction "-" negates Hx, Hy and Ez (solver.py:370-373).  With the incidence formulation and PEC cells the problem's
  zero-marked fields are used (``Problem.fields``).
- tensorial problems, v = [Ex; Ey; Hx; Hy]: Ez = U, Hz = (-i / eta0) Tt from the derived fields t_zx / t_zz, t_zy / t_zz,
  1 / t_zz of eps and mu (``TensorCell``); H = (-i / eta0) (Hx, Hy, Tt).  tensorial_real with direction "-": E = conj(E),
  H = -conj(H) (solver.py:378-380).
- then E = J^T E', H = J^T H' with the angled / bend Jacobian (solver.py:254-259): only the z components change.

Next to each field entry the model returns the sum of the absolute values of its terms (the same expression with every
coefficient, value and difference replaced by absolute values and sums): the scale of its rounding error, so that a test
scaled by it sees through cancellation.

Nothing under ``tidy3d_b200/`` imports this module.
"""
from __future__ import annotations

import numpy as np

from oracle import restatement as R


def _nx(a):  # a[:, i + 1, :], zero past the last row
    out = np.zeros_like(a)
    out[:, :-1] = a[:, 1:]
    return out


def _px(a):  # a[:, i - 1, :], zero before the first row
    out = np.zeros_like(a)
    out[:, 1:] = a[:, :-1]
    return out


def _ny(a):
    out = np.zeros_like(a)
    out[:, :, :-1] = a[:, :, 1:]
    return out


def _py(a):
    out = np.zeros_like(a)
    out[:, :, 1:] = a[:, :, :-1]
    return out


def eps_complex(prob):
    """The device's tensorial kind: tensorial_complex when eps has an imaginary part (solver.py:389-411)."""
    return bool(R._is_complex(prob.st["eps"]))


def conj_flip(prob, direction):
    return prob.tensorial and direction == "-" and not eps_complex(prob)


def _coef(prob):
    (xf0, xf1, xb0, xbm), (yf0, yf1, yb0, ybm) = prob.axes[0].coefficients(), prob.axes[1].coefficients()
    X = lambda c: c[None, :, None]  # noqa: E731
    Y = lambda c: c[None, None, :]  # noqa: E731
    return (X(xf0), X(xf1), X(xb0), X(xbm)), (Y(yf0), Y(yf1), Y(yb0), Y(ybm))


def _diagonal(prob, v1, v2, n):
    """(Ex, Ey, Ez, Hx, Hy, Hz) before the direction sign and J^T, and their term sums."""
    (xf0, xf1, xb0, xbm), (yf0, yf1, yb0, ybm) = _coef(prob)
    exx, eyy, iez, _, _, imz = (f[None] for f in prob.fields)
    a1, a2 = np.abs(v1), np.abs(v2)
    t = imz * (xf0 * v2 + xf1 * _nx(v2) - yf0 * v1 - yf1 * _ny(v1))
    ts = np.abs(imz) * (np.abs(xf0) * a2 + np.abs(xf1) * _nx(a2) + np.abs(yf0) * a1 + np.abs(yf1) * _ny(a1))
    q1 = xb0 * t + xbm * _px(t) + eyy * v2
    q1s = np.abs(xb0) * ts + np.abs(xbm) * _px(ts) + np.abs(eyy) * a2
    q2 = yb0 * t + ybm * _py(t) - exx * v1
    q2s = np.abs(yb0) * ts + np.abs(ybm) * _py(ts) + np.abs(exx) * a1
    ev1, ev2 = exx * v1, eyy * v2
    es1, es2 = np.abs(exx) * a1, np.abs(eyy) * a2
    u = -iez * (xb0 * ev1 + yb0 * ev2 + xbm * _px(ev1) + ybm * _py(ev2))
    us = np.abs(iez) * (np.abs(xb0) * es1 + np.abs(yb0) * es2 + np.abs(xbm) * _px(es1) + np.abs(ybm) * _py(es2))
    inv = (1 / (1j * np.asarray(n, complex)))[:, None, None]
    hs = -1j / R.ETA_0
    F = [v1 + 0j, v2 + 0j, u * inv, hs * q1 * inv, hs * q2 * inv, hs * t]
    S = [a1, a2, us * abs(inv), abs(hs) * q1s * abs(inv), abs(hs) * q2s * abs(inv), abs(hs) * ts]
    return F, S


def _tensorial(prob, ex, ey, hx, hy):
    (xf0, xf1, xb0, xbm), (yf0, yf1, yb0, ybm) = _coef(prob)
    nx, ny = prob.nx, prob.ny
    e, m = (np.asarray(prob.st[k], complex).reshape(3, 3, nx, ny) for k in ("eps", "mu"))
    f0, f1, f2 = (e[2, 0] / e[2, 2])[None], (e[2, 1] / e[2, 2])[None], (1 / e[2, 2])[None]
    f9, f10, f11 = (m[2, 0] / m[2, 2])[None], (m[2, 1] / m[2, 2])[None], (1 / m[2, 2])[None]
    A = np.abs
    K = xb0 * hy + xbm * _px(hy) - yb0 * hx - ybm * _py(hx)
    Ks = A(xb0) * A(hy) + A(xbm) * _px(A(hy)) + A(yb0) * A(hx) + A(ybm) * _py(A(hx))
    G = xf0 * ey + xf1 * _nx(ey) - yf0 * ex - yf1 * _ny(ex)
    Gs = A(xf0) * A(ey) + A(xf1) * _nx(A(ey)) + A(yf0) * A(ex) + A(yf1) * _ny(A(ex))
    U = f2 * K - f0 * ex - f1 * ey
    Us = A(f2) * Ks + A(f0) * A(ex) + A(f1) * A(ey)
    Tt = f11 * G - f9 * hx - f10 * hy
    Tts = A(f11) * Gs + A(f9) * A(hx) + A(f10) * A(hy)
    hs = -1j / R.ETA_0
    F = [ex + 0j, ey + 0j, U, hs * hx, hs * hy, hs * Tt]
    S = [A(ex), A(ey), Us, abs(hs) * A(hx), abs(hs) * A(hy), abs(hs) * Tts]
    return F, S


def fields(prob, vecs, n=None, perm=None, direction="+"):
    """The six components of every mode.

    vecs: (k, len) complex, the eigenvectors in Ritz-slot order (len = 2 N, or 4 N tensorial); n: (k,) complex n_eff + i k_eff
    of output mode q in solver units (the delivered n_complex / knorm; unused for tensorial problems); perm: (k,) ints,
    output mode q is slot perm[q] (identity when None).  Returns (F, S), each (2, 3, nx, ny, k): the fields in the delivered
    layout and the sums of the absolute values of their terms."""
    nx, ny = prob.nx, prob.ny
    N = nx * ny
    vecs = np.asarray(vecs, complex)
    k = vecs.shape[0]
    perm = np.arange(k) if perm is None else np.asarray(perm)
    w = vecs[perm].reshape(k, -1, nx, ny)
    assert w.shape[1] == (4 if prob.tensorial else 2) and vecs.shape[1] == w.shape[1] * N
    if prob.tensorial:
        F, S = _tensorial(prob, *w.transpose(1, 0, 2, 3))
        if conj_flip(prob, direction):
            F = [np.conj(f) if c < 3 else -np.conj(f) for c, f in enumerate(F)]
    else:
        F, S = _diagonal(prob, w[:, 0], w[:, 1], n)
        if direction == "-":
            F[2], F[3], F[4] = -F[2], -F[3], -F[4]
    # E = J^T E', H = J^T H':  z = J[0][2] x + J[1][2] y + J[2][2] z, the in-plane components unchanged
    for off, jac in ((0, prob.st["jac_e"]), (3, prob.st["jac_h"])):
        ja, jb, jd = (np.asarray(jac[a, 2], float).reshape(1, nx, ny) for a in range(3))
        F[off + 2] = ja * F[off] + jb * F[off + 1] + jd * F[off + 2]
        S[off + 2] = np.abs(ja) * S[off] + np.abs(jb) * S[off + 1] + np.abs(jd) * S[off + 2]
    to = lambda c: np.stack(c).reshape(2, 3, k, nx, ny).transpose(0, 1, 3, 4, 2)  # noqa: E731
    return to(F), to(S)


def vectors(prob, F, direction="+"):
    """The eigenvectors (k, len) behind delivered fields F (2, 3, nx, ny, k): (Ex, Ey), or (Ex, Ey, Hx, Hy) / (1, 1, -i/eta0,
    -i/eta0) with the conjugate flip undone.  J^T leaves the in-plane components unchanged."""
    F = np.asarray(F).reshape(2, 3, prob.nx * prob.ny, -1).astype(complex)
    if not prob.tensorial:
        return np.concatenate((F[0, 0], F[0, 1])).T.copy()
    e, h = F[0, :2], F[1, :2]
    if conj_flip(prob, direction):
        e, h = np.conj(e), -np.conj(h)
    hs = -1j / R.ETA_0
    return np.concatenate((e[0], e[1], h[0] / hs, h[1] / hs)).T.copy()
