"""Float64 / complex128 model of the Krylov vector operations of the eigen-solver (csrc/krylov_kernels.cuh, csrc/solver.cuh),
with the device's conventions, for the GPU tests of b200ms_debug_krylov:

- dots are conjugate-linear in the basis vector: h_i = <V_i, w> = sum conj(V_i) w;
- the inner Gram-Schmidt is CGS2: two classical passes, their coefficients summed; ||w''||^2 = 0 (below 1e-60) gives y = 0;
- the outer orthonormalisation is ARPACK's DGKS: a second pass only when ||w'||^2 < 0.5 (||w'||^2 + sum |h|^2) for some active
  problem of the batch (the test runs on the first pass's h);
- the least-squares problem of an FGMRES cycle is solved by Givens rotations from e_1, stopping at the first column whose
  residual estimate is <= tol or whose subdiagonal is zero (breakdown); y is zero past the columns used;
- a refinement step adds ||r|| sum_k y_k Z_k to x.

Vectors are (nprob, len) arrays, bases (nv, nprob, len)."""
import numpy as np


def dots(V, w):
    """h[b, i] = sum_e conj(V[i, b, e]) w[b, e]."""
    return np.einsum("ibe,be->bi", np.conj(V), w)


def abs_dots(V, w):
    """sum_e |V[i, b, e]| |w[b, e]|: the scale of each dot product (an error bound that cancellation cannot shrink)."""
    return np.einsum("ibe,be->bi", np.abs(V), np.abs(w))


def _project(V, w, h):
    return w - np.einsum("bi,ibe->be", h, V)


def normalise(w):
    """(y, ||w||^2) with y = w / ||w||, y = 0 where ||w||^2 <= 1e-60."""
    n2 = np.sum(np.abs(w) ** 2, axis=-1)
    al = np.where(n2 > 1e-60, 1.0 / np.sqrt(np.where(n2 > 1e-60, n2, 1.0)), 0.0)
    return al[:, None] * w, n2


def cgs2(V, w):
    """Inner CGS2: (y, h, n2) with h the two passes' coefficients summed and n2 = ||w''||^2."""
    h1 = dots(V, w)
    w1 = _project(V, w, h1)
    h2 = dots(V, w1)
    w2 = _project(V, w1, h2)
    y, n2 = normalise(w2)
    return y, h1 + h2, n2


def dgks(V, w, skip=None):
    """Outer orthonormalisation with the DGKS test (BatchSolver::orthonormalise_dev): (y, h, ||w||, second)."""
    h = dots(V, w)
    w1 = _project(V, w, h)
    n2 = np.sum(np.abs(w1) ** 2, axis=-1)
    before = n2 + np.sum(np.abs(h) ** 2, axis=-1)
    active = np.ones(len(w), bool) if skip is None else ~np.asarray(skip, bool)
    second = bool(np.any(~(n2[active] >= 0.5 * before[active])))
    if second:
        h2 = dots(V, w1)
        w1 = _project(V, w1, h2)
        h = h + h2
        n2 = np.sum(np.abs(w1) ** 2, axis=-1)
    y, _ = normalise(w1)
    return y, h, np.sqrt(np.maximum(n2, 0.0)), second


def round1(V, w, selective, skip=None):
    """Round-1 orthonormalisation (BatchSolver::orthonormalise): CGS2, or with `selective` one pass and a second one only when
    ||w'||^2 < 1e-4 ||w||^2 for some active problem.  Returns (y, h, ||w||, second)."""
    h = dots(V, w)
    w1 = _project(V, w, h)
    second = not selective
    if selective:
        ww = np.sum(np.abs(w) ** 2, axis=-1)
        after = np.sum(np.abs(w1) ** 2, axis=-1)
        active = np.ones(len(w), bool) if skip is None else ~np.asarray(skip, bool)
        second = bool(np.any(~(after[active] >= 1e-4 * ww[active])))
    if second:
        h2 = dots(V, w1)
        w1 = _project(V, w1, h2)
        h = h + h2
    y, n2 = normalise(w1)
    return y, h, np.sqrt(n2), second


def givens_lsq(H, kc, tol):
    """FGMRES least squares from e_1.  H: (nprob, kc, kc + 1) columns (h_0j..h_jj, then ||w_j||^2 in row j + 1, real part
    read); tol: (nprob,), < 0 = inactive.  Returns (y (nprob, kc), res (nprob,), jused (nprob,))."""
    nb = H.shape[0]
    y = np.zeros((nb, kc), complex)
    res = np.zeros(nb)
    jused = np.zeros(nb, int)
    for b in range(nb):
        if tol[b] < 0:
            continue
        R = np.zeros((kc + 1, kc), complex)
        cs, sn = [], []
        g = np.zeros(kc + 1, complex)
        g[0] = 1.0
        ju, r = 0, 1.0
        for j in range(kc):
            col = H[b, j, : j + 1].astype(complex)
            sub = np.sqrt(max(0.0, H[b, j, j + 1].real))
            for i in range(j):
                a0, a1 = col[i], col[i + 1]
                col[i] = np.conj(cs[i]) * a0 + np.conj(sn[i]) * a1
                col[i + 1] = cs[i] * a1 - sn[i] * a0
            d = np.hypot(abs(col[j]), sub)
            c, s = (col[j] / d, sub / d) if d > 0 else (1.0 + 0j, 0.0 + 0j)
            cs.append(c)
            sn.append(s)
            col[j] = d
            R[: j + 1, j] = col
            g[j + 1] = -s * g[j]
            g[j] = np.conj(c) * g[j]
            ju = j + 1
            r = abs(g[j + 1])
            if r <= tol[b] or not sub > 0:
                break
        for i in range(ju - 1, -1, -1):
            acc = g[i] - np.dot(R[i, i + 1 : ju], y[b, i + 1 : ju])
            y[b, i] = acc / R[i, i] if abs(R[i, i]) ** 2 > 1e-300 else 0.0
        res[b], jused[b] = r, ju
    return y, res, jused


def lstsq_reference(H, kc):
    """min || e_1 - Hbar y || by numpy.linalg.lstsq, Hbar the (kc + 1) x kc Hessenberg matrix of H (subdiagonal = sqrt of the
    exported ||w_j||^2): the model's Givens solve with tol = 0 must agree with it when no breakdown occurs."""
    nb = H.shape[0]
    y = np.zeros((nb, kc), complex)
    res = np.zeros(nb)
    for b in range(nb):
        Hb = np.zeros((kc + 1, kc), complex)
        for j in range(kc):
            Hb[: j + 1, j] = H[b, j, : j + 1]
            Hb[j + 1, j] = np.sqrt(max(0.0, H[b, j, j + 1].real))
        e1 = np.zeros(kc + 1, complex)
        e1[0] = 1.0
        y[b] = np.linalg.lstsq(Hb, e1, rcond=None)[0]
        res[b] = np.linalg.norm(e1 - Hb @ y[b])
    return y, res


def ir_step(r, Z, y, skip=None):
    """Refinement step on x = r: (r / ||r|| (0 when skipped or ||r||^2 <= 1e-300), r + ||r|| sum_k y_k Z_k, ||r||^2)."""
    n2 = np.sum(np.abs(r) ** 2, axis=-1)
    on = n2 > 1e-300 if skip is None else (n2 > 1e-300) & ~np.asarray(skip, bool)
    al = np.where(on, 1.0 / np.sqrt(np.where(n2 > 0, n2, 1.0)), 0.0)
    x = r + np.sqrt(n2)[:, None] * np.einsum("bk,kbe->be", y, Z)
    return al[:, None] * r, x, n2


def lincomb(V, Q, nk):
    """out[q, b] = sum_i Q[b, i, q] V[i, b], q < nk."""
    return np.einsum("biq,ibe->qbe", Q[:, :, :nk], V)
