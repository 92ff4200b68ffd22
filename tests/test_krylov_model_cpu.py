"""CPU: the Krylov model oracle/krylov_model.py against numpy's own QR and least squares, on random and constructed cases.  The
GPU tests (test_gpu_krylov_kernels.py) compare the device kernels with this model, so the model is pinned first."""
import numpy as np
import pytest

from oracle import krylov_model as K


def _vecs(rng, shape, real):
    v = rng.standard_normal(shape)
    return v + 0j if real else v + 1j * rng.standard_normal(shape)


def _orthonormal(rng, nv, nb, n, real):
    V = np.empty((nv, nb, n), complex)
    for b in range(nb):
        V[:, b, :] = np.linalg.qr(_vecs(rng, (n, nv), real))[0].T
    return V


@pytest.mark.parametrize("real", [True, False])
@pytest.mark.parametrize("nv", [1, 3, 9])
def test_cgs2_matches_qr(real, nv):
    """[V, w] = [V, y] R: the last column of numpy's QR is y up to a unit phase, the coefficients are V^H w and ||w - V h||."""
    rng = np.random.default_rng(nv)
    nb, n = 3, 57
    V = _orthonormal(rng, nv, nb, n, real)
    w = _vecs(rng, (nb, n), real)
    y, h, n2 = K.cgs2(V, w)
    for b in range(nb):
        q, r = np.linalg.qr(np.column_stack([V[:, b, :].T, w[b]]))
        ph = r[nv, nv] / abs(r[nv, nv])
        assert np.allclose(y[b], ph * q[:, nv], atol=1e-13)
        assert np.allclose(h[b], V[:, b, :].conj() @ w[b], atol=1e-13)
        assert np.isclose(np.sqrt(n2[b]), abs(r[nv, nv]), rtol=1e-13)
        assert np.abs(V[:, b, :].conj() @ y[b]).max() < 1e-14


def test_w_in_the_span_and_w_zero():
    rng = np.random.default_rng(3)
    V = _orthonormal(rng, 4, 2, 40, False)
    w = np.stack([V[:, 0, :].T @ np.array([1.0, -2.0, 0.5j, 3.0]), np.zeros(40)])
    y, h, n2 = K.cgs2(V, w)
    assert np.allclose(h[0], [1.0, -2.0, 0.5j, 3.0], atol=1e-14) and n2[0] < 1e-28
    assert (h[1] == 0).all() and n2[1] == 0 and (y[1] == 0).all()  # ||w||^2 = 0: y = 0, no division
    # w in the span: the DGKS test fires (||w'||^2 ~ 0 < 0.5 ||w||^2) and the second pass is taken
    _, hd, nrm, second = K.dgks(V, w)
    assert second and np.allclose(hd[0], [1.0, -2.0, 0.5j, 3.0], atol=1e-14) and nrm[0] < 1e-13
    # ... unless that problem is skipped: then w = 0 alone does not fire it (0 >= 0.5 * 0)
    assert not K.dgks(V, w, skip=[True, False])[3]
    # a w well away from the span: one pass
    w2 = _vecs(rng, (2, 40), False)
    w2 -= 0.1 * np.einsum("bi,ibe->be", K.dots(V, w2), V)
    assert not K.dgks(V, w2)[3]


def test_round1_selective_pass():
    rng = np.random.default_rng(8)
    V = _orthonormal(rng, 3, 2, 30, True)
    w = _vecs(rng, (2, 30), True)
    assert not K.round1(V, w, True)[3] and K.round1(V, w, False)[3]
    w[1] = V[:, 1, :].T @ np.array([1.0, 2.0, 3.0]) + 1e-6 * w[1]  # ||w'|| ~ 1e-6 ||w||: cancellation, second pass
    y, h, nrm, second = K.round1(V, w, True)
    assert second
    yr, hr, nr = K.cgs2(V, w)
    assert np.allclose(y, yr, atol=1e-12) and np.allclose(h, hr, atol=1e-14) and np.allclose(nrm, np.sqrt(nr))


def _hessenberg(rng, nb, kc, real):
    """Exported layout [b][j][kc + 1]: h_0j..h_jj, then ||w_j||^2 (positive)."""
    H = np.zeros((nb, kc, kc + 1), complex)
    for b in range(nb):
        for j in range(kc):
            H[b, j, : j + 1] = _vecs(rng, j + 1, real)
            H[b, j, j + 1] = rng.uniform(0.1, 2.0) ** 2
    return H


@pytest.mark.parametrize("real", [True, False])
@pytest.mark.parametrize("kc", [1, 2, 5, 17])
def test_givens_lsq_matches_lstsq(real, kc):
    rng = np.random.default_rng(kc)
    H = _hessenberg(rng, 3, kc, real)
    y, res, ju = K.givens_lsq(H, kc, np.zeros(3))
    yr, rr = K.lstsq_reference(H, kc)
    assert (ju == kc).all()
    assert np.allclose(y, yr, rtol=1e-10, atol=1e-12) and np.allclose(res, rr, rtol=1e-10, atol=1e-14)


def test_givens_lsq_early_stop_breakdown_and_inactive():
    rng = np.random.default_rng(5)
    kc = 8
    H = _hessenberg(rng, 3, kc, False)
    _, res_all, _ = K.givens_lsq(H, kc, np.zeros(3))
    # problem 0 stops at the first column whose estimate is <= tol
    _, r_cols, _ = zip(*[K.givens_lsq(H[:1], j, np.zeros(1)) for j in range(1, kc + 1)])
    tol0 = 0.5 * (r_cols[3][0] + r_cols[2][0])  # between the estimates after 3 and 4 columns: stops at 4
    assert r_cols[3][0] < tol0 < r_cols[2][0]
    # problem 1 breaks down in column 2 (zero subdiagonal: the Krylov space is invariant, the solve is exact)
    H[1, 2, 3] = 0.0
    y, res, ju = K.givens_lsq(H, kc, np.array([tol0, 0.0, -1.0]))
    assert ju[0] == 4 and res[0] <= tol0 and (y[0, 4:] == 0).all()
    yr, rr = K.lstsq_reference(H[:1, :4, :5], 4)
    assert np.allclose(y[0, :4], yr[0], rtol=1e-10) and np.isclose(res[0], rr[0], rtol=1e-10)
    assert ju[1] == 3 and res[1] < 1e-14 and (y[1, 3:] == 0).all()
    yr, rr = K.lstsq_reference(H[1:2, :3, :4], 3)
    assert np.allclose(y[1, :3], yr[0], rtol=1e-10) and rr[0] < 1e-14
    # problem 2 is inactive: y = 0, estimate 0, no columns
    assert ju[2] == 0 and res[2] == 0 and (y[2] == 0).all()
    assert res_all.shape == (3,)


def test_ir_step_and_lincomb():
    rng = np.random.default_rng(2)
    nb, n, nv = 3, 20, 4
    r = _vecs(rng, (nb, n), False)
    r[2] = 0
    Z = _vecs(rng, (nv, nb, n), False)
    y = _vecs(rng, (nb, nv), False)
    rp, x, n2 = K.ir_step(r, Z, y, skip=[False, True, False])
    nr = np.linalg.norm(r, axis=1)
    assert np.allclose(rp[0], r[0] / nr[0]) and (rp[1] == 0).all() and (rp[2] == 0).all()
    assert np.allclose(n2, nr**2)
    for b in range(nb):
        assert np.allclose(x[b], r[b] + nr[b] * (Z[:, b, :].T @ y[b]))
    Q = _vecs(rng, (nb, nv, 6), False)
    out = K.lincomb(Z, Q, 5)
    assert out.shape == (5, nb, n)
    for b in range(nb):
        assert np.allclose(out[:, b, :], (Z[:, b, :].T @ Q[b, :, :5]).T)
