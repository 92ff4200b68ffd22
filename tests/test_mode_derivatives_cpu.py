"""CPU: the float64 derivative model (oracle/mode_derivatives.py) against dense eigen-decompositions of the assembled operator.

For every case the left eigenvector w = G J Q v must satisfy A^T w = lambda w, the frequency derivative must match the central
difference of the eigenvalue itself, and summed permittivity sensitivities over a region must match the eigenvalue's central
difference under a perturbation of that region."""
import types

import numpy as np
import pytest

from oracle import mode_derivatives as D
from oracle import restatement as R

F0 = R.C_0 / 1.55


def _case(nx=14, ny=12, npml=(0, 0), sym=(0, 0), bend=None, lossy=False, nonuni=False, mu=False, disp=False):
    rng = np.random.default_rng(3)
    if nonuni:
        x = np.cumsum(np.r_[0, 0.12 + 0.08 * rng.random(nx)])
        y = np.cumsum(np.r_[0, 0.12 + 0.08 * rng.random(ny)])
    else:
        x, y = np.linspace(0, 0.16 * nx, nx + 1), np.linspace(0, 0.16 * ny, ny + 1)
    x, y = x - x.mean(), y - y.mean()
    if ny == 1:
        y = np.array([-0.1, 0.1])
    xc, yc = 0.5 * (x[1:] + x[:-1]), 0.5 * (y[1:] + y[:-1])
    core = (np.abs(xc)[:, None] < 0.5) & ((np.abs(yc)[None, :] < 0.3) | (ny == 1))

    def eps_at(f):
        e_core = 12.0 + (15.0 * (f / F0 - 1) if disp else 0.0) + (0.2j if lossy else 0)
        e = np.where(core, e_core, 2.07).astype(complex)
        out = [np.zeros((nx, ny), complex) for _ in range(9)]
        out[0], out[4], out[8] = e, e * 1.02, e * 0.97
        return out

    def deps_at(f):  # analytic d eps / df of eps_at
        d = np.where(core, 15.0 / F0, 0.0).astype(complex) if disp else np.zeros((nx, ny), complex)
        out = [np.zeros((nx, ny), complex) for _ in range(9)]
        out[0], out[4], out[8] = d, d * 1.02, d * 0.97
        return out

    mu_cross = None
    if mu:
        mu_cross = [np.zeros((nx, ny), complex) for _ in range(9)]
        mu_cross[0] = np.where(core, 1.3, 1.0).astype(complex)
        mu_cross[4] = np.where(core, 0.8, 1.0).astype(complex)
        mu_cross[8] = np.where(core, 1.1, 1.0).astype(complex)
    ms = types.SimpleNamespace(num_modes=2, target_neff=None, num_pml=npml, filter_pol=None, angle_theta=0.0, angle_phi=0.0,
                               precision="double", bend_radius=bend, bend_axis=1 if bend else None)
    return dict(x=x, y=y, core=core, eps_at=eps_at, deps_at=deps_at, mu=mu_cross, ms=ms, sym=sym, disp=disp)


CASES = {
    "plain": dict(),
    "pml": dict(npml=(3, 2)),
    "pmc_x_pec_y": dict(npml=(3, 2), sym=(1, -1)),
    "pec_x_pmc_y": dict(npml=(2, 3), sym=(-1, 1)),
    "pmc_both": dict(sym=(1, 1)),
    "bend": dict(npml=(3, 2), bend=4.0),
    "lossy_nonuniform": dict(npml=(3, 3), lossy=True, nonuni=True),
    "all": dict(npml=(3, 2), bend=4.0, lossy=True, nonuni=True, sym=(1, -1)),
    "mu_diag": dict(npml=(3, 2), mu=True, sym=(0, 1)),
    "slab_1d": dict(nx=40, ny=1, npml=(4, 0)),
    "dispersive": dict(npml=(3, 2), disp=True, sym=(1, 0)),
}


def _operator(c, f, eps=None):
    st = R.setup(c["eps_at"](f) if eps is None else eps, (c["x"], c["y"]), f, c["ms"], c["sym"], c["mu"])
    return R.assemble_diagonal(st)[2].toarray()


def _track(A, lam0):
    lam = np.linalg.eigvals(A)
    return lam[np.argmin(np.abs(lam - lam0))]


def _fundamental(c):
    A = _operator(c, F0)
    lam, V = np.linalg.eig(A)
    m = int(np.argmin(lam.real))  # largest Re(n^2)
    return lam[m], V[:, m]


@pytest.mark.parametrize("name", sorted(CASES))
def test_left_vector_frequency_and_region_derivatives(name):
    c = _case(**CASES[name])
    lam, v = _fundamental(c)
    out = D.derivatives(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"],
                        eps_dfreq=c["deps_at"](F0) if c["disp"] else None)
    assert out["residual"] <= 1e-12

    # d lambda / df against the eigenvalue's central difference (the medium moves with f only in the dispersive case)
    h = 1e-5 * F0
    fd = (_track(_operator(c, F0 + h), lam) - _track(_operator(c, F0 - h), lam)) / (2 * h)
    assert abs(out["dlam_dfreq"] - fd) <= 1e-8 * abs(fd)
    n = np.sqrt(-lam + 0j)
    assert np.isclose(out["dn_dfreq"], -fd / (2 * n), rtol=1e-8, atol=0)
    assert np.isclose(out["n_group"], n.real + F0 * (-fd / (2 * n)).real, rtol=1e-8, atol=0)

    # summed core sensitivities of each diagonal component against the eigenvalue's central difference; the step error
    # is bounded by Richardson: |FD(d) - exact| ~ (4/3) |FD(d) - FD(d/2)|
    core = c["core"]
    for comp, a in ((0, 0), (4, 1), (8, 2)):
        def fd_at(d):
            ep, em = c["eps_at"](F0), c["eps_at"](F0)
            ep[comp] = ep[comp] + d * core
            em[comp] = em[comp] - d * core
            return (_track(_operator(c, F0, ep), lam) - _track(_operator(c, F0, em), lam)) / (2 * d)

        step = 1e-3 * 12.0
        f1, f2 = fd_at(step), fd_at(step / 2)
        dn_region = np.sum(out["dn_deps"][a][core])
        want = -f1 / (2 * n)
        bound = 2 * abs(f1 - f2) / abs(2 * n) + 1e-9 * abs(want)
        assert abs(dn_region - want) <= bound, (a, dn_region, want, bound)


def test_pec_cells_report_zero():
    c = _case(npml=(2, 2))
    eps = c["eps_at"](F0)
    for comp in (0, 4, 8):
        eps[comp] = eps[comp].copy()
        eps[comp][0, 5] = R.PEC_VAL
    st = R.setup(eps, (c["x"], c["y"]), F0, c["ms"], c["sym"])
    A = R.assemble_diagonal(st)[2].toarray()
    lam, V = np.linalg.eig(A)
    m = int(np.argmin(lam.real))
    out = D.derivatives(eps, (c["x"], c["y"]), F0, c["ms"], V[:, m], lam[m], c["sym"])
    assert (out["dn_deps"][:, 0, 5] == 0).all()
    assert np.abs(out["dn_deps"]).max() > 0

