"""CPU: the float64 second-derivative model (oracle/mode_dispersion.py) against dense eigen-decompositions of the assembled
operator, on the cases of the first-order CPU test plus a medium with both eps' and eps''.

For every case the correction x must solve its bordered system, and d^2 lambda / df^2 must match the second central
difference of the tracked eigenvalue within twice the Richardson estimate of that difference's step error.  The unit
conversion ``plugin.dispersion_of`` must be the step -> 0 limit of ``plugin.group_index``."""
import numpy as np
import pytest

from oracle import mode_dispersion as M
from oracle import restatement as R
from tests.test_mode_derivatives_cpu import CASES, F0, _case, _fundamental, _operator

CASES2 = dict(CASES)
CASES2["dispersive_curved"] = dict(npml=(3, 2), sym=(0, 1))


def _curved(c):
    """Core eps(f) = 12 (1 + 0.3 u + 2 u^2), u = f / F0 - 1, with its analytic first and second derivatives."""
    core = c["core"]

    def comps(val):
        out = [np.zeros(core.shape, complex) for _ in range(9)]
        out[0], out[4], out[8] = val, val * 1.02, val * 0.97
        return out

    def eps_at(f):
        u = f / F0 - 1
        return comps(np.where(core, 12.0 * (1 + 0.3 * u + 2.0 * u * u), 2.07).astype(complex))

    def deps_at(f):
        u = f / F0 - 1
        return comps(np.where(core, 12.0 * (0.3 + 4.0 * u) / F0, 0.0).astype(complex))

    def d2eps_at(f):
        return comps(np.where(core, 12.0 * 4.0 / F0**2, 0.0).astype(complex))

    c.update(eps_at=eps_at, deps_at=deps_at, d2eps_at=d2eps_at, disp=True)
    return c


def _setup(name):
    c = _case(**CASES2[name])
    if name == "dispersive_curved":
        c = _curved(c)
    return c


def _inputs(c):
    if not c["disp"]:
        return None, None
    d2 = c["d2eps_at"](F0) if "d2eps_at" in c else None
    return c["deps_at"](F0), d2


@pytest.mark.parametrize("name", sorted(CASES2))
def test_correction_and_second_derivative(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    de, d2e = _inputs(c)
    out = M.second_derivatives(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"], eps_dfreq=de, eps_d2freq=d2e)

    # the correction solves its bordered system: (A - lambda) x = r (mu ~ 0 for an exact eigenpair) and w^T x = 0
    x, r, A, w = out["x"], out["r"], out["A"], out["w"]
    assert np.linalg.norm(A @ x - lam * x - r) <= 1e-12 * np.linalg.norm(r)
    assert abs(w @ x) <= 1e-12 * np.linalg.norm(w) * np.linalg.norm(x)

    # d^2 lambda / df^2 against the eigenvalue's second central difference, Richardson-bounded
    dl = out["dlam_dfreq"]

    def fd2(h):
        lp = _track_near(_operator(c, F0 + h), lam + dl * h)
        lm = _track_near(_operator(c, F0 - h), lam - dl * h)
        return (lp - 2 * lam + lm) / h**2

    h = 2e-3 * F0
    f1, f2 = fd2(h), fd2(h / 2)
    want = f2
    bound = 2 * (4.0 / 3.0) * abs(f1 - f2) + 1e-9 * abs(want)
    assert abs(out["d2lam_dfreq2"] - want) <= bound, (out["d2lam_dfreq2"], want, bound)
    # and the material terms matter in the dispersive cases
    if c["disp"]:
        plain = M.second_derivatives(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"])
        assert abs(plain["d2lam_dfreq2"] - want) > 10 * bound


def _track_near(A, lam0):
    lam = np.linalg.eigvals(A)
    return lam[np.argmin(np.abs(lam - lam0))]


def test_dispersion_of_is_the_limit_of_group_index():
    from tidy3d_b200 import plugin

    f0 = np.array([R.C_0 / 1.55, R.C_0 / 1.31])

    def n_of(f):  # cubic n(f) of two modes
        u = f / f0[0] - 1
        return np.stack([2.4 + 0.8 * u - 3.0 * u**2 + 5.0 * u**3, 1.9 + 0.5 * u + 1.5 * u**2 - 2.0 * u**3], axis=-1)

    def dn(f):
        u = f / f0[0] - 1
        return np.stack([0.8 - 6.0 * u + 15.0 * u**2, 0.5 + 3.0 * u - 6.0 * u**2], axis=-1) / f0[0]

    def d2n(f):
        u = f / f0[0] - 1
        return np.stack([-6.0 + 30.0 * u, 3.0 - 12.0 * u], axis=-1) / f0[0] ** 2

    exact = plugin.dispersion_of(f0[:, None], dn(f0), d2n(f0))
    est = []
    for step in (1e-3, 1e-4):
        f3 = np.outer(f0, (1 - step, 1, 1 + step)).ravel()
        est.append(plugin.group_index(n_of(f3), f3, step)[3])
    # the three-point formula is exact for quadratics: its error is O(step^2) from the cubic term
    assert np.all(np.abs(est[0] - exact) <= 1e-4 * np.abs(exact))
    assert np.all(np.abs(est[1] - exact) <= 1e-6 * np.abs(exact))
    assert np.all(np.abs(est[1] - exact) < np.abs(est[0] - exact))
    assert np.sign(exact).tolist() == np.sign(est[1]).tolist()
