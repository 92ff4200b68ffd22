"""CPU: the float64 third-derivative model (oracle/mode_third_order.py) against dense eigen-decompositions of the assembled
operator, on the cases of the first-order CPU test plus a core with a cubic eps(f).

For every case d^3 lambda / df^3 must match the third central difference of the tracked eigenvalue (steps f (1 +- h),
f (1 +- 2h)) within twice the Richardson estimate of that difference's step error, and the model's f^3 d^3A/df^3 must match a
Richardson-extrapolated third difference of the assembled operator.  lambda''' must not depend on the multiple of v in x (and
of w in w_hat), and the first-order identity w_hat^T (A' - lambda') v = w^T (A' - lambda') x must hold.  The unit conversions
``plugin.dispersion_slope_of`` and ``plugin.beta3_of`` must be the step -> 0 limits of finite differences of
``plugin.dispersion_of`` over wavelength and of beta(omega)."""
import numpy as np
import pytest

from oracle import mode_third_order as M3
from oracle import restatement as R
from tests.test_mode_derivatives_cpu import CASES, F0, _case, _fundamental, _operator

CASES3 = dict(CASES)
CASES3["dispersive_cubic"] = dict(npml=(3, 2), sym=(0, 1))
EPS0 = 12.0
CUBIC = (0.05, 0.2, 0.3)  # eps(f) = eps0 (1 + a u + b u^2 + c u^3), u = f / F0 - 1


def _cubic(c):
    """Core eps(f) = 12 (1 + 0.05 u + 0.2 u^2 + 0.3 u^3) with its analytic first, second and third derivatives."""
    core = c["core"]
    a, b, k = CUBIC

    def comps(val):
        out = [np.zeros(core.shape, complex) for _ in range(9)]
        out[0], out[4], out[8] = val, val * 1.02, val * 0.97
        return out

    def eps_at(f):
        u = f / F0 - 1
        return comps(np.where(core, EPS0 * (1 + a * u + b * u * u + k * u**3), 2.07).astype(complex))

    def deps_at(f):
        u = f / F0 - 1
        return comps(np.where(core, EPS0 * (a + 2 * b * u + 3 * k * u * u) / F0, 0.0).astype(complex))

    def d2eps_at(f):
        u = f / F0 - 1
        return comps(np.where(core, EPS0 * (2 * b + 6 * k * u) / F0**2, 0.0).astype(complex))

    def d3eps_at(f):
        return comps(np.where(core, EPS0 * 6 * k / F0**3, 0.0).astype(complex))

    c.update(eps_at=eps_at, deps_at=deps_at, d2eps_at=d2eps_at, d3eps_at=d3eps_at, disp=True)
    return c


def _setup(name):
    c = _case(**CASES3[name])
    return _cubic(c) if name == "dispersive_cubic" else c


def _inputs(c):
    if not c["disp"]:
        return dict()
    out = dict(eps_dfreq=c["deps_at"](F0))
    if "d2eps_at" in c:
        out.update(eps_d2freq=c["d2eps_at"](F0), eps_d3freq=c["d3eps_at"](F0))
    return out


def _model(c, v, lam, **kw):
    return M3.third_derivatives(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"], **_inputs(c), **kw)


def _track_near(A, lam0):
    lam = np.linalg.eigvals(A)
    return lam[np.argmin(np.abs(lam - lam0))]


def _third_difference(fn, h):
    """Scaled third central difference f^3 d^3/df^3 of fn(f) at F0 with relative step h: steps f (1 +- h), f (1 +- 2h)."""
    return (fn(F0 * (1 + 2 * h)) - 2 * fn(F0 * (1 + h)) + 2 * fn(F0 * (1 - h)) - fn(F0 * (1 - 2 * h))) / (2 * h**3)


@pytest.mark.parametrize("name", sorted(CASES3))
def test_third_derivative_matches_dense_eigenvalues(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    l1, l2, l3 = out["lam1"], out["lam2"], out["lam3"]

    def lam_at(f):  # the eigenvalue tracked from its own Taylor prediction
        t = f / F0 - 1
        return _track_near(_operator(c, f), lam + l1 * t + l2 * t * t / 2 + l3 * t**3 / 6)

    h = 2e-2
    f1, f2 = _third_difference(lam_at, h), _third_difference(lam_at, h / 2)
    want = f2
    bound = 2 * abs(f1 - f2) / 3 + 1e-7 * abs(want)
    print(f"[third] {name}: lambda''' {l3:.8e}, fd {want:.8e}, |diff| {abs(l3 - want):.2e}, bound {bound:.2e}")
    assert abs(l3 - want) <= bound, (l3, want, bound)
    assert np.isclose(out["d3lam_dfreq3"], l3 / F0**3, rtol=1e-15, atol=0)
    if c["disp"] and name == "dispersive_cubic":  # the third-order material terms matter here
        nd = _model(dict(c, disp=False), v, lam)
        assert abs(nd["lam3"] - want) > 10 * bound


@pytest.mark.parametrize("name", sorted(CASES3))
def test_third_operator_is_exact(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    A3 = _model(c, v, lam)["A3"].toarray()
    d = [_third_difference(lambda f: _operator(c, f), h) for h in (4e-2, 2e-2)]
    rich = (4 * d[1] - d[0]) / 3
    scale = np.abs(A3).max()
    err = np.abs(A3 - rich).max()
    bound = 2 * np.abs(d[0] - d[1]).max() / 3 + 1e-8 * scale
    assert err <= bound, (err, bound)
    assert scale > 0


@pytest.mark.parametrize("name", ["plain", "pml", "all", "mu_diag", "dispersive_cubic"])
def test_invariance_and_first_order_identity(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    x, w, w_hat = out["x"], out["w"], out["w_hat"]
    for alpha in (0.3 - 0.7j, 2.0):
        moved = _model(c, v, lam, x=x + alpha * v, w_hat=w_hat + alpha * w)
        assert abs(moved["lam3"] - out["lam3"]) <= 1e-12 * abs(out["lam3"]), (alpha, moved["lam3"], out["lam3"])
    A1 = out["A1"]
    lhs = w_hat @ (A1 @ v - out["lam1"] * v)
    rhs = w @ (A1 @ x - out["lam1"] * x)
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), np.linalg.norm(w) * np.linalg.norm(A1 @ x)), (lhs, rhs)


def test_unit_helpers_are_the_limits_of_finite_differences():
    from tidy3d_b200 import plugin

    f0 = np.array([R.C_0 / 1.55, R.C_0 / 1.31])

    def coeffs(f):
        u = f / f0[0] - 1
        return u, 1.0 / f0[0]

    def n_of(f):  # quartic n(f) of two modes
        u, _ = coeffs(f)
        return np.stack([2.4 + 0.8 * u - 3.0 * u**2 + 5.0 * u**3 - 7.0 * u**4, 1.9 + 0.5 * u + 1.5 * u**2 - 2.0 * u**3 + 4.0 * u**4], axis=-1)

    def dn(f):
        u, s = coeffs(f)
        return np.stack([0.8 - 6.0 * u + 15.0 * u**2 - 28.0 * u**3, 0.5 + 3.0 * u - 6.0 * u**2 + 16.0 * u**3], axis=-1) * s

    def d2n(f):
        u, s = coeffs(f)
        return np.stack([-6.0 + 30.0 * u - 84.0 * u**2, 3.0 - 12.0 * u + 48.0 * u**2], axis=-1) * s**2

    def d3n(f):
        u, s = coeffs(f)
        return np.stack([30.0 - 168.0 * u, -12.0 + 96.0 * u], axis=-1) * s**3

    f = f0[:, None]  # (F, 1) against the (F, M) derivatives
    slope = plugin.dispersion_slope_of(f, dn(f0), d2n(f0), d3n(f0))
    b3 = plugin.beta3_of(f, d2n(f0), d3n(f0))
    assert np.allclose(slope, M3.dispersion_slope(f, dn(f0), d2n(f0), d3n(f0)), rtol=1e-14, atol=0)
    assert np.allclose(b3, M3.beta3(f, d2n(f0), d3n(f0)), rtol=1e-14, atol=0)

    # S = dD / d(wavelength): central difference of dispersion_of over the wavelength in nm
    wl = M3.C0_NM / f0  # nm

    def disp_at(wl_nm):
        ff = M3.C0_NM / wl_nm
        return plugin.dispersion_of(ff[:, None], dn(ff), d2n(ff))

    # beta3 = d^3 beta / d omega^3 with beta = omega n / c: third central difference in omega (converted to ps^3/km)
    w0 = 2 * np.pi * f0

    def beta_at(w):
        return w[:, None] * n_of(w / (2 * np.pi)) / M3.C0_M

    err_s, err_b = [], []
    for rel in (1e-3, 5e-4):
        h = rel * wl
        s_fd = (disp_at(wl + h) - disp_at(wl - h)) / (2 * h[:, None])
        hw = rel * w0
        b_fd = (beta_at(w0 + 2 * hw) - 2 * beta_at(w0 + hw) + 2 * beta_at(w0 - hw) - beta_at(w0 - 2 * hw)) / (2 * hw[:, None] ** 3) * 1e39
        err_s.append(np.abs(s_fd - slope).max() / np.abs(slope).max())
        err_b.append(np.abs(b_fd - b3).max() / np.abs(b3).max())
    # both differences are second order: halving the step divides the error by about 4
    assert err_s[0] <= 1e-4 and err_b[0] <= 1e-3, (err_s, err_b)
    assert err_s[1] < 0.35 * err_s[0] and err_b[1] < 0.35 * err_b[0], (err_s, err_b)
