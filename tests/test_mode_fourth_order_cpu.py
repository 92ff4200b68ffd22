"""CPU: the float64 fourth-derivative model (oracle/mode_fourth_order.py) against dense eigen-decompositions of the assembled
operator, on the cases of the third-order CPU test plus a core with a quartic eps(f).

For every case the second-order correction x2 must solve its equation, the structural left correction w_hat2 must match a
Richardson-extrapolated second difference of w(f) = G J Q v(f) (v(f) normalised by w^T v(f) = w^T v), the model's f^4 d^4A/df^4
must match a Richardson-extrapolated fourth difference of the assembled operator, and d^4 lambda / df^4 must match the fourth
central difference of the tracked eigenvalue (steps f (1 +- h), f (1 +- 2h)) within twice the Richardson estimate of that
difference's step error.  lambda'''' must not depend on the multiples of v in x and x2 (with the matching multiple of x in x2) or
of w in w_hat and w_hat2.  ``plugin.beta4_of`` must be the step -> 0 limit of central differences of ``plugin.beta3_of`` over
omega."""
import numpy as np
import pytest

from oracle import mode_fourth_order as M4
from oracle import restatement as R
from tests.test_mode_derivatives_cpu import F0, _case, _fundamental, _operator
from tests.test_mode_third_order_cpu import CASES3

CASES4 = dict(CASES3)
CASES4["dispersive_quartic"] = dict(npml=(3, 2), sym=(0, 1))
EPS0 = 12.0
QUARTIC = (0.05, 0.2, 0.3, 0.8)  # eps(f) = eps0 (1 + a u + b u^2 + c u^3 + d u^4), u = f / F0 - 1


def _poly(c, coefs):
    """Core eps(f) = 12 (1 + sum_k coefs[k-1] u^k) with its analytic derivatives up to the fourth."""
    core = c["core"]
    a = np.r_[1.0, coefs]

    def comps(val):
        out = [np.zeros(core.shape, complex) for _ in range(9)]
        out[0], out[4], out[8] = val, val * 1.02, val * 0.97
        return out

    def deriv(k, bg):
        def at(f):
            u = f / F0 - 1
            val = sum(a[j] * np.prod(np.arange(j - k + 1, j + 1)) * u ** (j - k) for j in range(k, a.size)) / F0**k
            return comps(np.where(core, EPS0 * val, bg).astype(complex))

        return at

    c.update(eps_at=deriv(0, 2.07), deps_at=deriv(1, 0.0), d2eps_at=deriv(2, 0.0), d3eps_at=deriv(3, 0.0), d4eps_at=deriv(4, 0.0),
             disp=True)
    return c


def _setup(name):
    c = _case(**CASES4[name])
    if name == "dispersive_cubic":
        return _poly(c, (0.05, 0.2, 0.3))
    return _poly(c, QUARTIC) if name == "dispersive_quartic" else c


def _inputs(c):
    if not c["disp"]:
        return dict()
    out = dict(eps_dfreq=c["deps_at"](F0))
    if "d2eps_at" in c:
        out.update(eps_d2freq=c["d2eps_at"](F0), eps_d3freq=c["d3eps_at"](F0), eps_d4freq=c["d4eps_at"](F0))
    return out


def _model(c, v, lam, **kw):
    return M4.fourth_derivatives(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"], **_inputs(c), **kw)


def _fourth_difference(fn, h):
    """Scaled fourth central difference f^4 d^4/df^4 of fn(f) at F0 with relative step h: steps f (1 +- h), f (1 +- 2h)."""
    return (fn(F0 * (1 + 2 * h)) - 4 * fn(F0 * (1 + h)) + 6 * fn(F0) - 4 * fn(F0 * (1 - h)) + fn(F0 * (1 - 2 * h))) / h**4


@pytest.mark.parametrize("name", sorted(CASES4))
def test_second_order_corrections(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    A, x2, r2, w = out["A"], out["x2"], out["r2"], out["w"]
    res = np.linalg.norm(A @ x2 - lam * x2 - r2) / np.linalg.norm(r2)
    print(f"[fourth] {name}: |(A - lambda) x2 - r2| / |r2| = {res:.2e}")
    assert res <= 1e-12, res

    def w_at(f):  # w(f) = G J Q v(f) with v(f) normalised by w^T v(f) = w^T v
        st = R.setup(c["eps_at"](f), (c["x"], c["y"]), f, c["ms"], c["sym"], c["mu"])
        _, Q, Af = R.assemble_diagonal(st)
        ev, V = np.linalg.eig(Af.toarray())
        t = f / F0 - 1
        m = int(np.argmin(np.abs(ev - (lam + out["lam1"] * t + out["lam2"] * t * t / 2))))
        vf = V[:, m] * ((w @ v) / (w @ V[:, m]))
        from oracle import mode_derivatives as D

        return D.left_vector(st, Q, vf)

    d = [(w_at(F0 * (1 + h)) - 2 * w_at(F0) + w_at(F0 * (1 - h))) / h**2 for h in (2e-3, 1e-3)]
    rich = (4 * d[1] - d[0]) / 3
    scale = np.abs(rich).max()
    err = np.abs(2 * out["w_hat2"] - rich).max()
    bound = 2 * np.abs(d[0] - d[1]).max() / 3 + 1e-6 * scale
    print(f"[fourth] {name}: |2 w_hat2 - w''| {err:.2e}, bound {bound:.2e}")
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("name", sorted(CASES4))
def test_fourth_derivative_matches_dense_eigenvalues(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    l1, l2, l3, l4 = out["lam1"], out["lam2"], out["lam3"], out["lam4"]

    def lam_at(f):  # the eigenvalue tracked from its own Taylor prediction
        t = f / F0 - 1
        pred = lam + l1 * t + l2 * t * t / 2 + l3 * t**3 / 6 + l4 * t**4 / 24
        ev = np.linalg.eigvals(_operator(c, f))
        return ev[np.argmin(np.abs(ev - pred))]

    f1, f2 = _fourth_difference(lam_at, 4e-2), _fourth_difference(lam_at, 2e-2)
    want = f2
    bound = 2 * abs(f1 - f2) / 3 + 1e-6 * abs(want)
    print(f"[fourth] {name}: lambda'''' {l4:.8e}, fd {want:.8e}, |diff| {abs(l4 - want):.2e}, bound {bound:.2e}")
    assert abs(l4 - want) <= bound, (l4, want, bound)
    assert np.isclose(out["d4lam_dfreq4"], l4 / F0**4, rtol=1e-15, atol=0)
    if name == "dispersive_quartic":  # the fourth-order material terms matter here
        nd = _model(dict(c, disp=False), v, lam)
        assert abs(nd["lam4"] - want) > 10 * bound


@pytest.mark.parametrize("name", sorted(CASES4))
def test_fourth_operator_is_exact(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    A4 = _model(c, v, lam)["A4"].toarray()
    d = [_fourth_difference(lambda f: _operator(c, f), h) for h in (4e-2, 2e-2)]
    rich = (4 * d[1] - d[0]) / 3
    scale = np.abs(A4).max()
    err = np.abs(A4 - rich).max()
    bound = 2 * np.abs(d[0] - d[1]).max() / 3 + 1e-8 * scale
    assert err <= bound, (err, bound)
    assert scale > 0


@pytest.mark.parametrize("name", ["plain", "pml", "all", "mu_diag", "dispersive_quartic"])
def test_invariance_under_the_free_multiples(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    x, x2, w, wh, wh2 = out["x"], out["x2"], out["w"], out["w_hat"], out["w_hat2"]
    for alpha, beta in ((0.3 - 0.7j, 0.0), (2.0, -1.1 + 0.4j), (0.0, 0.5j)):
        moved = _model(c, v, lam, x=x + alpha * v, x2=x2 + alpha * x + beta * v)  # w_hat, w_hat2 formed from the moved x, x2
        given = _model(c, v, lam, x=x + alpha * v, x2=x2 + alpha * x + beta * v, w_hat=wh + alpha * w, w_hat2=wh2 + alpha * wh + beta * w)
        for m in (moved, given):
            assert abs(m["lam4"] - out["lam4"]) <= 1e-12 * abs(out["lam4"]), (alpha, beta, m["lam4"], out["lam4"])
        assert np.allclose(moved["w_hat2"], wh2 + alpha * wh + beta * w, rtol=0, atol=1e-12 * np.abs(wh2).max())


def test_beta4_is_the_limit_of_differences_of_beta3():
    from tidy3d_b200 import plugin

    f0 = np.array([R.C_0 / 1.55, R.C_0 / 1.31])
    cn = np.array([[2.4, 0.8, -3.0, 5.0, -7.0, 9.0], [1.9, 0.5, 1.5, -2.0, 4.0, -6.0]])  # quintic n(u) of two modes, u = f / f0[0] - 1

    def deriv(f, k):  # d^k n / df^k, shape (F, M)
        u = f / f0[0] - 1
        out = np.zeros((f.size, 2))
        for j in range(k, 6):
            out += np.outer(u ** (j - k), cn[:, j] * np.prod(np.arange(j - k + 1, j + 1)))
        return out / f0[0] ** k

    f = f0[:, None]
    b4 = plugin.beta4_of(f, deriv(f0, 3), deriv(f0, 4))
    assert np.allclose(b4, M4.beta4(f, deriv(f0, 3), deriv(f0, 4)), rtol=1e-14, atol=0)

    def b3_at(w):  # beta3 as a function of omega
        ff = w / (2 * np.pi)
        return plugin.beta3_of(ff[:, None], deriv(ff, 2), deriv(ff, 3))

    w0 = 2 * np.pi * f0
    errs = []
    for rel in (1e-3, 5e-4):
        hw = rel * w0
        fd = (b3_at(w0 + hw) - b3_at(w0 - hw)) / (2 * hw[:, None]) * 1e12  # ps^3/km per rad/s -> ps^4/km
        errs.append(np.abs(fd - b4).max() / np.abs(b4).max())
    # a central difference is second order: halving the step divides the error by about 4
    assert errs[0] <= 1e-4, errs
    assert errs[1] < 0.35 * errs[0], errs
