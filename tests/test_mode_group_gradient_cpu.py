"""CPU: the float64 model of the group-index gradient (oracle/mode_group_gradient.py) against dense eigen-decompositions of the
assembled operator, on the first-order CPU cases plus a core with curved eps(f).

For every case w' must match a central difference of w(f) (v(f) under a fixed normalisation), the core-summed d_g lambda'
must match the mixed second difference of the eigenvalue in f and eps (Richardson-bounded), and the core-summed dng_deps must
match the central difference of ``mode_derivatives.n_group`` under eps +- delta on the core."""
import numpy as np
import pytest

from oracle import mode_derivatives as D
from oracle import mode_dispersion as MD
from oracle import mode_group_gradient as G
from oracle import restatement as R
from tests.test_mode_derivatives_cpu import F0, _operator
from tests.test_mode_dispersion_cpu import CASES2, _setup

COMPS = ((0, 0), (4, 1), (8, 2))  # (eps_cross component, map row)


def _pair_near(A, lam0):
    lam, V = np.linalg.eig(A)
    m = int(np.argmin(np.abs(lam - lam0)))
    return lam[m], V[:, m]


def _eps_at(c, f, comp=None, d=0.0):
    e = c["eps_at"](f)
    if comp is not None:
        e[comp] = e[comp] + d * c["core"]
    return e


def _model(c, v, lam):
    return G.group_gradient(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"],
                            eps_dfreq=c["deps_at"](F0) if c["disp"] else None)


@pytest.mark.parametrize("name", sorted(CASES2))
def test_w_prime_matches_central_difference(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    ell = np.conj(v)

    def w_of(f):
        st = R.setup(c["eps_at"](f), (c["x"], c["y"]), f, c["ms"], c["sym"], c["mu"])
        Q = R.assemble_diagonal(st)[1]
        _, vf = _pair_near(R.assemble_diagonal(st)[2].toarray(), lam)
        vf = vf * (ell @ v) / (ell @ vf)  # the normalisation ell^T v(f) = ell^T v(F0)
        return D.left_vector(st, Q, vf)

    def cd(h):
        return F0 * (w_of(F0 + h) - w_of(F0 - h)) / (2 * h)

    h = 1e-3 * F0
    fd = (4 * cd(h / 2) - cd(h)) / 3  # Richardson: the O(h^2) step error of the central difference cancels, O(h^4) is left
    st = R.setup(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], c["sym"], c["mu"])
    p1, _ = MD.material_directions(st, c["eps_at"](F0), F0, c["deps_at"](F0) if c["disp"] else None)
    Q = R.assemble_diagonal(st)[1]
    x = out["x"]
    vdot = x - v * (ell @ x) / (ell @ v)  # v' under that normalisation
    wp = G.w_prime(st, Q, G.q_prime(st, F0, p1), v, vdot)
    assert np.linalg.norm(wp - fd) <= 1e-8 * np.linalg.norm(fd), np.linalg.norm(wp - fd) / np.linalg.norm(fd)


def _fundamental(c):
    A = _operator(c, F0)
    lam, V = np.linalg.eig(A)
    m = int(np.argmin(lam.real))
    return lam[m], V[:, m]


@pytest.mark.parametrize("name", sorted(CASES2))
def test_mixed_derivative_matches_joint_second_difference(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    core = c["core"]
    for comp, a in COMPS:
        def mixed(h, d):
            ev = {}
            for sf in (1, -1):
                for se in (1, -1):
                    ev[sf, se] = _pair_near(_operator(c, F0 + sf * h, _eps_at(c, F0 + sf * h, comp, se * d)), lam)[0]
            return F0 * (ev[1, 1] - ev[1, -1] - ev[-1, 1] + ev[-1, -1]) / (4 * h * d)

        h, d = 2e-3 * F0, 2e-2
        f1, f2 = mixed(h, d), mixed(h / 2, d / 2)
        got = np.sum(out["d2lam_dfreq_deps"][a][core])
        bound = 2 * (4.0 / 3.0) * abs(f1 - f2) + 1e-8 * abs(f2)
        assert abs(got - f2) <= bound, (a, got, f2, bound)
        assert bound <= 1e-2 * abs(f2), (a, bound, f2)  # the check is not vacuous


@pytest.mark.parametrize("name", sorted(CASES2))
def test_group_index_gradient_matches_difference_of_n_group(name):
    c = _setup(name)
    lam, v = _fundamental(c)
    out = _model(c, v, lam)
    core = c["core"]
    de = c["deps_at"](F0) if c["disp"] else None
    for comp, a in COMPS:
        def ng_at(d):
            eps = _eps_at(c, F0, comp, d)
            lp, vp = _pair_near(_operator(c, F0, eps), lam)
            return D.derivatives(eps, (c["x"], c["y"]), F0, c["ms"], vp, lp, c["sym"], c["mu"], eps_dfreq=de)["n_group"]

        def fd(d):
            return (ng_at(d) - ng_at(-d)) / (2 * d)

        step = 1e-3 * 12.0
        f1, f2 = fd(step), fd(step / 2)
        got = np.sum(out["dng_deps"][a][core])
        bound = 2 * (4.0 / 3.0) * abs(f1 - f2) + 1e-8 * abs(f2)
        assert abs(got - f2) <= bound, (a, got, f2, bound)
        # and the first-order map is the mode_derivatives one
        ref = D.derivatives(c["eps_at"](F0), (c["x"], c["y"]), F0, c["ms"], v, lam, c["sym"], c["mu"], eps_dfreq=de)["dn_deps"]
        assert np.allclose(out["dn_deps"], ref, rtol=1e-12, atol=1e-14 * np.abs(ref).max())


def test_pec_cells_report_zero():
    c = _setup("pml")
    eps = c["eps_at"](F0)
    for comp in (0, 4, 8):
        eps[comp] = eps[comp].copy()
        eps[comp][0, 5] = R.PEC_VAL
    st = R.setup(eps, (c["x"], c["y"]), F0, c["ms"], c["sym"])
    lam, V = np.linalg.eig(R.assemble_diagonal(st)[2].toarray())
    m = int(np.argmin(lam.real))
    out = G.group_gradient(eps, (c["x"], c["y"]), F0, c["ms"], V[:, m], lam[m], c["sym"])
    assert (out["d2n_dfreq_deps"][:, 0, 5] == 0).all() and (out["dng_deps"][:, 0, 5] == 0).all()
    assert np.abs(out["d2n_dfreq_deps"]).max() > 0
