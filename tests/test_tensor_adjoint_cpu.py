"""CPU: the float64 model of the tensorial adjoint side (oracle/tensor_derivatives.py).

- the local pairing K satisfies K mat_d + mat_d^T K = 0 on every tensorial golden case and on non-uniform / PML / wall / bend
  variants, so -K (mat_d + sigma)^-1 K^-1 inverts mat_d^T - sigma (the transposed preconditioner of the device);
- left eigenvectors from the eigen-solve of mat^T at the forward shift have residual below 1e-10 and pair with the right ones;
- dn/df = w^T (d mat/df) u / w^T u matches a Richardson-extrapolated central difference of the eigenvalue within twice the
  Richardson estimate."""
import types

import numpy as np
import pytest
import scipy.sparse.linalg as spl

from oracle import restatement as R
from oracle import tensor_derivatives as T
from tests.golden import cases as G

F0 = R.C_0 / 1.55
GOLDEN = ["angled_64", "angled_48_minus", "angled_phi_48", "offdiag_48", "lossy_angled_40", "angle_bend_44"]


def _case(nx=12, ny=10, npml=(0, 0), sym=(0, 0), bend=None, nonuni=False, theta=0.25, phi=0.4, xz=0.0, xy=0.0, lossy=False):
    rng = np.random.default_rng(3)
    if nonuni:
        x = np.cumsum(np.r_[0, 0.12 + 0.08 * rng.random(nx)])
        y = np.cumsum(np.r_[0, 0.12 + 0.08 * rng.random(ny)])
    else:
        x, y = np.linspace(0, 0.16 * nx, nx + 1), np.linspace(0, 0.16 * ny, ny + 1)
    x, y = x - x.mean(), y - y.mean()
    xc, yc = 0.5 * (x[1:] + x[:-1]), 0.5 * (y[1:] + y[:-1])
    core = (np.abs(xc)[:, None] < 0.5) & (np.abs(yc)[None, :] < 0.3)
    e = np.where(core, 12.0 + (0.2j if lossy else 0), 2.07).astype(complex)
    eps = [np.zeros((nx, ny), complex) for _ in range(9)]
    eps[0], eps[4], eps[8] = e, e * 1.02, e * 0.97
    eps[2] = eps[6] = xz * e
    eps[1] = eps[3] = xy * e
    ms = types.SimpleNamespace(num_modes=2, target_neff=None, num_pml=npml, filter_pol=None, angle_theta=theta, angle_phi=phi,
                               precision="double", bend_radius=bend, bend_axis=1 if bend else None)
    return eps, [x, y], ms, sym


VARIANTS = {
    "angled": dict(),
    "angled_nonuniform": dict(nonuni=True),
    "angled_pml": dict(npml=(3, 2)),
    "angled_nonuniform_pml_pmc": dict(nonuni=True, npml=(3, 2), sym=(1, -1)),
    "angled_bend_pml_pec_pmc": dict(bend=4.0, npml=(3, 2), sym=(-1, 1)),
    "angled_lossy": dict(lossy=True, npml=(2, 2)),
    "offdiag_xz_pml": dict(theta=0.0, xz=0.1, npml=(3, 2)),
    "offdiag_xy_bend_pml": dict(theta=0.0, xy=0.1, bend=4.0, npml=(3, 2)),
}


def _golden_st(name):
    fac, kw, _ = G.CASES[name]
    wl = fac()
    kw = G.resolve_kwargs(wl, kw)
    return R.setup(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))


def _pairing_residual(st):
    Md, K = T.diagonal_part(st), T.pairing(st)
    return abs(K @ Md + Md.T @ K).max() / (abs(K).max() * abs(Md).max())


@pytest.mark.parametrize("name", GOLDEN)
def test_pairing_on_golden_cases(name):
    st = _golden_st(name)
    assert st["tensorial"]
    assert _pairing_residual(st) <= 1e-12


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_pairing_inverts_the_transposed_diagonal_part(name):
    eps, coords, ms, sym = _case(**VARIANTS[name])
    st = R.setup(eps, coords, F0, ms, sym)
    assert st["tensorial"]
    assert _pairing_residual(st) <= 1e-12
    n4 = 4 * st["n"]
    Md, K, I = -1j * T.diagonal_part(st), T.pairing(st).tocsc(), T.sp.identity(n4)
    sig = st["target"]
    x = np.random.default_rng(1).standard_normal(n4) + 0j
    v = (Md.T - sig * I) @ x
    z = -(K @ spl.spsolve((Md + sig * I).tocsc(), spl.spsolve(K, v)))
    assert np.linalg.norm(z - x) <= 1e-8 * np.linalg.norm(x)


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_left_eigenvectors_and_group_index(name):
    eps, coords, ms, sym = _case(**VARIANTS[name])
    st = R.setup(eps, coords, F0, ms, sym)
    n, u, nl, w = T.eigenpairs(st, 2)
    mat = T.operator(st)
    for q in range(2):
        assert abs(nl[q] - n[q]) <= 1e-10 * abs(n[q])
        assert np.linalg.norm(mat.T @ w[:, q] - nl[q] * w[:, q]) <= 1e-10 * abs(nl[q]) * np.linalg.norm(w[:, q])
        assert abs(w[:, q] @ u[:, q]) >= 1e-8 * np.linalg.norm(w[:, q]) * np.linalg.norm(u[:, q])
    dn = T.dn_dfreq(st, F0, u[:, 0], w[:, 0]) * F0

    def ev(f):
        s = R.setup(eps, coords, f, ms, sym)
        return T.eigenpairs(s, 1, sigma=n[0])[0][0]

    h = 2e-3
    d1 = (ev(F0 * (1 + h)) - ev(F0 * (1 - h))) / (2 * h)
    d2 = (ev(F0 * (1 + 2 * h)) - ev(F0 * (1 - 2 * h))) / (4 * h)
    rich = (4 * d1 - d2) / 3
    assert abs(dn - rich) <= max(2 * abs(rich - d1), 1e-9 * abs(dn)), (dn, rich, d1)


def _core_region(coords):
    xc = 0.5 * (coords[0][1:] + coords[0][:-1])
    yc = 0.5 * (coords[1][1:] + coords[1][:-1])
    return (np.abs(xc)[:, None] < 0.4) & (np.abs(yc)[None, :] < 0.25)


@pytest.mark.parametrize("name", ["angled_nonuniform_pml_pmc", "angled_bend_pml_pec_pmc", "offdiag_xz_pml", "offdiag_xy_bend_pml"])
def test_permittivity_gradient_against_region_differences(name):
    """For each of the nine eps_cross components, the core-region sum of the gradient against the Richardson-extrapolated central
    difference of the eigenvalue under that region's perturbation, within twice the Richardson estimate."""
    eps, coords, ms, sym = _case(**VARIANTS[name])
    st = R.setup(eps, coords, F0, ms, sym)
    n, u, _, w = T.eigenpairs(st, 1)
    g = T.dn_deps_tensor(eps, coords, F0, ms, u[:, 0], w[:, 0], sym)
    reg = _core_region(coords)
    for k in range(9):
        def ev(d):
            e2 = [a.copy() for a in eps]
            e2[k] = e2[k] + d * reg
            return T.eigenpairs(R.setup(e2, coords, F0, ms, sym), 1, sigma=n[0])[0][0]

        h = 1e-3
        d1 = (ev(h) - ev(-h)) / (2 * h)
        d2 = (ev(2 * h) - ev(-2 * h)) / (4 * h)
        rich = (4 * d1 - d2) / 3
        assert abs(g[k][reg].sum() - rich) <= max(2 * abs(rich - d1), 1e-9 * abs(rich)), (k, g[k][reg].sum(), rich, d1)


def test_direction_minus_and_nine_component_dispersion():
    """Lossy angled section solved with direction "-" (mat = -(-i) M) and an eps(f) that moves all nine components: dn/df of
    ``derivatives`` with eps_dfreq against the Richardson-extrapolated difference of the eigenvalue of the f-dependent problem."""
    eps0, coords, ms, sym = _case(lossy=True, npml=(2, 2), xz=0.05, xy=0.03)
    slope = [np.where(np.abs(e) > 0, (0.3 + 0.1 * k) * e / F0, 0) for k, e in enumerate(eps0)]

    def eps_at(f):
        return [e + s * (f - F0) for e, s in zip(eps0, slope)]

    st = R.setup(eps0, coords, F0, ms, sym)
    n, u, _, w = T.eigenpairs(st, 1, msign=-1.0)
    out = T.derivatives(eps0, coords, F0, ms, u[:, 0], w[:, 0], sym, eps_dfreq=slope, msign=-1.0)
    assert abs(out["n"] - n[0] * st["knorm"]) <= 1e-10 * abs(n[0])

    def ev(f):
        return T.eigenpairs(R.setup(eps_at(f), coords, f, ms, sym), 1, sigma=n[0], msign=-1.0)[0][0] * st["knorm"]

    h = 2e-3
    d1 = (ev(F0 * (1 + h)) - ev(F0 * (1 - h))) / (2 * h)
    d2 = (ev(F0 * (1 + 2 * h)) - ev(F0 * (1 - 2 * h))) / (4 * h)
    rich = (4 * d1 - d2) / 3
    dn = out["dn_dfreq"] * F0
    assert abs(dn - rich) <= max(2 * abs(rich - d1), 1e-9 * abs(dn)), (dn, rich, d1)
    without = T.dn_dfreq(st, F0, u[:, 0], w[:, 0], -1.0) * st["knorm"] * F0
    assert abs(without - dn) > 20 * abs(rich - d1)  # the material terms matter at this bound


@pytest.mark.parametrize("name", ["angled", "offdiag_xz_pml"])
def test_reciprocal_cases_pair_with_the_backward_mode(name):
    """On a uniform grid without z-coupled PML the left eigenvector is the pairing of the backward mode: w || K u(-n)."""
    kw = dict(VARIANTS[name])
    kw.pop("npml", None)
    eps, coords, ms, sym = _case(**kw)
    st = R.setup(eps, coords, F0, ms, sym)
    n, _, _, w = T.eigenpairs(st, 1)
    _, ub = spl.eigs(T.operator(st).tocsc(), k=1, sigma=-n[0], tol=1e-13)
    c = T.pairing(st) @ ub[:, 0]
    cos = abs(np.vdot(c, w[:, 0])) / (np.linalg.norm(c) * np.linalg.norm(w[:, 0]))
    assert abs(cos - 1) <= 1e-10


def test_small_off_diagonal_agrees_with_the_diagonal_model():
    """With 1e-4 off-diagonal eps (tensorial path) the xx / yy / zz rows of the gradient and dn/df agree with
    oracle/mode_derivatives on the diagonal problem to O(1e-4)."""
    from oracle import mode_derivatives as MD

    eps_t, coords, ms, sym = _case(theta=0.0, xz=1e-4, xy=1e-4, npml=(3, 2))
    eps_d, _, _, _ = _case(theta=0.0, npml=(3, 2))
    st_t = R.setup(eps_t, coords, F0, ms, sym)
    st_d = R.setup(eps_d, coords, F0, ms, sym)
    assert st_t["tensorial"] and not st_d["tensorial"]
    n, u, _, w = T.eigenpairs(st_t, 1)
    out = T.derivatives(eps_t, coords, F0, ms, u[:, 0], w[:, 0], sym)
    lam, v = spl.eigs(R.assemble_diagonal(st_d)[2].tocsc(), k=1, sigma=-(n[0] ** 2), tol=1e-13)
    ref = MD.derivatives(eps_d, coords, F0, ms, v[:, 0], lam[0], sym)
    assert abs(out["n"] - np.sqrt(-lam[0] + 0j) * st_d["knorm"]) <= 1e-4 * abs(out["n"])
    assert abs(out["dn_dfreq"] - ref["dn_dfreq"]) <= 1e-4 * abs(ref["dn_dfreq"])
    scale = np.abs(ref["dn_deps"]).max()
    for row, k in enumerate((0, 4, 8)):
        assert np.abs(out["dn_deps_tensor"][k] - ref["dn_deps"][row]).max() <= 1e-3 * scale, k
