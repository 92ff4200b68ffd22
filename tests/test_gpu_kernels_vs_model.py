"""GPU: every kernel on the preconditioner path against the float64 model oracle/mg_model.py, per level and per batch position.

The eigen-iteration converges to the right eigenpairs whatever the preconditioner does, so the parity tests cannot see a
wrong restriction weight, a coarse coefficient field averaged wrongly or a fused tail reading another problem's
coefficients -- only a slower solve.  Here each piece is compared with the model of the same operation:

a. the fp64 Krylov-side operator on level 0 (apply, residual) against the reference's assembled matrix, 1e-12;
b. the multigrid operator of every level (apply, residual, stored-diagonal sweep, omega D^-1, the fused first two sweeps):
   fp64 multigrid (mg_precision = 0) to 1e-12, and the fp32 kernel families (TMA pair, one-column, tiled) to FP32_OP_TOL;
c. one V-cycle (fused coarse tail on and off; coarse GMRES for indefinite shifts, Jacobi otherwise): fp64 to 1e-10, fp32 to
   FP32_VCYCLE_TOL;
d. the inner solve: its true residual, computed here from the assembled matrix, is within the handle's inner_tol and agrees
   with the residual the solver reports (with and without fp32 iterative refinement);
e. the same through b200ms_debug_batch on batches built as production builds them (a shared-medium frequency sweep,
   distinct cross-sections, 64 problems): every problem matches the model of that problem and the one-problem hook.

Operator errors are scaled by max(|A| |x|) (row-wise absolute product), not by max|y|, so that cancellation hides nothing."""
import ctypes as C

import numpy as np
import pytest

from oracle import mg_model as M
from oracle import restatement as R
from tests import mg_cases
from tidy3d_b200 import _cabi
from tidy3d_b200 import workloads as W

pytestmark = pytest.mark.gpu

DIAG_CASES = ["c1_64", "c1_64_sym_pmc_pec", "nonuniform_56", "c3_96", "c4_96", "c4_96_axis0", "lossy_48", "mu_cross_40",
              "pec_block_40_mu", "slab1d_x1", "slab1d_y1", "strip_75x131", "strip_256"]
TENSOR_CASES = ["angled_48_minus", "lossy_angled_40"]
# ten times the largest fp32-vs-model errors measured on an H100 80GB HBM3 over the whole case matrix (single problems and
# batches, all three kernel families): 2.65e-7 for the level operators (omega D^-1 on a batch level), 2.63e-6 for a V-cycle.
# fp64 measured 7.0e-16 (levels) and 3.9e-15 (V-cycle).
FP32_OP_TOL = 3e-6
FP32_VCYCLE_TOL = 3e-5
OBSERVED = {}


def _vec(rng, shape, real):
    v = rng.standard_normal(shape)
    return v + 0j if real else v + 1j * rng.standard_normal(shape)


def batch(h, pks, what, x, rhs=None, level=0, mode=0):
    """b200ms_debug_batch on the problems pks; x / rhs / result: (nprob, ...) complex arrays."""
    n = len(pks)
    probs = (_cabi.Problem * n)(*[p.struct for p in pks])
    xa = np.ascontiguousarray(x, dtype=complex)
    ra = None if rhs is None else np.ascontiguousarray(rhs, dtype=complex)
    out = np.zeros_like(xa)
    it, rr = C.c_int(), np.zeros(n)
    rc = _cabi.lib().b200ms_debug_batch(h._h, n, probs, what, level, mode, _cabi._ptr(xa.view(float)), None if ra is None else _cabi._ptr(ra.view(float)),
                                        _cabi._ptr(out.view(float)), C.byref(it), _cabi._ptr(rr))
    assert rc == 0, (rc, h.last_error())
    return out, it.value, rr


def walls(prob, v):
    """Zero the PEC-wall rows and the removed PEC unknowns (a preconditioner input never has them)."""
    v = prob.mask(v.copy())
    pmc = prob.st["pmc"]
    if not pmc[1] and prob.ny > 1:
        v[0][:, 0] = 0
    if not pmc[0] and prob.nx > 1:
        v[1][0, :] = 0
    return v


def rel_err(y, ref, scale):
    """max|y - ref| / max(scale); infinite when y holds a NaN or an infinity (max() would pass a NaN over)."""
    scale = float(np.max(scale))
    assert np.isfinite(scale) and scale > 0
    d = float(np.abs(y - ref).max())
    return d / scale if np.isfinite(d) else np.inf


@pytest.fixture(scope="module")
def handles(built_lib):
    hs = {"fp64": _cabi.Handle(mg_precision=0), "fp64_unfused": _cabi.Handle(mg_precision=0, mg_fused_tail=0),
          "fp32": _cabi.Handle(), "fp32_unfused": _cabi.Handle(mg_fused_tail=0),
          "fp32_onecol": _cabi.Handle(stencil_pair=0), "fp32_tiled": _cabi.Handle(stencil_variant=1),
          "ir0": _cabi.Handle(inner_ir=0)}
    yield hs
    for h in hs.values():
        h.close()
    if OBSERVED:
        print("\nlargest scaled errors:", {k: f"{v:.2e}" for k, v in sorted(OBSERVED.items())})


def _observe(key, err):
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), err)
    return err


# ---- a. the fp64 operator on level 0 -------------------------------------------------------------------------------------
def assembled(prob, wl, kw):
    """(A - sigma) as the reference assembles it: diagonal path (with the incidence formulation's zeroed 1/ezz and removed
    unknowns), or msign (-i) M of the tensorial path (solver.py:655-670)."""
    st = prob.st
    n = 2 * prob.nx * prob.ny
    if prob.tensorial:
        ms = -1.0 if (kw.get("direction") == "-" and R._is_complex(st["eps"])) else 1.0
        A = (ms * -1j) * R.assemble_tensorial(st)
        return (A - st["target"] * R.sp.identity(2 * n)).tocsr(), None
    if prob.masked:
        st = dict(st)
        st["eps"] = st["eps"].copy()
        st["eps"][2, 2][prob.pec[2].ravel()] = np.inf
    A = (R.assemble_diagonal(st)[2] - prob.sigma * R.sp.identity(n)).tocsr()
    keep = ~np.concatenate((prob.pec[0].ravel(), prob.pec[1].ravel())) if prob.masked else None
    return A, keep


@pytest.mark.parametrize("name", DIAG_CASES + TENSOR_CASES)
def test_fp64_operator_matches_the_assembled_matrix(handles, name):
    wl, kw = mg_cases.case(name)
    pk, prob = mg_cases.packed(_cabi, wl, kw), mg_cases.model_problem(wl, kw)
    A, keep = assembled(prob, wl, kw)
    rng = np.random.default_rng(11)
    real = mg_cases.is_real(wl, kw)
    x, rhs = _vec(rng, A.shape[0], real), _vec(rng, A.shape[0], real)
    if keep is not None:
        x[~keep] = 0
        rhs[~keep] = 0
    ax = A @ x
    scale = abs(A) @ np.abs(x) + np.abs(rhs)
    y = batch(handles["fp64"], [pk], 0, x[None], rhs[None], 0, 0)[0][0]
    r = batch(handles["fp64"], [pk], 0, x[None], rhs[None], 0, 1)[0][0]
    if keep is not None:
        ax[~keep] = 0
        assert (y[~keep] == 0).all() and (r[~keep] == 0).all()
    assert rel_err(y, ax, scale) <= 1e-12
    assert rel_err(r, np.where(keep, rhs - ax, 0) if keep is not None else rhs - ax, scale) <= 1e-12


# ---- b. multigrid operators of every level -------------------------------------------------------------------------------
def level_ops(h, pks, levels, rng, real, key, d0=True):
    """Run apply / residual / sweep / omega D^-1 / two sweeps from zero of every level on the batch pks and return the largest
    scaled error against the model levels (levels[b][l] for problem b)."""
    worst = 0.0
    nb = len(pks)
    for l in range(len(levels[0])):
        lvs = [lv[l] for lv in levels]
        shp = (2, lvs[0].nx, lvs[0].ny)
        x = np.stack([_vec(rng, shp, real) for _ in range(nb)])
        rhs = np.stack([_vec(rng, shp, real) for _ in range(nb)])
        modes = [0, 1, 2, 3]
        if d0 and lvs[0].nx >= 32 and lvs[0].ny >= 2:
            modes.append(4)  # the fused first sweeps run where production runs them
        for mode in modes:
            y = batch(h, pks, 0, x, rhs, l, mode + (16 if l == 0 else 0))[0]
            for b, lv in enumerate(lvs):
                ax = lv.abs_apply(x[b])
                if mode == 0:
                    ref, sc = lv.apply(x[b]), ax
                elif mode == 1:
                    ref, sc = rhs[b] - lv.apply(x[b]), np.abs(rhs[b]) + ax
                elif mode == 2:
                    ref, sc = lv.sweep(x[b], rhs[b]), np.abs(x[b]) + np.abs(lv.dinv) * (np.abs(rhs[b]) + ax)
                elif mode == 3:
                    ref, sc = lv.jacobi0(rhs[b]), np.abs(lv.dinv * rhs[b])
                else:
                    x1 = lv.jacobi0(rhs[b])
                    ref, sc = lv.two_sweeps_from_zero(rhs[b]), np.abs(x1) + np.abs(lv.dinv) * (np.abs(rhs[b]) + lv.abs_apply(x1))
                e = rel_err(y[b], ref, sc)
                worst = max(worst, e)
                _observe(f"{key} mode {mode}", e)
    return worst


@pytest.mark.parametrize("name", DIAG_CASES)
def test_multigrid_levels_fp64(handles, name):
    wl, kw = mg_cases.case(name)
    pk, prob = mg_cases.packed(_cabi, wl, kw), mg_cases.model_problem(wl, kw)
    mg = M.Multigrid(prob, M.Opts(handles["fp64"].options))
    assert level_ops(handles["fp64"], [pk], [mg.levels], np.random.default_rng(5), mg_cases.is_real(wl, kw), "fp64 levels") <= 1e-12


@pytest.mark.parametrize("name", DIAG_CASES)
@pytest.mark.parametrize("family", ["fp32", "fp32_onecol", "fp32_tiled"])
def test_multigrid_levels_fp32(handles, name, family):
    """fp32 kernels (TMA pair kernel by default, stencil_pair = 0: one-column kernel, stencil_variant = 1: tiled kernel)."""
    wl, kw = mg_cases.case(name)
    pk, prob = mg_cases.packed(_cabi, wl, kw), mg_cases.model_problem(wl, kw)
    h = handles[family]
    mg = M.Multigrid(prob, M.Opts(h.options))
    err = level_ops(h, [pk], [mg.levels], np.random.default_rng(5), mg_cases.is_real(wl, kw), "fp32 levels", d0=family != "fp32_tiled")
    assert err <= FP32_OP_TOL, (family, err)


# ---- c. the V-cycle ------------------------------------------------------------------------------------------------------
VCYCLE_CASES = ["c1_64", "c1_64_sym_pmc_pec", "nonuniform_56", "c3_96", "c4_96", "lossy_48", "mu_cross_40", "pec_block_40_mu",
                "slab1d_x1", "slab1d_y1", "strip_75x131", "strip_256"]


def vcycle_errors(h, pks, mgs, rng, real):
    rs = np.stack([walls(mg.prob, _vec(rng, (2, mg.prob.nx, mg.prob.ny), real)) for mg in mgs])
    z = batch(h, pks, 1, rs.reshape(len(pks), -1))[0].reshape(rs.shape)
    errs = []
    for b, mg in enumerate(mgs):
        ref = mg.precondition(rs[b])
        errs.append(rel_err(z[b], ref, np.abs(ref)))
    return z, errs


@pytest.mark.parametrize("name", VCYCLE_CASES)
@pytest.mark.parametrize("prec", ["fp64", "fp32"])
@pytest.mark.parametrize("fused", [True, False])
def test_vcycle_matches_the_model(handles, name, prec, fused):
    wl, kw = mg_cases.case(name)
    pk, prob = mg_cases.packed(_cabi, wl, kw), mg_cases.model_problem(wl, kw)
    h = handles[prec + ("" if fused else "_unfused")]
    mg = M.Multigrid(prob, M.Opts(h.options))
    if name in ("c3_96", "c4_96", "nonuniform_56", "pec_block_40_mu", "slab1d_x1"):
        assert mg.coarse_krylov  # indefinite shift: coarse GMRES(kc), no fused tail
    if name in ("c1_64", "lossy_48", "strip_256", "strip_75x131"):
        assert not mg.coarse_krylov  # Jacobi on the coarsest level, fused tail where it fits
    err = vcycle_errors(h, [pk], [mg], np.random.default_rng(9), mg_cases.is_real(wl, kw))[1][0]
    _observe(f"{prec} vcycle", err)
    assert err <= (1e-10 if prec == "fp64" else FP32_VCYCLE_TOL), err


# ---- d. the inner solve ---------------------------------------------------------------------------------------------------
SOLVE_CASES = ["c1_64", "c3_96", "lossy_48", "pec_block_40_mu", "angled_48_minus"]


def check_solve(h, pks, probs, wls, kws, rng):
    tol = h.options.inner_tol
    bs, As, keeps = [], [], []
    for prob, wl, kw in zip(probs, wls, kws):
        A, keep = assembled(prob, wl, kw)
        b = _vec(rng, A.shape[0], mg_cases.is_real(wl, kw))
        if keep is not None:
            b[~keep] = 0
        bs.append(b)
        As.append(A)
        keeps.append(keep)
    x, iters, est = batch(h, pks, 2, np.stack(bs))
    assert iters > 0
    for q, (A, b, keep) in enumerate(zip(As, bs, keeps)):
        r = b - A @ x[q]
        if keep is not None:  # removed PEC unknowns: not in the system, zero in the solution
            assert (x[q][~keep] == 0).all()
            r[~keep] = 0
        true = np.linalg.norm(r) / np.linalg.norm(b)
        _observe("solve true/tol", true / tol)
        assert true <= 1.25 * tol, (q, true, est[q])
        o = h.options
        if o.mg_precision == 0 or o.inner_ir == 0 or probs[q].masked or probs[q].tensorial:
            # fp64 cycles only (BatchSolver::solve_op, fgmres): the reported residual is the Givens estimate or the fp64
            # residual, both the true residual up to rounding
            _observe("solve fp64 |true - est| / true", abs(true - est[q]) / true)
            assert abs(true - est[q]) <= 1e-3 * true, (q, true, est[q])
        else:
            # fp32 refinement: the reported residual is the fp64 residual of the refinement or, when the refinement trusts
            # its last fp32 cycle (cycle tolerance >= ir_trust), that cycle's estimate, good to ~1e-5 of its starting residual
            assert abs(true - est[q]) <= 0.25 * max(true, est[q]) + 0.2 * tol, (q, true, est[q])


@pytest.mark.parametrize("name", SOLVE_CASES)
@pytest.mark.parametrize("ir", [1, 0])
def test_inner_solve_reaches_and_reports_inner_tol(handles, name, ir):
    wl, kw = mg_cases.case(name)
    check_solve(handles["fp32" if ir else "ir0"], [mg_cases.packed(_cabi, wl, kw)], [mg_cases.model_problem(wl, kw)], [wl], [kw],
                np.random.default_rng(4))


# ---- e. batches as production builds them ---------------------------------------------------------------------------------
def _sweep_batch(name, freqs):
    wl, kw = mg_cases.case(name)
    eps = np.ascontiguousarray(np.stack([np.asarray(e, complex) for e in wl.eps_cross]))  # one medium: shared fields
    pks = [mg_cases.packed(_cabi, wl, kw, freq=f, eps=eps) for f in freqs]
    # the library shares a medium between problems that point at the same eps / mu / coordinate arrays
    addr = lambda p: [C.cast(getattr(p.struct, f), C.c_void_p).value for f in ("eps", "mu", "coords_x", "coords_y")]  # noqa: E731
    assert all(addr(p) == addr(pks[0]) for p in pks)
    probs = [mg_cases.model_problem(wl, kw, freq=f) for f in freqs]
    return pks, probs, [wl] * len(freqs), [kw] * len(freqs)


def _planes_batch():
    wls = W.c5_planes(n_planes=3, n=96, nf=1)
    pks = [mg_cases.packed(_cabi, wl, {}) for wl in wls]
    return pks, [mg_cases.model_problem(wl, {}) for wl in wls], wls, [{}] * 3


BATCHES = {
    "c3_96_sweep4": lambda: _sweep_batch("c3_96", W.C_0 / np.linspace(1.5, 1.6, 4)),
    "c5_planes3": _planes_batch,
    "strip_64_x64": lambda: _sweep_batch("c1_64", W.sweep_freqs(64)),  # the production batch size; distinct k0 per problem
}


@pytest.mark.parametrize("bname", list(BATCHES))
def test_production_batches_match_model_and_single_problem(handles, bname):
    pks, probs, wls, kws = BATCHES[bname]()
    real = mg_cases.is_real(wls[0], kws[0])
    nb = len(pks)
    rng = np.random.default_rng(21)
    # a. fp64 operator of every problem
    n = 2 * probs[0].nx * probs[0].ny
    x = np.stack([_vec(rng, n, real) for _ in range(nb)])
    y = batch(handles["fp64"], pks, 0, x, None, 0, 0)[0]
    for q in range(nb):
        A, _ = assembled(probs[q], wls[q], kws[q])
        assert rel_err(y[q], A @ x[q], abs(A) @ np.abs(x[q])) <= 1e-12, q
        if q in (0, nb - 1):
            y1 = batch(handles["fp64"], [pks[q]], 0, x[q][None], None, 0, 0)[0][0]
            assert np.abs(y1 - y[q]).max() <= 1e-13 * np.abs(y[q]).max(), q
    # the device plans the batch's hierarchy from problem 0 and limits it by the largest k of the batch
    kmax = np.sqrt(max(p.max_k2 for p in probs))
    for prec, tol_op, tol_vc, tol_single in (("fp64", 1e-12, 1e-10, 1e-13), ("fp32", FP32_OP_TOL, FP32_VCYCLE_TOL, 2e-6)):
        h = handles[prec]
        mg0 = M.Multigrid(probs[0], M.Opts(h.options), kmax=kmax)
        mgs = [M.Multigrid(p, M.Opts(h.options), plan=mg0.plan, kmax=kmax) for p in probs]
        # b. every level of every problem
        assert level_ops(h, pks, [mg.levels for mg in mgs], np.random.default_rng(5), real, f"{prec} batch levels") <= tol_op
        # c. V-cycle: each problem against its model and against the one-problem hook
        z, errs = vcycle_errors(h, pks, mgs, np.random.default_rng(9), real)
        assert max(errs) <= tol_vc, errs
        rs = np.stack([walls(mg.prob, _vec(np.random.default_rng(9 + q), (2, mg.prob.nx, mg.prob.ny), real)) for q, mg in enumerate(mgs)])
        zb = batch(h, pks, 1, rs.reshape(nb, -1))[0]
        for q in sorted({0, 1, nb - 1}):
            single = M.Multigrid(probs[q], M.Opts(h.options))
            if single.coarse_krylov != mg0.coarse_krylov or [a.tolist() for ag in single.plan for a in ag] != [a.tolist() for ag in mg0.plan for a in ag]:
                continue  # this problem alone would get another hierarchy: the one-problem hook runs a different V-cycle
            z1 = batch(h, [pks[q]], 1, rs[q].reshape(1, -1))[0][0]
            assert np.abs(z1 - zb[q]).max() <= tol_single * np.abs(zb[q]).max(), (prec, q)
    # d. inner solve of the whole batch
    check_solve(handles["fp32"], pks, probs, wls, kws, np.random.default_rng(4))


@pytest.mark.parametrize("differs", ["shape", "direction", "num_modes"])
def test_debug_batch_rejects_problems_production_would_not_batch(handles, differs):
    """b200ms_solve_batch puts problems of another shape, direction or mode count in another device batch."""
    wl, kw = mg_cases.case("c1_64")
    wl2, kw2 = mg_cases.case({"shape": "lossy_48", "direction": "c1_64_minus", "num_modes": "c1_64"}[differs])
    if differs == "num_modes":
        wl2.mode_spec.num_modes = 4
    pks = [mg_cases.packed(_cabi, wl, kw), mg_cases.packed(_cabi, wl2, kw2)]
    probs = (_cabi.Problem * 2)(*[p.struct for p in pks])
    x = np.zeros(2 * 2 * 64 * 64, complex)
    rc = _cabi.lib().b200ms_debug_batch(handles["fp64"]._h, 2, probs, 0, 0, 0, _cabi._ptr(x.view(float)), None, _cabi._ptr(x.view(float)), None, None)
    assert rc == _cabi.ERR_ARG and "differs from problem 0" in handles["fp64"].last_error()
