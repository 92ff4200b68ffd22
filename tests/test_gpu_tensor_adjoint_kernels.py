"""GPU: the transposed operator and the transposed preconditioner of the tensorial path against the float64 model
oracle/tensor_derivatives.py.

An eigen-solve with mat^T (the left eigenvectors that first-order perturbation theory needs) runs the tensorial Krylov machinery
with two pieces swapped in: tensor_apply_kernel<C, true>, and the block preconditioner wrapped in the local pairing K,
(mat_d^T - sigma)^-1 = -K (mat_d + sigma)^-1 K^-1.  Both are reached through b200ms_debug_batch (what 3 / 4):

a. (mat^T - sigma) x and rhs - (mat^T - sigma) x against the assembled matrix, to 1e-12 scaled by the absolute products,
   for single problems and for a two-frequency batch (per-problem coefficients);
b. the transposed preconditioner against exact sparse solves with mat_d^T - sigma, on a handle whose multigrid is iterated
   to convergence, next to the forward preconditioner against mat_d - sigma on the same handle: a wrong pairing, metric or
   shift sign leaves an O(1) error where the forward one converged.  Without PML the forward one is exact (1e-6); with PML
   the multigrid inverts its phase-limited operator, and the transposed error must stay within ten times the forward one."""
import numpy as np
import pytest

from oracle import restatement as R
from oracle import tensor_derivatives as T
from tests import mg_cases
from tests.golden import cases as G
from tests.test_gpu_kernels_vs_model import _vec, batch, rel_err
from tidy3d_b200 import _cabi
from tidy3d_b200 import workloads as W

pytestmark = pytest.mark.gpu

CASES = ["angled_48_minus", "lossy_angled_40", "lossy_angled_40_minus", "angle_bend_44", "offdiag_48", "angled_nonuniform_pml"]
OBSERVED = {}


def _angled_nonuniform_pml():
    """Angled strip on a graded grid with PML: the case where reciprocity does not give the left eigenvector."""
    wl = G._nonuniform(48)
    wl.mode_spec = W.ModeSpecLike(num_modes=3, angle_theta=0.25, angle_phi=0.4, num_pml=(6, 6), target_neff=2.2)
    wl.name = "angled_nonuniform_pml"
    return wl, {}


def _case(name):
    return _angled_nonuniform_pml() if name == "angled_nonuniform_pml" else mg_cases.case(name)


def _msign(prob, kw):
    return -1.0 if (kw.get("direction") == "-" and R._is_complex(prob.st["eps"])) else 1.0


@pytest.fixture(scope="module")
def handles(built_lib):
    hs = {"fp64": _cabi.Handle(mg_precision=0), "converged": _cabi.Handle(mg_precision=0, tensor_mg_cycles=40)}
    yield hs
    for h in hs.values():
        h.close()
    if OBSERVED:
        print("\nlargest scaled errors:", {k: f"{v:.2e}" for k, v in sorted(OBSERVED.items())})


def _observe(key, err):
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), err)
    return err


def _check_transposed_apply(h, pks, probs, kws, key):
    rng = np.random.default_rng(5)
    mats = [(T.operator(p.st, _msign(p, kw)) - p.st["target"] * T.sp.identity(4 * p.nx * p.ny)).T.tocsr() for p, kw in zip(probs, kws)]
    x = np.stack([_vec(rng, A.shape[0], False) for A in mats])
    rhs = np.stack([_vec(rng, A.shape[0], False) for A in mats])
    y = batch(h, pks, 3, x, rhs, 0, 0)[0]
    r = batch(h, pks, 3, x, rhs, 0, 1)[0]
    for q, A in enumerate(mats):
        scale = abs(A) @ np.abs(x[q]) + np.abs(rhs[q])
        assert _observe(key, rel_err(y[q], A @ x[q], scale)) <= 1e-12, (key, q)
        assert _observe(key, rel_err(r[q], rhs[q] - A @ x[q], scale)) <= 1e-12, (key, q)


@pytest.mark.parametrize("name", CASES)
def test_transposed_operator_matches_the_assembled_matrix(handles, name):
    wl, kw = _case(name)
    pk, prob = mg_cases.packed(_cabi, wl, kw), mg_cases.model_problem(wl, kw)
    assert prob.tensorial
    _check_transposed_apply(handles["fp64"], [pk], [prob], [kw], f"apply_T {name}")


def test_transposed_operator_per_batch_position(handles):
    """Two frequencies of one section in one device batch: each position uses its own coefficients and shift."""
    wl, kw = _case("angled_nonuniform_pml")
    freqs = [wl.freqs[0], 1.07 * wl.freqs[0]]
    pks = [mg_cases.packed(_cabi, wl, kw, freq=f) for f in freqs]
    probs = [mg_cases.model_problem(wl, kw, freq=f) for f in freqs]
    _check_transposed_apply(handles["fp64"], pks, probs, [kw, kw], "apply_T batch")


def _start_like(rng, prob):
    """Random 4N vector with the ix = 0 / iy = 0 rows zeroed, like the solver's start vector."""
    x = _vec(rng, (4, prob.nx, prob.ny), False)
    x[:, 0, :] = 0
    x[:, :, 0] = 0
    return x.ravel()


@pytest.mark.parametrize("name", CASES)
def test_transposed_preconditioner_inverts_the_transposed_diagonal_part(handles, name):
    wl, kw = _case(name)
    pk, prob = mg_cases.packed(_cabi, wl, kw), mg_cases.model_problem(wl, kw)
    st = prob.st
    n4 = 4 * prob.nx * prob.ny
    Ad = (-1j * _msign(prob, kw)) * T.diagonal_part(st) - st["target"] * T.sp.identity(n4)
    rng = np.random.default_rng(9)
    errs = {}
    for what, A in ((1, Ad.tocsc()), (4, Ad.T.tocsc())):
        x = _start_like(rng, prob)
        z = batch(handles["converged"], [pk], what, (A @ x)[None])[0][0]
        errs[what] = float(np.linalg.norm(z - x) / np.linalg.norm(x))
        _observe(f"precond {what} {name}", errs[what])
    # without PML the converged multigrid inverts mat_d - sigma exactly; with PML it inverts the phase-limited multigrid operator
    assert errs[1] <= (0.5 if any(wl.mode_spec.num_pml) else 1e-6), errs
    assert errs[4] <= max(10 * errs[1], 1e-9), errs
