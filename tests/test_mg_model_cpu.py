"""CPU: the float64 multigrid model (oracle/mg_model.py) that the GPU kernel tests compare against is itself right where it
can be checked without a device -- its hierarchy is the library's (b200ms_debug_hierarchy), its level-0 operator is the
reference's assembled matrix, its restriction averages, and the PEC-wall unknowns stay out of the V-cycle."""
import ctypes as C

import numpy as np
import pytest

from oracle import mg_model as M
from oracle import restatement as R
from tests import mg_cases
from tests.golden.cases import CASES

SMALL_DIAGONAL = [n for n in CASES if "256" not in n and "512" not in n and "angle" not in n and "offdiag" not in n and "rand10" not in n
                  and "relative" not in n and "split" not in n]


@pytest.mark.parametrize("name", SMALL_DIAGONAL + ["strip_75x131", "strip_256", "pec_block_40_mu"])
def test_model_hierarchy_is_the_librarys(built_lib, name):
    wl, kw = mg_cases.case(name)
    pk = mg_cases.packed(built_lib, wl, kw)
    sh = (C.c_int * 40)()
    n = built_lib.lib().b200ms_debug_hierarchy(C.byref(pk.struct), None, 20, sh)
    mg = M.Multigrid(mg_cases.model_problem(wl, kw))
    assert mg.shapes == [(sh[2 * i], sh[2 * i + 1]) for i in range(n)]


@pytest.mark.parametrize("name", ["c1_64", "c1_64_sym_pmc_pec", "nonuniform_56", "c3_96", "c4_96", "lossy_48", "mu_cross_40", "pec_block_40", "slab1d_x1"])
def test_model_level0_is_the_assembled_operator(name):
    """Without the phase clamp the model's level 0 is A - sigma of solver.py:471-490 to rounding."""
    wl, kw = mg_cases.case(name)
    prob = mg_cases.model_problem(wl, kw)
    lv = M.Multigrid(prob, M.Opts(mg_pml_phase=0.0, mg_precision=0)).levels[0]
    A = R.assemble_diagonal(prob.st)[2]
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, prob.nx, prob.ny)) + 1j * rng.standard_normal((2, prob.nx, prob.ny))
    ref = A @ x.ravel() - prob.sigma * x.ravel()
    scale = (abs(A) @ np.abs(x.ravel()) + abs(prob.sigma) * np.abs(x.ravel())).max()
    assert np.abs(lv.apply(x).ravel() - ref).max() <= 1e-12 * scale
    assert np.abs(lv.diag.ravel() - (A.diagonal() - prob.sigma)).max() <= 1e-12 * np.abs(A.diagonal()).max()
    assert (lv.abs_apply(x).ravel() >= (1 - 1e-12) * np.abs(ref)).all()


@pytest.mark.parametrize("name", ["c1_64", "nonuniform_56", "c3_96", "slab1d_y1", "strip_75x131"])
def test_model_restriction_rows_sum_to_one(name):
    wl, kw = mg_cases.case(name)
    mg = M.Multigrid(mg_cases.model_problem(wl, kw))
    assert mg.tr
    for tr in mg.tr:
        for Rm in (tr.Rxn, tr.Rxe, tr.Ryn, tr.Rye):
            assert np.abs(Rm.sum(1) - 1).max() < 1e-14
            assert (Rm >= 0).all()


def test_model_coarse_reciprocal_field_of_a_removed_pec_cell_is_zero():
    """1/ezz zeroed on a removed PEC cell: its reciprocal is infinite, so every coarse cell it feeds has 1/ezz = 0."""
    wl, kw = mg_cases.case("pec_block_40_mu")
    prob = mg_cases.model_problem(wl, kw)
    assert prob.masked and prob.pec[2].any()
    mg = M.Multigrid(prob, M.Opts(mg_precision=0))
    iez = mg.levels[1].iez
    assert np.isfinite(iez).all() and (iez == 0).any()
    hit = (mg.tr[0].Rxn @ prob.pec[2].astype(float) @ mg.tr[0].Ryn.T) > 0
    assert (iez[hit] == 0).all() and (iez[~hit] != 0).all()


@pytest.mark.parametrize("name", ["c1_64", "c3_96", "c1_64_sym_pmc_pec"])
def test_model_pec_wall_rows_stay_zero_through_a_vcycle(name):
    wl, kw = mg_cases.case(name)
    prob = mg_cases.model_problem(wl, kw)
    mg = M.Multigrid(prob)
    pmc = prob.st["pmc"]
    rng = np.random.default_rng(2)
    r = rng.standard_normal((2, prob.nx, prob.ny)) + 0j
    if not pmc[1]:
        r[0][:, 0] = 0
    if not pmc[0]:
        r[1][0, :] = 0
    z = mg.vcycle(r)
    assert np.abs(z).max() > 0
    if not pmc[1]:
        assert (z[0][:, 0] == 0).all()
    if not pmc[0]:
        assert (z[1][0, :] == 0).all()
    assert pmc[0] or pmc[1] or name != "c1_64_sym_pmc_pec"
