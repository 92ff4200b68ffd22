"""The problems the multigrid model tests run: golden cases plus a few made for the kernels' edge cases, each as the
library sees it (a PackedProblem) and as the float64 model sees it (oracle.mg_model.Problem)."""
import numpy as np

from oracle import mg_model as M
from oracle import restatement as R
from tests.golden import cases as G
from tidy3d_b200 import workloads as W


def strip(nx, ny):
    """Real lossless strip without PML: odd widths take the one-column kernel, 256^2 the TMA pair kernel and a fused tail."""
    eps, coords = W.strip_eps(nx, ny)
    return W.Workload(name=f"strip_{nx}x{ny}", eps_cross=W._iso(eps), coords=coords, freqs=np.array([W.C_0 / 1.55]),
                      mode_spec=W.ModeSpecLike(num_modes=2, precision="double"))


def pec_block_mu():
    """pec_block_40 with a magnetic cladding: the incidence formulation with PEC cells, so unknowns are removed."""
    wl = G._pec_block(40)
    wl.extra["mu_cross"] = G._mu_and_split(40).extra["mu_cross"]
    wl.name = "pec_block_40_mu"
    return wl, {"mu_cross": "extra"}


EXTRA = {
    "strip_75x131": lambda: (strip(75, 131), {}),
    "strip_256": lambda: (strip(256, 256), {}),
    "pec_block_40_mu": pec_block_mu,
}


def case(name):
    """(workload, compute_modes kwargs with the "extra" markers resolved)"""
    if name in EXTRA:
        wl, kw = EXTRA[name]()
    else:
        fac, kw, _ = G.CASES[name]
        wl = fac()
    return wl, G.resolve_kwargs(wl, kw)


def packed(cabi, wl, kw, freq=None, eps=None, coords=None):
    """The library's view of the problem, with the incidence flag compute_modes sets (mu_cross or split-curl scaling given)."""
    return cabi.PackedProblem(wl.eps_cross, coords if coords is not None else wl.coords, wl.freqs[0] if freq is None else freq,
                              wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("direction", "+"), eps_packed=eps,
                              mu_cross=kw.get("mu_cross"), incidence=kw.get("mu_cross") is not None)


def model_problem(wl, kw, freq=None):
    st = R.setup(wl.eps_cross, wl.coords, wl.freqs[0] if freq is None else freq, wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))
    return M.Problem(st, incidence=kw.get("mu_cross") is not None, num_modes=wl.mode_spec.num_modes)


def is_real(wl, kw):
    st = R.setup(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec, kw.get("symmetry", (0, 0)), kw.get("mu_cross"))
    return not np.issubdtype(R.solver_dtype(st, "double"), np.complexfloating)
