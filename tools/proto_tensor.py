"""DEV TOOL (CPU, numpy): the block preconditioner of the tensorial (4N first-order) path with an inexact E-block inverse.

The library preconditions (mat - sigma), mat = -i [[Aee, P'],[Q', Ahh]], with the inverse of its diagonal-tensor part
mat_d = -i [[0, P],[Q, 0]]:  (mat_d - sigma)^-1 = -(mat_d + sigma) blockdiag((PQ - s)^-1, (QP - s)^-1), s = -sigma^2, with
(PQ - s)^-1 ~ B_E = one multigrid V-cycle and (QP - s)^-1 = -(1/s)(I - Q B_E P).  The second identity holds for the exact inverse only:
with a V-cycle (relative error ~0.15) the difference of two O(K^2) terms carries an O(0.15 K^2) error where the exact result is O(K^-2),
K = 1/(k0 h).  This script measures FGMRES iteration counts for (a) exact B_E, (b) one V-cycle in both places (the library today),
(c) the H-block through n steps of defect correction x <- x + B_E (r - (PQ - s) x) on the E-side system.
The multigrid is oracle/mg_model.py with the settings the experiment was run with (unclamped PML, 16 Jacobi sweeps on the coarsest
level); with it, variant (b) takes 25 / 53 iterations at 64^2 / 96^2 (csrc/solver.cuh quotes 25 / 52 from the original run).
usage: python tools/proto_tensor.py [n ...]"""
import sys
import time

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

sys.path.insert(0, "/root/repo")
sys.path.insert(0, "/root/repo/tools")
import proto as P  # noqa: E402
from oracle import restatement as R  # noqa: E402
from tidy3d_b200 import workloads as W  # noqa: E402

rng = np.random.default_rng(5)


def run(n, theta=0.2):
    wl = W.angled(n, theta=theta, phi=0.0, num_modes=4)
    st = R.setup(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec)
    N = st["nx"] * st["ny"]
    sigma = st["target"]  # eigenvalue of mat is n_eff
    M4 = (-1j * R.assemble_tensorial(st)).tocsr()
    pm, qm, A = R.assemble_diagonal(st)
    s = -sigma**2
    As = (A - s * sp.identity(2 * N)).tocsc()
    lu = spl.splu(As)
    # the multigrid this experiment was run with: unclamped PML, no wavelength limit on the hierarchy, 16 Jacobi sweeps on the
    # coarsest level (mg_ppw = 0 keeps the indefinite shift from switching the coarsest level to GMRES)
    mg = P.Multigrid(P.Problem(st), P.Opts(mg_precision=0, mg_pml_phase=0.0, mg_ppw=0.0))
    shp = (2, st["nx"], st["ny"])

    def vc(r):
        return mg.vcycle(r.reshape(shp)).ravel()

    def exact(r):
        return lu.solve(r)

    def defect(nsteps):
        def f(r):
            x = vc(r)
            for _ in range(nsteps - 1):
                x = x + vc(r - As @ x)
            return x
        return f

    def prec(BE, BH_from):
        # z = -(mat_d + sigma) [B_E v_e ; B_H v_h],  B_H = -(1/s)(I - Q BH_from P)
        def f(v):
            ve, vh = v[: 2 * N], v[2 * N:]
            ye = BE(ve)
            yh = -(1 / s) * (vh - qm @ BH_from(pm @ vh))
            ze = -sigma * ye + 1j * (pm @ yh)
            zh = -sigma * yh + 1j * (qm @ ye)
            return np.concatenate([ze, zh])
        return f

    Ms = (M4 - sigma * sp.identity(4 * N)).tocsr()
    b = rng.standard_normal(4 * N) + 0j
    print(f"== angled n={n} theta={theta}: N={N} sigma={sigma:.4f} levels={[(l.nx, l.ny) for l in mg.levels]}", flush=True)
    variants = [("exact B_E", prec(exact, exact), 0), ("V-cycle / V-cycle (library)", prec(vc, vc), 2)]
    for ne, nh in ((1, 3), (2, 2), (3, 3), (4, 4), (2, 4), (3, 6), (6, 6)):
        variants.append((f"{ne} / {nh} defect-correction cycles", prec(defect(ne), defect(nh)), ne + nh))
    if QUICK:
        variants = [v for v in variants if v[2] in (0, 2, 4, 6, 8)]
    for name, pr, ncyc in variants:
        t0 = time.time()
        x, its, rr = P.fgmres(lambda z: Ms @ z, pr, b, tol=1e-8, restart=40, maxit=200)
        print(f"   {name:36s} its {its:4d} relres {rr:.1e}  V-cycles {its * ncyc:5d}  ({time.time() - t0:.1f} s)", flush=True)


QUICK = "quick" in sys.argv
for n in [int(a) for a in sys.argv[1:] if a.isdigit()] or [64, 96]:
    run(n)
