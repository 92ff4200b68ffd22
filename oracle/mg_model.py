"""Float64 model of the device multigrid preconditioner (test-only).

Mirrors ``tidy3d_b200/csrc`` operation for operation so that the GPU tests can pin every multigrid kernel to it:

- ``plan_hierarchy`` / ``aggregate_axis`` / ``build_axis_transfer`` / ``coarsen_axis``: ``csrc/host_setup.hpp``.  The plan
  aggregates by |lf| of the *unclamped* axes of the batch's first problem; the coarse 1-D coefficients come from the
  phase-clamped axes of each problem (``BatchSolver::build``, ``mg_pml_phase``).
- ``Level``: the second-order diagonal-path operator A - sigma of one level (``stencil_kernel`` and relatives), its
  diagonal (``jacobi0_kernel``) and the stored ``dinv = omega / diag`` smoother.
- ``Transfer``: the tensor-product prolongation / restriction with the PEC-wall rows held at zero (``restrict_kernel``,
  ``prolong_add_kernel``) and the coefficient-field restriction ``restrict_field_kernel`` (R f, and 1 / R(1 / f) for
  1/ezz and 1/mzz, where a zero marker of a removed PEC cell makes the coarse value 0).
- ``Multigrid.vcycle``: ``BatchSolver::vcycle`` and ``fused_vcycle_kernel`` -- jacobi0 plus nu - 1 sweeps, residual,
  restriction, recursion, prolong-add, nu sweeps; on the coarsest level max(2, mg_coarse_iters) Jacobi sweeps from zero,
  or, for indefinite shifts, exactly kc steps of GMRES right-preconditioned by dinv (``BatchSolver::coarse_gmres``).

Nothing under ``tidy3d_b200/`` imports this module.
"""
from __future__ import annotations

import numpy as np

from oracle import restatement as R

PEC_THR = 0.9 * abs(R.PEC_VAL)  # medium.cuh is_pec_val on the real part; the lossy-metal model 1 + 1e8 i is found by |.|
GS_MAX_COEF = 64  # csrc/krylov_kernels.cuh kGsMaxCoef


class Opts:
    """The b200ms_options fields the multigrid depends on (defaults of b200ms_default_options)."""

    FIELDS = dict(mg_min_size=12, mg_nu=2, mg_omega=0.8, mg_coarse_iters=16, mg_ppw=4.0, mg_pml_phase=np.pi / 4, mg_precision=1,
                  ncv=0, gmres_restart=40)

    def __init__(self, src=None, **kw):
        for k, v in self.FIELDS.items():
            setattr(self, k, getattr(src, k, v) if src is not None else v)
        for k, v in kw.items():
            setattr(self, k, v)


# ------------------------------------------------------------------------------------------------
# one problem as the device sets it up
# ------------------------------------------------------------------------------------------------
class Problem:
    """oracle.restatement.setup() output plus what the device derives from it: PEC marks, incidence masking, max_k2."""

    def __init__(self, st, incidence=False, num_modes=1):
        self.st = st
        self.nx, self.ny, self.k0 = st["nx"], st["ny"], st["k0"]
        self.sigma = -(st["target"] ** 2)
        self.num_modes = num_modes
        self.tensorial = st["tensorial"]
        e, m = st["eps"], st["mu"]
        g = lambda a: np.asarray(a, complex).reshape(self.nx, self.ny)  # noqa: E731
        self.pec = [(np.abs(e[q, q]) >= PEC_THR).reshape(self.nx, self.ny) for q in range(3)]
        self.has_pec = bool(any(p.any() for p in self.pec))
        self.masked = self.has_pec and bool(incidence) and not self.tensorial
        self.model_fields = (g(e[0, 0]), g(e[1, 1]), 1 / g(e[2, 2]), g(m[0, 0]), g(m[1, 1]), 1 / g(m[2, 2]))
        ex, ey, iez = (np.where(self.pec[q], 0, f) for q, f in enumerate(self.model_fields[:3]))
        self.marked_fields = (ex, ey, iez) + self.model_fields[3:]
        ok = (np.abs(g(e[0, 0])) < 1e7) & (np.abs(g(e[1, 1])) < 1e7)
        mr = np.maximum(g(e[0, 0]).real, g(e[1, 1]).real)[ok]
        self.max_k2 = max(0.0, (mr.max() if mr.size else -1e300) - st["target"] ** 2)
        self.axes = [Axis(st["slen"][a][0] * self.k0, st["slen"][a][1] * self.k0, st["new_coords"][a], st["pmc"][a]) for a in range(2)]

    @property
    def fields(self):
        """Level-0 coefficient fields of the Krylov-side operator (zero markers where unknowns are removed)."""
        return self.marked_fields if self.masked else self.model_fields

    def mask(self, v):
        """Zero the components of removed PEC unknowns (BatchSolver::mask_E)."""
        if self.masked:
            v = v.copy()
            v[0][self.pec[0]] = 0
            v[1][self.pec[1]] = 0
        return v


class Axis:
    def __init__(self, lf, lb, pos, pmc):
        self.lf, self.lb, self.pos, self.pmc = np.asarray(lf, complex), np.asarray(lb, complex), np.asarray(pos, float), bool(pmc)
        self.n = self.lf.size

    def coefficients(self):
        """Axis::coefficients: rows (f0, f1, b0, bm) of the bidiagonal difference operators."""
        n, lf, lb = self.n, self.lf, self.lb
        f0, f1, b0, bm = (np.zeros(n, complex) for _ in range(4))
        if n > 1:
            f0[:] = -1 / lf
            f1[:-1] = 1 / lf[:-1]
            b0[:] = 1 / lb
            bm[1:] = -1 / lb[1:]
            if not self.pmc:
                f0[0] = 0
            b0[0] = 2 / lb[0] if self.pmc else 0
        return f0, f1, b0, bm

    def clamped(self, phase):
        """The multigrid-side PML stretch: same |s|, phase limited to +-phase (BatchSolver::build)."""
        if not phase > 0:
            return self

        def lim(z):
            ang = np.angle(z)
            return np.where(np.abs(ang) > phase, np.abs(z) * np.exp(1j * np.sign(ang) * phase), z)

        return Axis(lim(self.lf), lim(self.lb), self.pos, self.pmc)

    def coarsen(self, a):
        """coarsen_axis: summed primal lengths, dual lengths averaged, nodes at the aggregate starts."""
        lf = np.add.reduceat(self.lf, a[:-1])
        lb = np.empty_like(lf)
        lb[0] = lf[0]
        lb[1:] = 0.5 * (lf[:-1] + lf[1:])
        return Axis(lf, lb, self.pos[a], self.pmc)


# ------------------------------------------------------------------------------------------------
# hierarchy geometry
# ------------------------------------------------------------------------------------------------
def aggregate_axis(lf, H, slack=1.25, max_cells=3):
    ell = np.abs(lf)
    n = ell.size
    st, i = [], 0
    while i < n:
        st.append(i)
        tot, cnt = ell[i], 1
        while i + cnt < n and cnt < max_cells and tot + ell[i + cnt] <= slack * H:
            tot += ell[i + cnt]
            cnt += 1
            if cnt >= 2 and tot >= 0.75 * H:
                break
        i += cnt
    st.append(n)
    return np.array(st)


def plan_hierarchy(axes, min_size=12, max_levels=12, kh_limit=0.0, kmax=0.0):
    """Aggregations (ax, ay) from level l to l + 1, as plan_hierarchy builds them from the unclamped axes."""
    cur = list(axes)
    h0 = min(np.abs(ax.lf).min() for ax in cur if ax.n > 1)
    H, plan, guard = h0, [], 0
    while len(plan) + 1 < max_levels and max(cur[0].n, cur[1].n) > min_size and guard < 40:
        guard += 1
        H *= 2
        if kh_limit > 0 and kmax * H > kh_limit:
            break
        agg = [aggregate_axis(ax.lf, H) if ax.n > 1 else np.array([0, 1]) for ax in cur]
        if len(agg[0]) - 1 == cur[0].n and len(agg[1]) - 1 == cur[1].n:
            continue
        plan.append(agg)
        cur = [ax.coarsen(a) for ax, a in zip(cur, agg)]
    return plan


def transfer_1d(a, pos):
    """build_axis_transfer: dense prolongation P (n x nc) of node- and edge-type unknowns."""
    nc, n = len(a) - 1, a[-1]
    Pn, Pe = np.zeros((n, nc)), np.zeros((n, nc))
    Xc = 0.5 * (pos[a[:-1]] + pos[a[1:]])
    for I in range(nc):
        x0, x1 = pos[a[I]], pos[a[I + 1]]
        for i in range(a[I], a[I + 1]):
            t = (pos[i] - x0) / (x1 - x0)
            Pn[i, I] += 1 - t
            if I + 1 < nc:
                Pn[i, I + 1] += t
            xc = 0.5 * (pos[i] + pos[i + 1])
            if xc < Xc[I] and I > 0:
                u = (xc - Xc[I - 1]) / (Xc[I] - Xc[I - 1])
                Pe[i, I - 1] += 1 - u
                Pe[i, I] += u
            elif xc > Xc[I] and I + 1 < nc:
                u = (xc - Xc[I]) / (Xc[I + 1] - Xc[I])
                Pe[i, I] += 1 - u
                Pe[i, I + 1] += u
            else:
                Pe[i, I] += 1.0
    return Pn, Pe


class Transfer:
    """Tensor-product transfer between level l (fine) and l + 1.  Restriction = normalised transpose (rows sum to one)."""

    def __init__(self, agg, axes):
        (ax, ay), (fx, fy) = agg, axes
        self.Pxn, self.Pxe = transfer_1d(ax, fx.pos)
        self.Pyn, self.Pye = transfer_1d(ay, fy.pos)
        nrm = lambda P: (P / np.where(P.sum(0) > 0, P.sum(0), 1.0)).T  # noqa: E731
        self.Rxn, self.Rxe, self.Ryn, self.Rye = nrm(self.Pxn), nrm(self.Pxe), nrm(self.Pyn), nrm(self.Pye)
        # PEC min walls: Ex[:, 0] (mask_y) and Ey[0, :] (mask_x) are decoupled unknowns held at zero on every level
        self.mask_y = not fy.pmc and fy.n > 1
        self.mask_x = not fx.pmc and fx.n > 1

    def _walls(self, v):
        if self.mask_y and v.shape[2] > 1:
            v[0][:, 0] = 0
        if self.mask_x and v.shape[1] > 1:
            v[1][0, :] = 0
        return v

    def restrict(self, f):  # Ex: x edge / y node, Ey: x node / y edge
        return self._walls(np.stack((self.Rxe @ f[0] @ self.Ryn.T, self.Rxn @ f[1] @ self.Rye.T)))

    def prolong(self, c):  # the wall rows of the fine vector are not updated
        return self._walls(np.stack((self.Pxe @ c[0] @ self.Pyn.T, self.Pxn @ c[1] @ self.Pye.T)))

    def field(self, f, xt, yt, reciprocal=False):
        """restrict_field_kernel on one coefficient field of site type (xt, yt) in {"e", "n"}."""
        Rx = self.Rxe if xt == "e" else self.Rxn
        Ry = self.Rye if yt == "e" else self.Ryn
        if not reciprocal:
            return Rx @ f @ Ry.T
        zero = f == 0  # 1/ezz zeroed on a removed PEC cell: infinite reciprocal, coarse value 0
        acc = Rx @ np.where(zero, 0, 1 / np.where(zero, 1, f)) @ Ry.T
        hit = (Rx @ zero.astype(float) @ Ry.T) > 0
        return np.where(hit, 0, 1 / np.where(hit, 1, acc))

    def coarse_fields(self, fields):
        exx, eyy, iez, mxx, myy, imz = fields
        return (self.field(exx, "e", "n"), self.field(eyy, "n", "e"), self.field(iez, "n", "n", True),
                self.field(mxx, "n", "e"), self.field(myy, "e", "n"), self.field(imz, "e", "e", True))


# ------------------------------------------------------------------------------------------------
# one level's operator
# ------------------------------------------------------------------------------------------------
class Level:
    """(A - sigma) of one level: 1-D coefficients of its two axes, six coefficient fields (nx, ny) and the shift."""

    def __init__(self, axes, fields, sigma, omega):
        self.axes = axes
        self.nx, self.ny = axes[0].n, axes[1].n
        self.exx, self.eyy, self.iez, self.mxx, self.myy, self.imz = fields
        self.fields = fields
        self.sigma = sigma
        self.coef = [ax.coefficients() for ax in axes]
        self.diag = self._diagonal() - sigma
        self.dinv = omega / self.diag

    def apply(self, v, shifted=True):
        (xf0, xf1, xb0, xbm), (yf0, yf1, yb0, ybm) = self.coef
        v1, v2 = v[0], v[1]
        t = xf0[:, None] * v2 - yf0[None, :] * v1
        t[:-1] += xf1[:-1, None] * v2[1:]
        t[:, :-1] -= yf1[None, :-1] * v1[:, 1:]
        t = t * self.imz
        a, b = self.exx * v1, self.eyy * v2
        u = xb0[:, None] * a + yb0[None, :] * b
        u[1:] += xbm[1:, None] * a[:-1]
        u[:, 1:] += ybm[None, 1:] * b[:, :-1]
        u = -u * self.iez
        p1 = xf0[:, None] * u
        p1[:-1] += xf1[:-1, None] * u[1:]
        dybt = yb0[None, :] * t
        dybt[:, 1:] += ybm[None, 1:] * t[:, :-1]
        p1 = p1 + self.myy * (dybt - a)
        p2 = yf0[None, :] * u
        p2[:, :-1] += yf1[None, :-1] * u[:, 1:]
        dxbt = xb0[:, None] * t
        dxbt[1:] += xbm[1:, None] * t[:-1]
        p2 = p2 - self.mxx * (dxbt + b)
        out = np.stack((p1, p2))
        return out - self.sigma * v if shifted else out

    def abs_apply(self, v):
        """An upper bound of the row-wise |A - sigma| |v| (the scale of an apply's rounding error): the stencil with every
        coefficient, field and value replaced by its absolute value and every difference by a sum."""
        (xf0, xf1, xb0, xbm), (yf0, yf1, yb0, ybm) = [[np.abs(c) for c in cc] for cc in self.coef]
        exx, eyy, iez, mxx, myy, imz = (np.abs(f) for f in self.fields)
        w1, w2 = np.abs(v[0]), np.abs(v[1])
        t = xf0[:, None] * w2 + yf0[None, :] * w1
        t[:-1] += xf1[:-1, None] * w2[1:]
        t[:, :-1] += yf1[None, :-1] * w1[:, 1:]
        t = t * imz
        a, b = exx * w1, eyy * w2
        u = xb0[:, None] * a + yb0[None, :] * b
        u[1:] += xbm[1:, None] * a[:-1]
        u[:, 1:] += ybm[None, 1:] * b[:, :-1]
        u = u * iez
        p1 = xf0[:, None] * u
        p1[:-1] += xf1[:-1, None] * u[1:]
        dybt = yb0[None, :] * t
        dybt[:, 1:] += ybm[None, 1:] * t[:, :-1]
        p2 = yf0[None, :] * u
        p2[:, :-1] += yf1[None, :-1] * u[:, 1:]
        dxbt = xb0[:, None] * t
        dxbt[1:] += xbm[1:, None] * t[:-1]
        return np.stack((p1 + myy * (dybt + a), p2 + mxx * (dxbt + b))) + abs(self.sigma) * np.abs(v)

    def _diagonal(self):
        (xf0, xf1, xb0, xbm), (yf0, yf1, yb0, ybm) = self.coef
        iez, imz = self.iez, self.imz
        z = lambda: np.zeros((self.nx, self.ny), complex)  # noqa: E731
        s = z(); s += (xf0 * xb0)[:, None] * iez; s[:-1] += (xf1[:-1] * xbm[1:])[:, None] * iez[1:]  # noqa: E702
        d1 = -self.exx * s
        s = z(); s += (yb0 * yf0)[None, :] * imz; s[:, 1:] += (ybm[1:] * yf1[:-1])[None, :] * imz[:, :-1]  # noqa: E702
        d1 = d1 - self.myy * s - self.myy * self.exx
        s = z(); s += (yf0 * yb0)[None, :] * iez; s[:, :-1] += (yf1[:-1] * ybm[1:])[None, :] * iez[:, 1:]  # noqa: E702
        d2 = -self.eyy * s
        s = z(); s += (xb0 * xf0)[:, None] * imz; s[1:] += (xbm[1:] * xf1[:-1])[:, None] * imz[:-1]  # noqa: E702
        d2 = d2 - self.mxx * s - self.mxx * self.eyy
        return np.stack((d1, d2))

    # the smoother, as the device runs it with the stored dinv
    def jacobi0(self, rhs):
        return self.dinv * rhs

    def sweep(self, x, rhs):
        return x + self.dinv * (rhs - self.apply(x))

    def two_sweeps_from_zero(self, rhs):  # MODE_JACOBI_D0
        return self.sweep(self.jacobi0(rhs), rhs)


def true_level(prob):
    """Level 0 of the Krylov-side operator: true PML, the problem's own (possibly zero-marked) fields."""
    return Level(prob.axes, prob.fields, prob.sigma, 1.0)


# ------------------------------------------------------------------------------------------------
# the preconditioner
# ------------------------------------------------------------------------------------------------
class Multigrid:
    """The multigrid hierarchy of one problem of a device batch and its V-cycle.

    plan / kmax: the batch's hierarchy geometry and largest k (the device takes the plan from problem 0 and kmax over the
    whole batch); by default those of this problem alone.  fused_tail only changes the device's kernels, not the model."""

    def __init__(self, prob, opts=None, plan=None, kmax=None):
        o = opts if isinstance(opts, Opts) else Opts(opts)
        self.prob, self.opts = prob, o
        k2 = prob.max_k2 if kmax is None else kmax**2
        kh_limit, km = 0.0, 0.0
        if k2 > 1e-6 and o.mg_ppw > 0:
            km, kh_limit = np.sqrt(k2), 2 * np.pi / o.mg_ppw
        self.coarse_krylov = kh_limit > 0
        self.plan = plan_hierarchy(prob.axes, o.mg_min_size, 12, kh_limit, km) if plan is None else plan
        # fp64 multigrid: the level-0 fields are those of the Krylov-side operator (zero markers included); the fp32 twin
        # keeps the PEC model (medium.cuh fields_kernel)
        fields = prob.fields if o.mg_precision == 0 else prob.model_fields
        axes = [ax.clamped(o.mg_pml_phase) for ax in prob.axes]
        self.levels = [Level(axes, fields, prob.sigma, o.mg_omega)]
        self.tr = []
        plan_axes = prob.axes
        for agg in self.plan:
            tr = Transfer(agg, axes)
            fields = tr.coarse_fields(fields)
            axes = [ax.coarsen(a) for ax, a in zip(axes, agg)]
            plan_axes = [ax.coarsen(a) for ax, a in zip(plan_axes, agg)]
            self.tr.append(tr)
            self.levels.append(Level(axes, fields, prob.sigma, o.mg_omega))
        n2 = 2 * prob.nx * prob.ny
        length = 2 * n2 if prob.tensorial else n2
        ncv = o.ncv if o.ncv > 0 else max(2 * prob.num_modes + 1, 20)
        m = min(ncv, length - 1)
        if m < prob.num_modes + 2:
            m = min(prob.num_modes + 2, length)
        restart = min(max(2, o.gmres_restart), GS_MAX_COEF - 4)
        self.kc = max(2, min(o.mg_coarse_iters, max(m, restart) - 1))

    @property
    def shapes(self):
        return [(lv.nx, lv.ny) for lv in self.levels]

    def coarse_gmres(self, lv, b):
        """Exactly kc GMRES steps, right-preconditioned by dinv, no early stop; x = Z y with y the least-squares solution."""
        kc = self.kc
        beta = np.linalg.norm(b)
        V, Z = [b / beta], []
        H = np.zeros((kc + 1, kc), complex)
        for j in range(kc):
            z = lv.jacobi0(V[j])
            w = lv.apply(z)
            for _ in range(2):
                h = np.array([np.vdot(v, w) for v in V])
                w = w - sum(hi * v for hi, v in zip(h, V))
                H[: j + 1, j] += h
            H[j + 1, j] = np.linalg.norm(w)
            V.append(w / H[j + 1, j])
            Z.append(z)
        g = np.zeros(kc + 1, complex)
        g[0] = beta
        y = np.linalg.lstsq(H, g, rcond=None)[0]
        return sum(yi * z for yi, z in zip(y, Z))

    def vcycle(self, b, level=0):
        o = self.opts
        lv = self.levels[level]
        last = level == len(self.levels) - 1
        if last and self.coarse_krylov:
            return self.coarse_gmres(lv, b)
        nu = max(1, o.mg_nu)
        nsw = max(2, o.mg_coarse_iters) if last else nu
        x = lv.jacobi0(b)
        for _ in range(nsw - 1):
            x = lv.sweep(x, b)
        if last:
            return x
        r = b - lv.apply(x)
        tr = self.tr[level]
        x = x + tr.prolong(self.vcycle(tr.restrict(r), level + 1))
        for _ in range(nu):
            x = lv.sweep(x, b)
        return x

    def precondition(self, b):
        """One preconditioner application of the diagonal path (BatchSolver::precondition): V-cycle, then the PEC mask."""
        return self.prob.mask(self.vcycle(b))
