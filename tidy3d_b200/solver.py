"""Host-side mirror of the reference mode-solver interface, backed by the CUDA library.

``compute_modes`` has the signature, return value and error behaviour of
``tidy3d.plugins.mode.solver.compute_modes`` (tidy3d/plugins/mode/solver.py:33-44, 941-943):

    fields, n_complex, eps_spec = compute_modes(eps_cross, coords, freq, mode_spec, symmetry=..., direction=...)

``fields`` has shape ``(2, 3, Nx, Ny, 1, num_modes)`` (E/H, component, x, y, 1, mode), ``n_complex`` is
``n_eff + 1j*k_eff`` sorted by descending ``n_eff`` and ``eps_spec`` is ``"diagonal"``, ``"tensorial_real"`` or
``"tensorial_complex"``.  ``compute_modes_batch`` is the batched entry point that corresponds to the
frequency loop of ``ModeSolver._solve_all_freqs`` (tidy3d/plugins/mode/mode_solver.py:655-672): all problems are
solved concurrently on the GPU.
"""
from __future__ import annotations

import threading
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _cabi

_handles = {}
_hlock = threading.Lock()

# Tolerance presets.  "reference" (the default of the library) asks for what the reference asks ARPACK for
# (tol = TOL_EIGS = fp_eps, solver.py:20, 745); "tight" is the setting the parity tests use to pin n_eff to 1e-8.
TOLERANCES = {"reference": dict(eig_tol=1.1920928955078125e-07, inner_tol=1e-8), "tight": dict(eig_tol=1e-9, inner_tol=1e-10)}


def get_handle(device: int = -1, tolerance: str = "reference") -> _cabi.Handle:
    """One cached solver handle per (GPU, tolerance preset).  Calls on one handle are serialised by a per-handle lock
    (ctypes releases the GIL during the solve and the C ABI forbids overlapping calls on a handle)."""
    key = (device, tolerance)
    with _hlock:
        if key not in _handles:
            _handles[key] = _cabi.Handle(device, **TOLERANCES[tolerance])
        return _handles[key]


def _raise_for(rc: int, handle, where="", msg=None):
    msg = handle.last_error() if msg is None else msg
    if rc == _cabi.ERR_SHAPE:
        raise ValueError("Mismatch between 'coords' and 'esp_cross' shapes.")  # solver.py:107
    if rc == _cabi.ERR_NO_MODES:
        raise RuntimeError("Could not find any eigenmodes for this waveguide.")  # solver.py:876
    if rc == _cabi.ERR_UNSUPPORTED:
        raise NotImplementedError(f"tidy3d_b200: {msg}")
    if rc == _cabi.ERR_NOCONV:
        raise RuntimeError(f"tidy3d_b200: eigen-iteration did not converge {where}: {msg}")  # ArpackNoConvergence
    if rc == _cabi.ERR_CUDA:
        raise RuntimeError(f"tidy3d_b200: CUDA failure (no CPU fallback): {msg}")
    if rc != _cabi.OK:
        raise RuntimeError(f"tidy3d_b200: error {rc}: {msg}")


PEC_VAL = -1e8  # tidy3d/constants.py


def _apply_split_curl(eps_cross, split):
    """solver.py:122-124: eps_rr -> eps_rr / scaling_r outside PEC (scaling == 0 marks PEC)."""
    eps = [np.array(eps_cross[i], dtype=np.complex128, copy=True) for i in range(9)]
    for comp, idx in enumerate((0, 4, 8)):
        sc = np.asarray(split[comp])
        outside = ~np.isclose(sc, 0)
        eps[idx][outside] /= sc[outside]
    return eps


def _undo_split_curl(fields, split):
    """solver.py:904-919 applied to the packed (2,3,Nx,Ny,1,M) array: E -> E / scaling, zero inside PEC."""
    split = np.asarray(split)
    outside = ~np.isclose(split, 0)
    scale = np.where(outside, split, 1.0)
    fields[0] = (fields[0] / scale[:, :, :, None, None] * outside[:, :, :, None, None]).astype(fields.dtype)
    return fields


def compute_modes_batch(
    problems: Sequence[dict], device: int = -1, want_fields: bool = True, return_info: bool = False, handle=None,
    fields_ptrs=None, post: Optional[Sequence[str]] = None, derivatives: Optional[Sequence[str]] = None, left_solve: bool = False,
):
    """Solve many independent mode problems in one device call.

    Each problem is a dict with the keyword arguments of ``compute_modes`` (``eps_cross, coords, freq, mode_spec``
    and optionally ``symmetry, direction``).  Problems that share the same ``eps_cross`` object are packed once.
    Returns a list of ``(fields, n_complex, eps_spec)`` tuples (``fields`` is None when ``want_fields=False``),
    plus a list of per-problem info dicts when ``return_info``.  ``fields_ptrs`` (list of raw addresses, host or device
    memory) makes the library write each problem's fields there instead (``fields`` is then None): used to keep the
    fields in HBM for the NCCL gather of ``tidy3d_b200.sharding`` / on-device post-processing.

    ``post``: on-device post-processing applied to the fields before they are delivered (``tidy3d_b200.postprocess``):
    any of ``"gauge"`` (mode_solver.py:802-810), ``"normalize"`` (flux normalisation, mode_solver.py:517-521), ``"flux"``
    (report each mode's flux and TE polarisation fraction in the info dict) and ``"overlaps"`` (M x M modal overlap matrix with the previous problem of
    the call, monitor_data.py:640-697, in the info dict as ``overlap_prev``; the input of ``postprocess.overlap_sort``).
    With ``want_fields=False`` only ``n_complex`` and these small results leave the GPU.  A problem may carry
    ``grid_correction=postprocess.grid_correction_table(...)``: flux, normalisation and overlaps then include the
    finite-grid correction factors of ``ModeSolver._grid_correction`` (mode_solver.py:847-904), like the reference's; and
    ``plane_bounds=(xmin, xmax, ymin, ymax)`` (``plugin.plane_bounds_of``): the extent of a finite mode plane, to which the
    integration weights are truncated like the reference's ``_diff_area`` (monitor_data.py:437-455).

    ``derivatives``: first-order derivatives of every mode from its own solve (left eigenvector, no extra solves; diagonal
    problems only, else ``NotImplementedError``).  ``"freq"`` adds ``dn_dfreq`` (d(n_eff + i k_eff)/df, 1/Hz) and ``n_group``
    (n_eff + f Re(dn/df), what ``ModeData._group_index_post_process`` approximates from three solves) to the info dict;
    ``"eps"`` adds ``dn_deps`` (3, Nx, Ny, M): d(n_eff + i k_eff) / d eps_{xx,yy,zz} of ``eps_cross`` at every Yee site (PML stretch
    held fixed).  Material dispersion enters ``dn_dfreq`` through a problem's ``eps_dfreq=`` (d eps_cross / df) or, for a
    ``section``, through the media whose ``eps`` is a callable.  ``"freq2"`` adds the group-velocity dispersion from one
    correction solve per mode on top of the same solve: ``d2n_dfreq2`` (d^2(n_eff + i k_eff)/df^2, 1/Hz^2; NaN for a mode whose
    correction solve stopped above 100 x the inner tolerance), ``d2n_residual`` (that solve's final relative residual) and
    ``dispersion`` (ps/(nm km), ``plugin.dispersion_of``: the step -> 0 limit of ``plugin.group_index``), and implies
    ``"freq"``; its material term comes from a problem's ``eps_dfreq=`` and ``eps_d2freq=`` (d^2 eps_cross / df^2) or a
    section's callable media.  ``n_complex``, the fields, ``dn_dfreq`` and ``dn_deps`` do not change.  ``"group_eps"`` adds the
    permittivity gradient of the group index from the same correction solves (no further solve): ``d2n_dfreq_deps`` (3, Nx, Ny, M),
    d(dn/df) / d eps_{xx,yy,zz} (1/Hz) at every Yee site at fixed d eps / df and PML stretch (NaN where ``d2n_dfreq2`` is), and
    ``dng_deps`` = Re ``dn_deps`` + f Re ``d2n_dfreq_deps``, the gradient of ``n_group`` for a real change of eps.  It implies
    ``"freq"``, ``"eps"`` and ``"freq2"``, whose outputs do not change.  ``"freq3"`` adds the third-order dispersion from the same
    correction solves (no further solve, by the 2n+1 rule): ``d3n_dfreq3`` (d^3(n_eff + i k_eff)/df^3, 1/Hz^3; NaN where
    ``d2n_dfreq2`` is), ``dispersion_slope`` (dD/d(wavelength), ps/(nm^2 km), ``plugin.dispersion_slope_of``) and ``beta3``
    (d^3 beta / d omega^3, ps^3/km, ``plugin.beta3_of``).  It implies ``"freq2"`` and ``"freq"``, whose outputs do not change;
    its material term also reads a problem's ``eps_d3freq=`` (d^3 eps_cross / df^3) or a section's callable media.  ``"freq4"``
    adds the fourth-order dispersion from one more correction solve per mode (the second-order correction of the eigenvector):
    ``d4n_dfreq4`` (d^4(n_eff + i k_eff)/df^4, 1/Hz^4; NaN for a mode whose first or second correction solve stopped above 100 x
    the inner tolerance), ``d4n_residual`` (the second solve's final relative residual) and ``beta4`` (d^4 beta / d omega^4,
    ps^4/km, ``plugin.beta4_of``).  It implies ``"freq3"``, ``"freq2"`` and ``"freq"``, whose outputs do not change; its material
    term also reads a problem's ``eps_d4freq=`` (d^4 eps_cross / df^4) or a section's callable media.  ``"disp_eps"`` adds the
    permittivity gradient of the group-velocity dispersion from the corrections of ``"group_eps"`` and ``"freq4"`` (no further
    solve): ``d2n_dfreq2_deps`` (3, Nx, Ny, M), d(d^2n/df^2) / d eps_{xx,yy,zz} (1/Hz^2) at every Yee site at fixed d eps / df,
    d^2 eps / df^2 and PML stretch (NaN where ``d4n_dfreq4`` is), and ``dispersion_deps`` (ps/(nm km) per unit eps,
    ``plugin.dispersion_gradient_of``), the gradient of ``dispersion`` for a real change of eps.  It implies ``"group_eps"`` and
    ``"freq4"``, whose outputs do not change.  Tensorial problems raise.

    ``left_solve=True`` extends ``"freq"`` and ``"eps"`` to tensorial problems (angled planes, off-diagonal eps such as rotated
    anisotropic crystals), which otherwise raise ``NotImplementedError``: their left eigenvectors come from a second eigen-solve
    with the transposed operator, about the cost of one more solve per device batch that holds such a problem.  ``dn_deps`` is
    then (9, Nx, Ny, M), d(n_eff + i k_eff) / d eps_ab of ``eps_cross`` in its component order (xx, xy, ..., zz) at fixed PML
    stretch and mu; material dispersion reads all nine components of ``eps_dfreq=`` or of a section's callable media.  A mode whose
    left eigenvector could not be paired with it gets NaN; ``left_paired`` in the info dict counts the modes that were (num_modes
    for diagonal problems, -1 without derivatives).  Diagonal problems solve as without the flag and report ``dn_deps`` as
    (3, Nx, Ny, M).  With it, ``"freq2"``, ``"group_eps"`` and ``"freq3"`` still raise on tensorial problems.

    ``"pert"``, ``"group_pert"`` and ``"disp_pert"`` contract the maps of ``"eps"``, ``"group_eps"`` and ``"disp_eps"`` on the
    device against K caller-given permittivity perturbations, so that no per-cell map is written or copied: each problem may carry
    ``eps_pert=``, a complex (K, 9, Nx, Ny) array in the layout of ``eps_cross`` ((9, Nx, Ny): K = 1; diagonal problems read
    xx, yy, zz, tensorial ones with ``left_solve=True`` all nine), or for a ``section`` a sequence of K dicts
    ``{Medium: scalar | 3 numbers | (3, 3) tensor}``, the change of each named medium's eps (others: 0), rasterised on the device
    like its permittivity.  Problems that pass the same array object share one upload.  Each kind takes the solves of the map
    kind it contracts, not its map, and adds (K, M) arrays to the info dict: ``"pert"`` ``dn_dpert``, d(n_eff + i k_eff) per unit
    amplitude of delta eps_k; ``"group_pert"`` (implies ``"pert"`` and ``"freq2"``) ``d2n_dfreq_dpert`` (1/Hz) and ``dng_dpert`` =
    Re ``dn_dpert`` + f Re ``d2n_dfreq_dpert``, the response of ``n_group`` (also for a complex delta eps); ``"disp_pert"``
    (implies ``"group_pert"`` and ``"freq4"``) ``d2n_dfreq2_dpert`` (1/Hz^2) and ``dispersion_dpert`` (ps/(nm km) per unit
    amplitude, ``plugin.dispersion_gradient_of``).  Every response is taken at fixed PML stretch, mu, d eps / df and
    d^2 eps / df^2: a perturbation of the material dispersion itself is not modelled.  Scope and NaNs follow the contracted map:
    ``"group_pert"`` and ``"disp_pert"`` raise on tensorial problems, ``"pert"`` needs ``left_solve=True`` there.  Problems without
    ``eps_pert`` get none of these keys; maps and contractions may be asked for together.
    """
    post = tuple(post or ())
    unknown = set(post) - {"gauge", "normalize", "flux", "overlaps"}
    if unknown:
        raise ValueError(f"unknown post-processing step(s): {sorted(unknown)}")
    derivatives = tuple(derivatives or ())
    unknown = set(derivatives) - {"freq", "eps", "freq2", "group_eps", "freq3", "freq4", "disp_eps", "pert", "group_pert", "disp_pert"}
    if unknown:
        raise ValueError(f"unknown derivative(s): {sorted(unknown)}")
    has_pert = [p.get("eps_pert") is not None for p in problems]
    if any(has_pert) and not {"pert", "group_pert", "disp_pert"} & set(derivatives):
        raise ValueError("eps_pert is read by derivatives=(\"pert\",), (\"group_pert\",) or (\"disp_pert\",): ask for one of them")
    if {"pert", "group_pert", "disp_pert"} & set(derivatives) and not any(has_pert):
        raise ValueError("derivatives \"pert\", \"group_pert\" and \"disp_pert\" contract against eps_pert: no problem gives it")
    disp_pert = "disp_pert" in derivatives
    if disp_pert:
        derivatives = derivatives + tuple(d for d in ("group_pert", "freq4") if d not in derivatives)
    group_pert = "group_pert" in derivatives
    if group_pert:
        derivatives = derivatives + tuple(d for d in ("pert", "freq2") if d not in derivatives)
    want_pert = "pert" in derivatives
    if left_solve and not derivatives:
        raise ValueError("left_solve=True serves derivatives=(\"freq\", \"eps\") of tensorial problems: ask for derivatives as well")
    disp_eps = "disp_eps" in derivatives
    if disp_eps:
        derivatives = derivatives + tuple(d for d in ("group_eps", "freq4") if d not in derivatives)
    group_eps = "group_eps" in derivatives
    if group_eps:
        derivatives = derivatives + tuple(d for d in ("eps", "freq2") if d not in derivatives)
    fourth = "freq4" in derivatives
    if fourth and "freq3" not in derivatives:
        derivatives = derivatives + ("freq3",)
    third = "freq3" in derivatives
    if third and "freq2" not in derivatives:
        derivatives = derivatives + ("freq2",)
    second = "freq2" in derivatives
    if second and "freq" not in derivatives:
        derivatives = derivatives + ("freq",)
    post_flags = (1 if "gauge" in post else 0) | (2 if "normalize" in post else 0)
    packed, cache, pcache = [], {}, {}
    for p in problems:
        split = p.get("split_curl_scaling")
        target_override = None
        if split is not None and getattr(p["mode_spec"], "target_neff", None) is None and not isinstance(p.get("eps_cross"), np.ndarray):
            # solver.py:204-207: the default target comes from `eps_cross` as passed; for a list/tuple input that is the
            # permittivity BEFORE the split-curl division (format_medium_data copies, solver.py:900)
            ec = np.array([np.asarray(c) for c in p["eps_cross"]])
            target_override = float(np.sqrt(np.max(np.abs(ec[np.abs(ec) < abs(PEC_VAL)]))))
        if split is not None and p.get("solver_basis_fields") is not None:
            raise RuntimeError("Split curl not yet implemented for relative mode solver.")  # solver.py:938
        section = p.get("section")
        if section is not None and (split is not None or p.get("eps_cross") is not None):
            raise ValueError("give either 'eps_cross' or 'section' (a section cannot be combined with split_curl_scaling)")
        key = id(p.get("eps_cross"))
        eps_in = None if section is not None else (_apply_split_curl(p["eps_cross"], split) if split is not None else p["eps_cross"])
        pk = _cabi.PackedProblem(
            eps_in, p["coords"], p["freq"], p["mode_spec"], p.get("symmetry", (0, 0)), p.get("direction", "+"),
            eps_packed=None if (split is not None or section is not None) else cache.get(key), basis_fields=p.get("solver_basis_fields"),
            section=section,
            mu_cross=p.get("mu_cross"), target_override=target_override,
            incidence=(split is not None or p.get("mu_cross") is not None),  # solver.py:93
            post=post_flags, grid_correction=p.get("grid_correction"), plane_bounds=p.get("plane_bounds"),
            eps_dfreq=p.get("eps_dfreq"), derivatives="freq" in derivatives, eps_d2freq=p.get("eps_d2freq"), second=second,
            eps_d3freq=p.get("eps_d3freq"), third=third, left_solve=left_solve, eps_d4freq=p.get("eps_d4freq"), fourth=fourth,
            eps_pert=p.get("eps_pert"), eps_pert_packed=None if section is not None else pcache.get(id(p.get("eps_pert"))),
        )  # fmt: skip
        if pk.eps_pert is not None:  # problems that pass the same eps_pert object share one array (one device copy)
            pcache[id(p["eps_pert"])] = pk.eps_pert
        if split is None and section is None:
            cache[key] = pk.eps
        if section is None and key in cache and len(packed) and packed[-1].eps is pk.eps:
            # share the coordinate arrays too so the library can detect identical cross-sections
            prev = packed[-1]
            if np.array_equal(prev.cx, pk.cx) and np.array_equal(prev.cy, pk.cy):
                pk.cx, pk.cy = prev.cx, prev.cy
                pk.struct.coords_x, pk.struct.coords_y = prev.struct.coords_x, prev.struct.coords_y
        packed.append(pk)
    h = handle or get_handle(device)  # after input validation: argument errors do not need a GPU
    with h.lock:
        want_eps = "eps" in derivatives
        dkw = dict(want_dfreq="freq" in derivatives, want_deps=want_eps and not left_solve, want_deps_tensor=want_eps and left_solve,
                   want_d2freq=second, want_group_eps=group_eps, want_d3freq=third, want_d4freq=fourth,
                   want_d2freq2_deps=disp_eps, want_pert=want_pert, want_group_pert=group_pert, want_disp_pert=disp_pert) if derivatives else {}
        rc, fields, ncs, results = h.solve_batch(packed, want_fields, fields_ptrs, want_flux=("flux" in post or "normalize" in post),
                                                 want_overlaps="overlaps" in post, **dkw)
        flux_out, te_out, ov_out = h.last_flux, h.last_te, h.last_overlaps
        dfreq_out, deps_out = (h.last_dn_dfreq, h.last_dn_deps) if derivatives else ([], [])
        d2_out, d2res_out = (h.last_d2n_dfreq2, h.last_d2n_residual) if second else ([], [])
        gmap_out = h.last_d2n_dfreq_deps if group_eps else []
        d3_out = h.last_d3n_dfreq3 if third else []
        d4_out, d4res_out = (h.last_d4n_dfreq4, h.last_d4n_residual) if fourth else ([], [])
        dmap_out = h.last_d2n_dfreq2_deps if disp_eps else []
        pert_out = (h.last_dn_dpert, h.last_d2n_dfreq_dpert, h.last_d2n_dfreq2_dpert) if want_pert else ([], [], [])
        err = h.last_error() if rc != _cabi.OK else ""
    if rc != _cabi.OK:
        bad = [i for i in range(len(packed)) if results[i].status != _cabi.OK]
        _raise_for(rc, h, f"(problems {bad[:8]})", err)
    out, infos = [], []
    for i, pk in enumerate(packed):
        f = fields[i] if fields is not None else None
        if f is not None and problems[i].get("split_curl_scaling") is not None:
            f = _undo_split_curl(f, problems[i]["split_curl_scaling"])
        out.append((f, ncs[i], _cabi.SPEC_NAMES[results[i].eps_spec]))
        r = results[i]
        infos.append(
            dict(converged=r.converged, restarts=r.outer_iters, op_applies=r.op_applies, inner_iters=r.inner_iters,
                 stencil_applies=r.stencil_applies, is_complex=bool(r.is_complex), solve_ms=r.solve_ms, total_ms=r.total_ms,
                 max_residual=r.max_residual, left_paired=r.left_paired)
        )  # fmt: skip
        if flux_out:
            infos[-1]["flux"] = flux_out[i]
            infos[-1]["te_fraction"] = te_out[i]
        if ov_out:
            infos[-1]["overlap_prev"] = ov_out[i]
        if dfreq_out:
            infos[-1]["dn_dfreq"] = dfreq_out[i]
            infos[-1]["n_group"] = ncs[i].real + float(packed[i].struct.freq) * dfreq_out[i].real
        if deps_out:
            # with left_solve the nine-row layout was asked for: diagonal problems report their xx / yy / zz rows
            infos[-1]["dn_deps"] = deps_out[i][[0, 4, 8]] if (left_solve and r.eps_spec == 0) else deps_out[i]
        if d2_out:
            from .plugin import dispersion_of  # noqa: PLC0415  (plugin imports this module)

            infos[-1]["d2n_dfreq2"] = d2_out[i]
            infos[-1]["d2n_residual"] = d2res_out[i]
            infos[-1]["dispersion"] = dispersion_of(float(packed[i].struct.freq), dfreq_out[i], d2_out[i])
        if gmap_out:
            infos[-1]["d2n_dfreq_deps"] = gmap_out[i]
            infos[-1]["dng_deps"] = infos[-1]["dn_deps"].real + float(packed[i].struct.freq) * gmap_out[i].real
        if d3_out:
            from .plugin import beta3_of, dispersion_slope_of  # noqa: PLC0415  (plugin imports this module)

            fq = float(packed[i].struct.freq)
            infos[-1]["d3n_dfreq3"] = d3_out[i]
            infos[-1]["dispersion_slope"] = dispersion_slope_of(fq, dfreq_out[i], d2_out[i], d3_out[i])
            infos[-1]["beta3"] = beta3_of(fq, d2_out[i], d3_out[i])
        if d4_out:
            from .plugin import beta4_of  # noqa: PLC0415  (plugin imports this module)

            infos[-1]["d4n_dfreq4"] = d4_out[i]
            infos[-1]["d4n_residual"] = d4res_out[i]
            infos[-1]["beta4"] = beta4_of(float(packed[i].struct.freq), d3_out[i], d4_out[i])
        if dmap_out:
            from .plugin import dispersion_gradient_of  # noqa: PLC0415  (plugin imports this module)

            infos[-1]["d2n_dfreq2_deps"] = dmap_out[i]
            infos[-1]["dispersion_deps"] = dispersion_gradient_of(float(packed[i].struct.freq), gmap_out[i], dmap_out[i])
        if pert_out[0] and pert_out[0][i] is not None:
            fq = float(packed[i].struct.freq)
            infos[-1]["dn_dpert"] = pert_out[0][i]
            if group_pert:
                infos[-1]["d2n_dfreq_dpert"] = pert_out[1][i]
                infos[-1]["dng_dpert"] = pert_out[0][i].real + fq * pert_out[1][i].real
            if disp_pert:
                from .plugin import dispersion_gradient_of  # noqa: PLC0415  (plugin imports this module)

                infos[-1]["d2n_dfreq2_dpert"] = pert_out[2][i]
                infos[-1]["dispersion_dpert"] = dispersion_gradient_of(fq, pert_out[1][i], pert_out[2][i])
    return (out, infos) if return_info else out


def compute_modes(
    eps_cross,
    coords,
    freq,
    mode_spec,
    mu_cross=None,
    split_curl_scaling=None,
    symmetry=(0, 0),
    direction="+",
    solver_basis_fields=None,
    handle=None,
) -> Tuple[np.ndarray, np.ndarray, str]:
    """Drop-in for ``tidy3d.plugins.mode.solver.compute_modes`` (solver.py:941).  ``handle`` (not in the reference
    signature) selects a solver handle, e.g. ``get_handle(tolerance="tight")``."""
    return compute_modes_batch(
        [dict(eps_cross=eps_cross, coords=coords, freq=freq, mode_spec=mode_spec, symmetry=symmetry, direction=direction,
              solver_basis_fields=solver_basis_fields, mu_cross=mu_cross, split_curl_scaling=split_curl_scaling)],
        handle=handle,
    )[0]
