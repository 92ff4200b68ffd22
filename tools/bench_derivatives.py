"""Group index and dispersion on the headline workload (Si strip 512x512, 4 modes), alternated in one process:
  plain        -- one solve per frequency, no derivatives;
  analytic     -- one solve per frequency with derivatives=("freq",) (n_group from the left eigenvector);
  analytic_gvd -- one solve per frequency with derivatives=("freq2",) (n_group and the dispersion, one correction solve per mode);
  gvd_eps      -- derivatives=("eps", "freq2"): the dispersion pass plus the first-order permittivity map;
  group_eps    -- derivatives=("group_eps",): the same plus the group-index gradient map from the same correction solves;
  analytic_tod -- derivatives=("freq3",): the dispersion pass plus the third-order dispersion from the same correction solves;
  analytic_fod -- derivatives=("freq4",): the same plus the fourth-order dispersion from one more correction solve per mode;
  fod_group_eps -- derivatives=("freq4", "group_eps"): the fourth-order pass together with the group-index gradient map;
  disp_eps     -- derivatives=("disp_eps",): the same plus the dispersion gradient map from the corrections of both passes;
  fd3          -- three solves per frequency at f(1 -/+ step) and f, n_group and dispersion by plugin.group_index (the reference's path).
Prints one JSON line: solves/s, frequencies-with-group-index/s, frequencies-with-dispersion/s, the device time the derivative
and dispersion passes add per problem, the time the group-index gradient map adds per problem (group_eps - gvd_eps), the time the third-order terms add per
problem (analytic_tod - analytic_gvd), the time the fourth-order terms add per problem (analytic_fod - analytic_tod) and the
inner iterations of their second-order correction solves per mode, the time the dispersion gradient map adds per problem
(disp_eps - fod_group_eps), the correction solves' inner iterations per mode, the largest differences against fd3 and
the derivative pass's algorithmic bytes against the 3.35 TB/s HBM3 data-sheet figure, with the card name and power limit read
in the same run.

    python tools/bench_derivatives.py [--nf 64] [--rounds 2] [--n 512] [--out results/bench_derivatives.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nf", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--step", type=float, default=1e-3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    from tidy3d_b200 import plugin
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.solver import compute_modes_batch, get_handle

    wl = W.headline(nf=a.nf, n=a.n)
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    h = get_handle()

    def probs(freqs):
        return [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in freqs]

    f3 = np.outer(wl.freqs, (1 - a.step, 1, 1 + a.step)).ravel()
    arms = {
        "plain": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True),
        "analytic": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("freq",)),
        "analytic_gvd": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("freq2",)),
        "gvd_eps": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("eps", "freq2")),
        "group_eps": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("group_eps",)),
        "analytic_tod": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("freq3",)),
        "analytic_fod": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("freq4",)),
        "fod_group_eps": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("freq4", "group_eps")),
        "disp_eps": lambda: compute_modes_batch(probs(wl.freqs), handle=h, want_fields=False, return_info=True, derivatives=("disp_eps",)),
        "fd3": lambda: compute_modes_batch(probs(f3), handle=h, want_fields=False, return_info=True),
    }
    for fn in arms.values():  # warm-up of every shape
        fn()
    t = {k: [] for k in arms}
    dev = {k: [] for k in arms}
    ng, disp = {}, {}
    inner = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out, infos = fn()
            torch.cuda.synchronize()
            t[k].append(time.perf_counter() - t0)
            dev[k].append(h.last_stats()["device_ms"])
            inner[k].append(h.last_stats()["inner_iters"])
            if k == "analytic":
                ng["analytic"] = np.array([i["n_group"] for i in infos])
            if k == "analytic_gvd":
                disp["analytic_gvd"] = np.array([i["dispersion"] for i in infos])
                res_gvd = np.array([i["d2n_residual"] for i in infos])
            if k == "group_eps":
                gmap_finite = all(np.isfinite(i["d2n_dfreq_deps"]).all() for i in infos)
            if k == "analytic_tod":
                tod_finite = all(np.isfinite(i["d3n_dfreq3"]).all() for i in infos)
                slope = np.array([i["dispersion_slope"] for i in infos])
                b3 = np.array([i["beta3"] for i in infos])
            if k == "analytic_fod":
                fod_finite = all(np.isfinite(i["d4n_dfreq4"]).all() for i in infos)
                b4 = np.array([i["beta4"] for i in infos])
                res_fod = np.array([i["d4n_residual"] for i in infos])
            if k == "disp_eps":
                dmap_finite = all(np.isfinite(i["d2n_dfreq2_deps"]).all() for i in infos)
            if k == "fd3":
                _, _, ng["fd3"], disp["fd3"] = plugin.group_index(np.array([o[1] for o in out]), f3, a.step)
    nsolve = {"plain": a.nf, "analytic": a.nf, "analytic_gvd": a.nf, "gvd_eps": a.nf, "group_eps": a.nf, "analytic_tod": a.nf, "analytic_fod": a.nf, "fod_group_eps": a.nf, "disp_eps": a.nf,
              "fd3": 3 * a.nf}
    N, M = a.n * a.n, wl.mode_spec.num_modes
    # one derivative pass reads, per (problem, mode), the real fp64 Ritz vector (2N x 8 B) and the three coefficient fields
    # (exx, eyy, 1/ezz: 3N x 8 B; shared by the sweep, counted once per mode pass as they are re-read)
    bytes_pass = a.nf * M * (2 * N * 8 + 3 * N * 8)
    extra_ms = (np.median(dev["analytic"]) - np.median(dev["plain"]))
    gvd_ms = (np.median(dev["analytic_gvd"]) - np.median(dev["analytic"]))
    gmap_ms = (np.median(dev["group_eps"]) - np.median(dev["gvd_eps"]))
    tod_ms = (np.median(dev["analytic_tod"]) - np.median(dev["analytic_gvd"]))
    fod_ms = (np.median(dev["analytic_fod"]) - np.median(dev["analytic_tod"]))
    dmap_ms = (np.median(dev["disp_eps"]) - np.median(dev["fod_group_eps"]))
    # the eigen-solves of the two arms are bit-identical, so the difference of the summed inner iterations is the correction
    # solves' (per problem: the slowest problem of its device batch, as for the eigen-solve's own counters)
    corr_iters = (np.median(inner["analytic_gvd"]) - np.median(inner["analytic"])) / (a.nf * M)
    corr2_iters = (np.median(inner["analytic_fod"]) - np.median(inner["analytic_tod"])) / (a.nf * M)
    res = dict(
        card=card(), workload=f"headline {a.n}x{a.n}, {M} modes, {a.nf} frequencies", rounds=a.rounds,
        solves_per_s={k: nsolve[k] / float(np.median(v)) for k, v in t.items()},
        freqs_with_group_index_per_s={"analytic": a.nf / float(np.median(t["analytic"])), "fd3": a.nf / float(np.median(t["fd3"]))},
        freqs_with_dispersion_per_s={"analytic_gvd": a.nf / float(np.median(t["analytic_gvd"])), "fd3": a.nf / float(np.median(t["fd3"]))},
        device_ms_median={k: float(np.median(v)) for k, v in dev.items()},
        derivative_pass_device_ms_per_problem=float(extra_ms / a.nf),
        dispersion_pass_device_ms_per_problem=float(gvd_ms / a.nf),
        group_gradient_map_device_ms_per_problem=float(gmap_ms / a.nf), group_gradient_map_finite=bool(gmap_finite),
        third_order_device_ms_per_problem=float(tod_ms / a.nf), third_order_finite=bool(tod_finite),
        dispersion_slope_range_ps_per_nm2_km=[float(slope.min()), float(slope.max())],
        beta3_range_ps3_per_km=[float(b3.min()), float(b3.max())],
        fourth_order_device_ms_per_problem=float(fod_ms / a.nf), fourth_order_finite=bool(fod_finite),
        beta4_range_ps4_per_km=[float(b4.min()), float(b4.max())],
        dispersion_gradient_map_device_ms_per_problem=float(dmap_ms / a.nf), dispersion_gradient_map_finite=bool(dmap_finite),
        second_correction_inner_iters_per_mode=float(corr2_iters), second_correction_residual_max=float(res_fod.max()),
        correction_inner_iters_per_mode=float(corr_iters),
        correction_residual_max=float(res_gvd.max()),
        derivative_pass_bytes=bytes_pass,
        derivative_pass_bw_TBps=float(bytes_pass / max(extra_ms, 1e-9) / 1e9),
        hbm_datasheet_TBps=3.35,
        n_group_max_abs_diff_analytic_vs_fd3=float(np.abs(ng["analytic"] - ng["fd3"]).max()),
        dispersion_max_abs_diff_analytic_gvd_vs_fd3_ps_per_nm_km=float(np.abs(disp["analytic_gvd"] - disp["fd3"]).max()),
        dispersion_range_fd3_ps_per_nm_km=[float(disp["fd3"].min()), float(disp["fd3"].max())],
    )  # fmt: skip
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
