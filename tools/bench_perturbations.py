"""Perturbation responses against the permittivity-gradient maps they contract, on the headline workload (Si strip 512x512,
4 modes), alternated in one process:
  eps / pert / pert4                   -- derivatives=("eps",) against ("pert",) with K = 1 and K = 4 perturbation fields;
  group_eps / group_pert / group_pert4 -- ("group_eps",) against ("group_pert",), K = 1 and 4;
  disp_eps / disp_pert / disp_pert4    -- ("disp_eps",) against ("disp_pert",), K = 1 and 4.
The perturbations are one field shared by the sweep (the same array object): the core's diagonal, then for K = 4 the cladding,
a complex core change and a zz-only change.  Prints one JSON line: the device time per problem of every arm (b200ms_get_stats),
the bytes each arm delivers to the host per problem beyond n_complex (maps: 3 Nx Ny M complex128 each; responses: K M complex128
each), the largest difference between the K = 1 responses and einsum over the same run's maps, with the card name and power
limit read in the same run.

    python tools/bench_perturbations.py [--nf 8] [--rounds 2] [--n 512] [--out results/bench_perturbations.json]
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
    ap.add_argument("--nf", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.solver import compute_modes_batch, get_handle

    wl = W.headline(nf=a.nf, n=a.n)
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    core = eps[0].real > 5
    pert = np.zeros((4, 9) + core.shape, complex)
    for c in (0, 4, 8):
        pert[0, c] = core
        pert[1, c] = ~core
        pert[2, c] = (1 + 0.1j) * core
    pert[3, 8] = core
    p1 = np.ascontiguousarray(pert[:1])
    h = get_handle()

    def run(kinds, ep=None):
        probs = [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in wl.freqs]
        if ep is not None:
            for p in probs:
                p["eps_pert"] = ep
        return compute_modes_batch(probs, handle=h, want_fields=False, return_info=True, derivatives=kinds)

    arms = {
        "eps": lambda: run(("eps",)), "pert": lambda: run(("pert",), p1), "pert4": lambda: run(("pert",), pert),
        "group_eps": lambda: run(("group_eps",)), "group_pert": lambda: run(("group_pert",), p1), "group_pert4": lambda: run(("group_pert",), pert),
        "disp_eps": lambda: run(("disp_eps",)), "disp_pert": lambda: run(("disp_pert",), p1), "disp_pert4": lambda: run(("disp_pert",), pert),
    }  # fmt: skip
    for fn in arms.values():  # warm-up of every shape
        fn()
    dev = {k: [] for k in arms}
    wall = {k: [] for k in arms}
    last = {}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, infos = fn()
            torch.cuda.synchronize()
            wall[k].append(time.perf_counter() - t0)
            dev[k].append(h.last_stats()["device_ms"])
            last[k] = infos
    N, M = a.n * a.n, wl.mode_spec.num_modes
    mapb = 3 * N * M * 16
    delivered = {"eps": mapb, "group_eps": 2 * mapb, "disp_eps": 3 * mapb, "pert": 16 * M, "pert4": 4 * 16 * M, "group_pert": 2 * 16 * M,
                 "group_pert4": 2 * 4 * 16 * M, "disp_pert": 3 * 16 * M, "disp_pert4": 3 * 4 * 16 * M}  # fmt: skip
    # the K = 1 responses against einsum over the maps of the same run (same solves: the eigen-solve does not depend on the kind)
    diag = p1[0][[0, 4, 8]]
    err = {}
    for mk, pk, key, mkey in (("eps", "pert", "dn_dpert", "dn_deps"), ("group_eps", "group_pert", "d2n_dfreq_dpert", "d2n_dfreq_deps"),
                              ("disp_eps", "disp_pert", "d2n_dfreq2_dpert", "d2n_dfreq2_deps")):
        e = 0.0
        for im, ip in zip(last[mk], last[pk]):
            want = np.einsum("axym,axy->m", im[mkey], diag)
            scale = np.einsum("axym,axy->m", np.abs(im[mkey]), np.abs(diag))
            e = max(e, float(np.max(np.abs(ip[key][0] - want) / scale)))
        err[key] = e
    ms = {k: float(np.median(v)) / a.nf for k, v in dev.items()}
    res = dict(
        card=card(), workload=f"headline {a.n}x{a.n}, {M} modes, {a.nf} frequencies", rounds=a.rounds,
        device_ms_per_problem=ms,
        wall_ms_per_problem={k: 1e3 * float(np.median(v)) / a.nf for k, v in wall.items()},
        contraction_minus_map_device_ms_per_problem={"pert": ms["pert"] - ms["eps"], "group_pert": ms["group_pert"] - ms["group_eps"],
                                                     "disp_pert": ms["disp_pert"] - ms["disp_eps"]},
        k4_minus_k1_device_ms_per_problem={"pert": ms["pert4"] - ms["pert"], "group_pert": ms["group_pert4"] - ms["group_pert"],
                                           "disp_pert": ms["disp_pert4"] - ms["disp_pert"]},
        bytes_to_host_per_problem=delivered,
        max_rel_err_k1_vs_einsum_of_maps=err,
    )  # fmt: skip
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
