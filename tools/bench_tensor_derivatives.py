"""Group index of tensorial modes: an angled Si strip (256x256, 4 modes, angle_theta 0.2, 16 frequencies), alternated in one process:
  plain   -- one solve per frequency, no derivatives;
  left    -- one solve per frequency with derivatives=("freq", "eps"), left_solve=True (transposed eigen-solve + derivative pass);
  fd3     -- three solves per frequency at f(1 -/+ step) and f, n_group by plugin.group_index (the reference's path).
Prints one JSON line: frequencies-with-group-index/s of left and fd3, the device time the transposed pass and the derivative
kernels add per problem (left - plain, CUDA events), the forward and transposed op applies and inner iterations per problem, the
largest |n_group(left) - n_group(fd3)|, the pairing figures of the transposed solve (largest |n_L - n| / |n|, smallest |w^T u|,
from the library's verbose output of one extra call), with the card name and power limit read in the same run.

    python tools/bench_tensor_derivatives.py [--nf 16] [--n 256] [--rounds 2] [--out results/bench_tensor_derivatives.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
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
    ap.add_argument("--nf", type=int, default=16)
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--step", type=float, default=1e-3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    from tidy3d_b200 import plugin
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.solver import compute_modes_batch, get_handle

    wl = W.angled(a.n, num_modes=4)
    eps = np.ascontiguousarray(np.stack(wl.eps_cross))
    freqs = W.sweep_freqs(a.nf)
    h = get_handle()

    def probs(fs):
        return [dict(eps_cross=eps, coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec) for f in fs]

    fd_freqs = np.outer(freqs, (1 - a.step, 1, 1 + a.step)).ravel()
    runs = {
        "plain": lambda: compute_modes_batch(probs(freqs), handle=h, want_fields=False, return_info=True),
        "left": lambda: compute_modes_batch(probs(freqs), handle=h, want_fields=False, return_info=True, derivatives=("freq", "eps"), left_solve=True),
        "fd3": lambda: compute_modes_batch(probs(fd_freqs), handle=h, want_fields=False, return_info=True),
    }
    for fn in runs.values():  # warm-up of every shape
        fn()
    wall = {k: [] for k in runs}
    dev = {k: [] for k in runs}
    last = {}
    for _ in range(a.rounds):
        for k, fn in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            last[k] = fn()
            wall[k].append(time.perf_counter() - t0)
            dev[k].append(h.last_stats()["device_ms"])
            print(f"{k}: {wall[k][-1]:.2f} s wall, {dev[k][-1]:.1f} ms device", file=sys.stderr, flush=True)
            if k == "left":
                st_left = h.last_stats()
    res_l, inf_l = last["left"]
    res_fd, _ = last["fd3"]
    _, _, ng_fd, _ = plugin.group_index(np.array([r[1] for r in res_fd]), fd_freqs, a.step)
    ng_l = np.array([i["n_group"] for i in inf_l])
    fwd_ops = np.mean([i["op_applies"] for i in inf_l])
    fwd_inner = np.mean([i["inner_iters"] for i in inf_l])
    # the pairing figures from the library's verbose lines (stderr of the process, captured at the file-descriptor level)
    h.set_options(verbose=1)
    with tempfile.TemporaryFile(mode="w+") as tmp:
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            runs["left"]()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            h.set_options(verbose=0)
        tmp.seek(0)
        log = tmp.read()
    rel = [float(x) for x in re.findall(r"largest \|n_L - n\| / \|n\| (\S+)", log)]
    wu = [float(x) for x in re.findall(r"smallest paired \|w\^T u\| (\S+)", log)]
    out = dict(
        card=card(), n=a.n, modes=4, nf=a.nf, rounds=a.rounds,
        freqs_per_s_left=a.nf / min(wall["left"]), freqs_per_s_fd3=a.nf / min(wall["fd3"]), solves_per_s_plain=a.nf / min(wall["plain"]),
        device_ms_per_problem=dict(plain=min(dev["plain"]) / a.nf, left=min(dev["left"]) / a.nf),
        transposed_pass_device_ms_per_problem=(min(dev["left"]) - min(dev["plain"])) / a.nf,
        forward_op_applies=fwd_ops, forward_inner_iters=fwd_inner,
        transposed_op_applies=st_left["op_applies"] / a.nf - fwd_ops, transposed_inner_iters=st_left["inner_iters"] / a.nf - fwd_inner,
        left_paired=[i["left_paired"] for i in inf_l],
        max_abs_ng_left_vs_fd3=float(np.abs(ng_l - ng_fd).max()),
        pairing_max_rel_dn=max(rel) if rel else None, pairing_min_wtu=min(wu) if wu else None,
    )  # fmt: skip
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
