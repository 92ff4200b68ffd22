"""Time the post-smoothing half of a level-0 V-cycle at the headline shape: the fused pass (prolongation + two sweeps in one
march, csrc/march2_tma.cuh MODE_PROLONG_JACOBI2) against the separate sequence (prolongation kernel + two stored-diagonal
sweeps), both through b200ms_bench_stencil (modes 3 and 4) on B device-resident copies of the headline operator.

    python tools/post_smooth_bench.py [--n 512] [--batch 64] [--reps 200]

Algorithmic bytes per fine cell (fp32): fused 44 (x_old 8, exx / eyy / 1/ezz 12, rhs 8, omega/diag 8, output 8); separate 104
(prolongation: read + write x 16; each sweep 44); both plus the coarse correction read once (8 B per coarse cell, about 2 B per
fine cell).  The fused pass also reads two halo rows above and below each CTA's rows (re-reads served mostly by L2); they
are not counted.  Prints us per launch, GB/s and the share of the H100 SXM data sheet's 3.35 TB/s, with the card's name and
power limit read in the same run.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    from tidy3d_b200 import _cabi
    from tidy3d_b200 import workloads as W

    wl = W.headline(nf=1, n=args.n)
    pk = _cabi.PackedProblem(wl.eps_cross, wl.coords, wl.freqs[0], wl.mode_spec)
    h = _cabi.Handle()
    print(f"card: {card()}")
    print(f"{args.batch} x {args.n}^2, {args.reps} launches per row")
    try:
        for mode, name in ((3, "fused prolongation + 2 sweeps"), (4, "separate: prolongation + 2 sweeps"), (1, "one stored-diagonal sweep")):
            ms, byts = C.c_double(), C.c_double()
            rc = _cabi.lib().b200ms_bench_stencil(h._h, C.byref(pk.struct), args.batch, mode, args.reps, 0, None, None, C.byref(ms),
                                                  C.byref(byts))
            assert rc == 0, h.last_error()
            gbs = byts.value / (ms.value * 1e-3) / 1e9
            cell = byts.value / (args.batch * pk.nx * pk.ny)
            print(f"{name:36s} {ms.value * 1e3:9.1f} us  {byts.value / 1e9:6.3f} GB ({cell:5.1f} B/cell)  {gbs:7.0f} GB/s  "
                  f"{gbs / HBM_GBS:5.2f} of 3.35 TB/s")
    finally:
        h.close()


if __name__ == "__main__":
    main()
