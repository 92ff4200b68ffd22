"""Per-kernel device-time shares of one warmed headline step, measured with torch.profiler (CUPTI).

    python tools/kernel_shares.py [--sweep 256] [--n 512] [--max-batch 64] [--top 40] [--out DIR]

Builds the problems bench.py builds (one distinct (9,Nx,Ny) eps array per sweep point), runs one step through
``solve_sharded`` to warm every shape, then profiles a second step with CUDA activities.  Kernels replayed from CUDA graphs
are reported by CUPTI one by one like ordinary launches.  Kernels are grouped by name (namespace and parameter list
stripped) and grid, so the levels of the multigrid hierarchy show up as separate rows.  The card's name and power limit
are read in the same run and printed with the table; ``--out`` also writes the table as JSON.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def short_name(name):
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)  # parameter list
    return name.replace("b200ms::", "")


def shares(trace_path):
    ev = json.load(open(trace_path))["traceEvents"]
    tot, cnt = defaultdict(float), defaultdict(int)
    memcpy = defaultdict(lambda: [0.0, 0])
    for e in ev:
        cat = e.get("cat", "")
        if cat == "kernel":
            g = e.get("args", {}).get("grid", "")
            key = f"{short_name(e['name'])}  grid={g}"
            tot[key] += float(e.get("dur", 0.0))
            cnt[key] += 1
        elif cat == "gpu_memcpy" or cat == "gpu_memset":
            m = memcpy[e["name"]]
            m[0] += float(e.get("dur", 0.0))
            m[1] += 1
    return tot, cnt, dict(memcpy)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweep", type=int, default=256)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--max-batch", type=int, default=64)
    ap.add_argument("--top", type=int, default=40)
    ap.add_argument("--out", default=None, help="directory for kernel_shares.json")
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import __graft_entry__ as g

    g.build()
    from tidy3d_b200 import workloads as W
    from tidy3d_b200.sharding import solve_sharded
    from tidy3d_b200.solver import get_handle

    torch.cuda.set_device(0)
    h = get_handle(0, "reference")
    h.set_options(max_batch=args.max_batch)
    wl = W.headline(nf=args.sweep, n=args.n)
    problems = [dict(eps_cross=np.ascontiguousarray(np.stack(wl.eps_cross)), coords=wl.coords, freq=float(f), mode_spec=wl.mode_spec)
                for f in wl.freqs]
    solve_sharded(problems)  # warm-up: module loads, graph capture, every level shape
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        solve_sharded(problems)
        torch.cuda.synchronize()
    st = h.last_stats()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        tot, cnt, mem = shares(path)

    ktot = sum(tot.values())
    mtot = sum(v[0] for v in mem.values())
    dev = ktot + mtot
    info = card()
    print(f"card: {info}")
    print(f"step: {len(problems)} problems of {args.n}x{args.n}, batches of <= {args.max_batch}; last batch: "
          f"{st['inner_iters']} inner iterations, {st['op_applies']} operator applies, device_ms {st['device_ms']:.1f}")
    print(f"kernels {ktot / 1e3:.2f} ms over {sum(cnt.values())} launches; memcpy/memset {mtot / 1e3:.2f} ms")
    rows = []
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        rows.append({"kernel": k, "ms": v / 1e3, "count": cnt[k], "share": v / dev})
    for k, (v, n) in sorted(mem.items(), key=lambda kv: -kv[1][0]):
        rows.append({"kernel": k, "ms": v / 1e3, "count": n, "share": v / dev})
    rows.sort(key=lambda r: -r["ms"])
    for r in rows[: args.top]:
        print(f"{100 * r['share']:6.2f}%  {r['ms']:10.3f} ms  n={r['count']:7d}  avg {1e3 * r['ms'] / r['count']:8.1f} us  {r['kernel'][:140]}")
    dtod = sum(v[0] for k, v in mem.items() if "DtoD" in k)
    print(f"device-to-device memcpy: {dtod / 1e3:.3f} ms ({100 * dtod / dev:.2f} %) over {sum(v[1] for k, v in mem.items() if 'DtoD' in k)} copies")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        json.dump({"card": info, "kernel_ms": ktot / 1e3, "memcpy_ms": mtot / 1e3, "dtod_ms": dtod / 1e3, "rows": rows},
                  open(os.path.join(args.out, "kernel_shares.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
