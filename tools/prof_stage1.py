"""Stall split of the wgmma stage-1 scan at the C2 shape (10 M x 768 fp16 rows, 1024 queries, cosine): one pass of the
kernel's profiling instantiation in filter mode over every row, with thresholds that pass about as many rows as the
search's own (the 8th best score of a 64 Ki-row strided sample).

Per CTA the kernel counts the cycles its first consumer warp waited on full barriers (starved for data), the cycles the
producer waited on empty barriers (every stage still held by the tensor cores), the first consumer warp's epilogue cycles
and its total cycles.  Printed as shares of the total, over all CTAs, with the card's name and power limit.

    python tools/prof_stage1.py [rows] [queries] [dim] [--json OUT]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import yams_b200 as Y  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rows", type=int, nargs="?", default=10_000_000)
    ap.add_argument("queries", type=int, nargs="?", default=1024)
    ap.add_argument("dim", type=int, nargs="?", default=768)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    n, nq, d = args.rows, args.queries, args.dim
    assert Y.plugin_init() == 0, Y.health()
    c = Y.Corpus(d, Y.F16, Y.COSINE, capacity_hint=n)
    for r0 in range(0, n, 1_000_000):
        c.append_synthetic(42, r0, min(1_000_000, n - r0))
    q_dev = torch.empty((nq, d), dtype=torch.float32, device="cuda")
    Y.synth_rows_device(43, 0, nq, d, q_dev.data_ptr())
    q = q_dev.cpu().numpy()
    S = min(n, 65536)
    stride = n // S
    sample = c.debug_stage1_scores(q, 1, row_start=0, row_stride=stride, nrows=S)
    tau = np.sort(sample, axis=1)[:, -8].astype(np.float32)
    runs = []
    for _ in range(args.repeat):
        cyc, layout, ms = c.debug_stage1_profile(q, tau, cap=8192)
        tot = cyc[:, 3].astype(np.float64)
        runs.append({"ms": ms, "layout": layout,
                     "full_wait": float(cyc[:, 0].sum() / tot.sum()), "empty_wait": float(cyc[:, 1].sum() / tot.sum()),
                     "epilogue": float(cyc[:, 2].sum() / tot.sum()),
                     "total_cycles_mean": float(tot.mean()), "total_cycles_max": float(tot.max()),
                     "total_cycles_min": float(tot.min())})
    c.close()
    out = {"card": card(), "rows": n, "queries": nq, "dim": d, "runs": runs}
    for r in runs:
        print(f"{r['ms']:8.2f} ms  {r['layout']}  consumer full-wait {r['full_wait']:.3f}  producer empty-wait {r['empty_wait']:.3f}  "
              f"epilogue {r['epilogue']:.3f}  cycles/CTA mean {r['total_cycles_mean']:.3e} (min {r['total_cycles_min']:.3e}, "
              f"max {r['total_cycles_max']:.3e})")
    print("card:", out["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
