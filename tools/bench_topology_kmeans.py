"""Times yams_b200_topology_kmeans, the k-means topology engine's clustering, on synthetic clustered rows with k auto
(round(sqrt(n))): 100 k and 1 M x 768 fp16 and 200 k x 768 fp32.  Prints one JSON line per shape with the card, the wall time
of the synchronous call (median of 3 after a warm-up), the device split between init, assignment and update, the iterations,
the init's HBM-bound floor, and the reference restatement's time on a subsample, extrapolated by n * k."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import yams_b200 as Y  # noqa: E402
from tests import topology_kmeans_restated as T  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def clustered(seed, n, d, n_centers=1000):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((n_centers, d)).astype(np.float32)
    out = np.empty((n, d), dtype=np.float32)
    for s in range(0, n, 65536):
        e = min(n, s + 65536)
        out[s:e] = centers[rng.integers(0, n_centers, e - s)] + np.float32(0.5) * rng.standard_normal((e - s, d)).astype(np.float32)
    return out


def run(n, d, dtype, oracle_n, iters):
    x = clustered(n, n, d)
    c = Y.Corpus(d, dtype, Y.COSINE)
    c.append(x.astype(np.float16) if dtype == Y.F16 else x)
    c.topology_kmeans(0, iters)   # warm-up
    walls, timings = [], []
    for _ in range(3):
        t0 = time.perf_counter()
        asg, _, k, it = c.topology_kmeans(0, iters)
        walls.append((time.perf_counter() - t0) * 1e3)
        timings.append(c.topology_kmeans_last_timings())
    c.close()
    i = int(np.argsort(walls)[1])
    elem = 2 if dtype == Y.F16 else 4
    init_bytes = float(k) * n * d * elem
    res = {"card": card(), "n": n, "d": d, "dtype": "fp16" if dtype == Y.F16 else "fp32", "k": k, "iterations": it,
           "wall_ms_median": round(walls[i], 2), "init_ms": round(timings[i]["init_ms"], 2),
           "assign_ms": round(timings[i]["assign_ms"], 2), "update_ms": round(timings[i]["update_ms"], 2), "init_hbm_floor_ms": round(init_bytes / HBM_BYTES_PER_S * 1e3, 2)}
    if oracle_n:
        sub = (x[:oracle_n].astype(np.float16).astype(np.float32) if dtype == Y.F16 else x[:oracle_n])
        t0 = time.perf_counter()
        _, _, ks, its = T.kmeans(sub, 0, iters)
        o_ms = (time.perf_counter() - t0) * 1e3
        # the work scales with n * k (init and every iteration); the subsample may stop after a different number of rounds
        scale = (n * k * (it + 1)) / (oracle_n * ks * (its + 1))
        res.update({"oracle_subsample_n": oracle_n, "oracle_subsample_ms": round(o_ms, 1),
                    "oracle_extrapolated_ms": round(o_ms * scale, 0), "oracle_threads": os.cpu_count(),
                    "oracle_note": "restatement (OpenMP over documents) on a subsample, extrapolated by n*k*(rounds+1)"})
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=0, help="max_iterations (0 = 10, the reference default)")
    ap.add_argument("--oracle-n", type=int, default=20_000)
    ap.add_argument("--shapes", default="100000:f16,1000000:f16,200000:f32")
    a = ap.parse_args()
    assert Y.device_count() > 0, "needs a GPU"
    for s in a.shapes.split(","):
        n, t = s.split(":")
        run(int(n), 768, Y.F16 if t == "f16" else Y.F32, a.oracle_n, a.iters)


if __name__ == "__main__":
    main()
