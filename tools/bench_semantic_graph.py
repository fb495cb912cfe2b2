"""The semantic-neighbour graph (yams_b200_semantic_neighbors) over whole corpora: every row a source, k = 8, adaptive mode
(threshold FLT_TRUE_MIN), the daemon's default graph.
  c5-f16   1M x 768 fp16 synthetic rows (the C5 corpus generator), the fp16 wgmma engine;
  f32      200k x 768 fp32 synthetic rows, the tf32 wgmma engine (the daemon's own float values);
  f16-tiny 100k x 768 fp16 synthetic rows plus ONE row of norm ~1e-5 (fp16 subnormal elements): the fp16 engine's error bound
           grows with the largest 1/|r| of the graph's rows (DESIGN.md §4.9), so most sources go to the exhaustive level 1.
Per case: wall time around the synchronous call (median of 3 after a warm-up), the batches of 1024 sources, the sources flagged
FALLBACK_PATH, and the whole-call rate 2 S N d / t -- a whole-call figure set against the data-sheet dense peaks (989 TFLOP/s
fp16, 495 tf32), not a kernel's share of peak.  Parity: 32 sources against the C restatement of the reference loop, whose time
for them is extrapolated to the whole graph (labelled as such).  Prints the card, its power limit and one JSON line per case.
Usage: python tools/bench_semantic_graph.py [--cases c5-f16,f32,f16-tiny] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import yams_b200 as Y
from oracle import oracle as O
from tests import semantic_restated as S

D, K, SEED, PARITY = 768, 8, 42, 32
CASES = {"c5-f16": (1_000_000, Y.F16, 989.0, False), "f32": (200_000, Y.F32, 495.0, False), "f16-tiny": (100_000, Y.F16, 989.0, True)}
TINY = 1e-5   # norm of the f16-tiny case's extra row


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def tiny_row():
    v = O.gen_rows_f32(SEED + 1, 0, 1, D)[0] * np.float32(TINY)
    return v.astype(np.float16)


def host_rows(n, dtype, tiny):
    """the synthetic rows append_synthetic writes (and the tiny row), as the fp32 values the corpus holds"""
    x = np.empty((n + tiny, D), dtype=np.float32)
    if tiny:
        x[n] = tiny_row().astype(np.float32)
    for a in range(0, n, 100_000):
        b = min(n, a + 100_000)
        part = O.gen_rows_f32(SEED, a, b - a, D)
        x[a:b] = O.f16_from_float(part).view(np.float16).astype(np.float32) if dtype == Y.F16 else part
    return x


def run(name, reps):
    n, dtype, peak, tiny = CASES[name]
    c = Y.Corpus(D, dtype, Y.COSINE, n + tiny)
    c.append_synthetic(SEED, 0, n)
    if tiny:
        c.append(tiny_row()[None, :], np.array([n], dtype=np.int64))
    c.semantic_neighbors(K)                       # warm-up: every shape the timed calls use
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r, s, cnt, flags = c.semantic_neighbors(K)
        ts.append(time.perf_counter() - t0)
    t = float(np.median(ts))
    x = host_rows(n, dtype, tiny)
    src = np.sort(np.random.default_rng(7).choice(n, PARITY, replace=False))
    t0 = time.perf_counter()
    wr, ws, wc, _ = S.semantic_neighbors(x, K, None, src)
    t_oracle = time.perf_counter() - t0
    parity = bool(np.array_equal(cnt[src], wc) and np.array_equal(r[src], wr) and np.array_equal(s[src].view(np.uint32), ws.view(np.uint32)))
    n += tiny
    flops = 2.0 * n * n * D
    line = {"case": name, "rows": n, "dim": D, "dtype": "f16" if dtype == Y.F16 else "f32", "k": K, "threshold": "adaptive",
            "sources": n, "batches": (n + 1023) // 1024, "wall_ms_median": round(t * 1e3, 1), "wall_ms_all": [round(v * 1e3, 1) for v in ts],
            "fallback_sources": int(((flags & Y.FLAG_FALLBACK_PATH) != 0).sum()), "neighbors_total": int(cnt.sum()),
            "whole_call_tflops": round(flops / t / 1e12, 1), "datasheet_peak_tflops": peak,
            "whole_call_share_of_datasheet_peak": round(flops / t / 1e12 / peak, 3),
            "parity_sources": PARITY, "parity_ok": parity, "oracle_s_for_parity_sources": round(t_oracle, 2),
            "oracle_s_whole_graph_extrapolated": round(t_oracle * n / PARITY, 0),
            "oracle_threads": os.cpu_count()}
    c.close()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="c5-f16,f32")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert Y.device_count() > 0, "needs a GPU"
    assert Y.plugin_init() == 0, Y.health()
    print("card:", card())
    for name in a.cases.split(","):
        print(json.dumps(run(name, a.reps)), flush=True)


if __name__ == "__main__":
    main()
