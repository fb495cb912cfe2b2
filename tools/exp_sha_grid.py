"""Ingest throughput and stage times at several segment sizes.  EXP_GIB sets the stream size."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GIB = int(os.environ.get("EXP_GIB", "16"))
code = r'''
import sys, torch, hashlib
sys.path.insert(0, %r)
import yams_b200 as Y
assert Y.plugin_init() == 0
n = %d << 30
buf = torch.empty(n, dtype=torch.uint8, device="cuda")
Y.synth_bytes_device(12345, 0, n, buf.data_ptr())
best = None
for _ in range(4):
    ch = Y.chunk_and_hash_device(buf.data_ptr(), n, Y.default_config())
    t = Y.ingest_last_timings()
    if best is None or t["total_ms"] < best["total_ms"]: best = t
h = hashlib.sha256()
for c in ch[:20000]: h.update(bytes(c["digest"]))
h.update(bytes(ch[-1]["digest"])); h.update(str(len(ch)).encode())
t = best
print("total %%.2f ms = %%.0f GB/s ; sha256(tail) %%.2f scan %%.2f select %%.2f ; table %%s" %% (t["total_ms"], n / t["total_ms"] / 1e6, t["sha256_ms"], t["scan_ms"], t["select_ms"], h.hexdigest()[:12]))
''' % (ROOT, GIB)
CASES = [
    {},
    {"YAMS_B200_SEGMENT_MIB": "8192"},
    {"YAMS_B200_SEGMENT_MIB": "16384"},
    {"YAMS_B200_SEGMENT_MIB": "2048"},
]
for extra in CASES:
    env = dict(os.environ)
    env.update(extra)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    print(" ".join("%s=%s" % (k.replace("YAMS_B200_", ""), v) for k, v in extra.items()) or "default", "|",
          out.stdout.strip() or out.stderr[-400:], flush=True)
