import sys, os, time, ctypes
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from rusty_kaspa_b200 import workload as W
pk, msg, sig, kind = W.schnorr_triples(1 << 14, seed=5, n_keys=4096, n_nonces=4096)
pk, msg, sig, kind = W.tile_triples(pk, msg, sig, kind, 1 << 17)
O = ctypes.CDLL(os.path.join(ROOT, "oracle", "libkaspa_oracle.so")); O.ok_secp_init()
vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
out = np.zeros(len(kind), dtype=np.uint8)
print("cpu_count", os.cpu_count(), "cpu.max", open("/sys/fs/cgroup/cpu.max").read().strip() if os.path.exists("/sys/fs/cgroup/cpu.max") else "?")
for th in (8, 16, 24, 32, 48, 64, 128):
    t0 = time.perf_counter()
    O.ok_schnorr_verify_batch(vp(pk), vp(msg), vp(sig), ctypes.c_size_t(len(kind)), vp(out), th)
    dt = time.perf_counter() - t0
    print(th, "threads:", round(len(kind) / dt), "verifies/s")
