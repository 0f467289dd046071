#!/usr/bin/env python
"""GPU self-test of the wgmma/TMA GEMM pipeline against fp64 numpy (run under `timeout`)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from ai2bmd_b200.engine import tc_selftest  # noqa: E402

rng = np.random.default_rng(0)
ok = True
for case, (a, w) in {
    "identity": (np.eye(128, dtype=np.float32), rng.normal(size=(128, 128)).astype(np.float32)),
    "rowcol": (np.arange(128 * 128, dtype=np.float32).reshape(128, 128) / 1000.0, np.eye(128, dtype=np.float32)),
    "random": (rng.normal(size=(128, 128)).astype(np.float32), rng.normal(size=(128, 128)).astype(np.float32) * 0.1),
}.items():
    d, ms = tc_selftest(a, w, reps=1)
    ref = a.astype(np.float64) @ w.astype(np.float64).T
    err = np.abs(d - ref).max()
    scale = np.abs(ref).max()
    ref32 = (a @ w.T)
    print(f"{case:9s} maxabs err {err:.3e} (ref scale {scale:.3e}, rel {err / scale:.2e}); fp32 numpy err {np.abs(ref32 - ref).max():.3e}; {ms:.3f} ms")
    if not err / scale < 2e-6:
        ok = False
        bad = np.argwhere(np.abs(d - ref) > 1e-4 * scale)
        print("   first mismatches (row, col):", bad[:8].tolist(), " d:", d[tuple(bad[0])] if len(bad) else None,
              " ref:", ref[tuple(bad[0])] if len(bad) else None)
d, ms = tc_selftest(a, w, reps=200)
print(f"200 reps in one launch: {ms:.3f} ms -> {ms / 200 * 1e3:.2f} us per 128x128x128 3xTF32 GEMM incl. A store + D load")
# tile capacities of <= 64 rows run the three-stage weight ring; 7 reps wrap it with both barrier parities
for rows in (64, 32):
    d, ms = tc_selftest(a, w, reps=7, rows=rows)
    ref = a[:rows].astype(np.float64) @ w.astype(np.float64).T
    rel = np.abs(d - ref).max() / np.abs(ref).max()
    print(f"rows {rows:3d}, 7 reps: rel err {rel:.2e}; {ms:.3f} ms")
    ok = ok and rel < 2e-6
print("SELFTEST", "PASS" if ok else "FAIL")
