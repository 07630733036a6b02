#!/usr/bin/env python
"""Rough cost of the norms' element-order fallback (csrc/matvec.cuh norm_stat): median time of ctb_norm_path calls on rows that
take it (refs.norm_order_rows) against Gaussian rows of the same width that do not.  Each call uploads the row, runs the kernel
and copies the result back, so the difference between the two medians is the fallback's cost; the absolute times are mostly
the call's own overhead.  Host clock around calls that end in a device synchronise.

    python tools/norm_fallback_cost.py
"""
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import refs  # noqa: E402
from ctransformers_b200.lib import load_library  # noqa: E402

lib = load_library()
ptr = refs.ptr
print("path 0: k_matvec's prologue, path 1: one k_step mat-vec phase")
for k in (4096, 11008):
    for mode in (1, 2):
        rows, w, b = refs.norm_order_rows(mode, k, seed=k + mode)
        natural = (np.random.default_rng(0).standard_normal((rows.shape[0], k)) * 3).astype(np.float32)
        y = np.zeros(k, np.float32)
        for path in (0, 1):
            med = {}
            for name, xs in (("natural", natural), ("planted", rows)):
                ts = []
                for _ in range(30):
                    for x in xs:
                        t = time.perf_counter()
                        assert lib.ctb_norm_path(path, mode, ptr(x), ptr(w), ptr(b) if mode == 2 else None, ptr(y), k, 1e-5) == 0
                        ts.append(time.perf_counter() - t)
                med[name] = np.median(ts) * 1e6
            print(f"K {k} norm mode {mode} path {path}: natural {med['natural']:.1f} us, planted {med['planted']:.1f} us per call, "
                  f"difference {med['planted'] - med['natural']:.1f} us", flush=True)
