#!/usr/bin/env python
"""Cost of the un-fragmented device MD step (the reference's ``--mode visnet``, ``DeviceLangevin.unfragmented``).

Times ``md_run`` with a host clock around work that ends in a device synchronise, ``--steps`` steps per measurement, in
``--rounds`` alternated rounds in one process, on
  * C1: the 22-atom ACE-ALA-NME input of tests/golden/reference_visnet_mode.npz (one graph);
  * whole Chignolin: 175 atoms as one graph.
Each handle runs ``--steps`` untimed steps first (graph capture, module load).  Prints one JSON line with microseconds
per step (every round and the median) and the card's name and power limit, read in the same run.

    python tools/md_visnet_cost.py [--steps 2000] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai2bmd_b200.fixtures import WEIGHTS
    from ai2bmd_b200.md import DeviceLangevin
    from ai2bmd_b200.weights import load_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("md_visnet_cost.py measures on the GPU; no CUDA device here")
    sd = load_state_dict(WEIGHTS)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "reference_visnet_mode.npz"))
    runs = {}
    for name, key in (("c1", "c1"), ("chig_whole", "chig")):
        md = DeviceLangevin.unfragmented(sd, gold[f"{key}_z"], gold[f"{key}_pos"].astype(np.float64), seed=0)
        md.run(a.steps)
        torch.cuda.synchronize()
        runs[name] = md
    us = {k: [] for k in runs}
    for _ in range(a.rounds):
        for name, md in runs.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            md.run(a.steps)
            torch.cuda.synchronize()
            us[name].append((time.perf_counter() - t) / a.steps * 1e6)
    out = {"tool": "md_visnet_cost", "card": card(), "steps": a.steps, "rounds": a.rounds,
           "atoms": {k: int(m.n) for k, m in runs.items()},
           "launches_per_step": {k: int(m.engine.launches_per_forward) + 3 for k, m in runs.items()},
           "us_per_step": {k: [round(x, 2) for x in v] for k, v in us.items()},
           "us_per_step_median": {k: round(float(np.median(v)), 2) for k, v in us.items()}}
    for k, m in runs.items():
        x, _, _, _ = m.state()
        assert np.isfinite(x).all(), k
    print(json.dumps(out))


if __name__ == "__main__":
    main()
