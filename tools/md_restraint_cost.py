"""Cost of the Hookean restraints in the device MD step, on Chignolin.

Times ``md_run`` with and without restraints (every atom tethered plus the hydrogen bond springs) in the same process,
alternating, ``--runs`` times each, and the reference's default protocol: 5 x 2000 pre-equilibration steps, then 1000
production steps with the hydrogen bond springs.  Prints one JSON line with the card's name and power limit.

    python tools/md_restraint_cost.py [--steps 1000] [--runs 3] [--protocol 2000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--protocol", type=int, default=2000, help="pre-equilibration steps per stage (0: skip)")
    a = ap.parse_args()
    import torch
    from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_fragments, load_protein
    from ai2bmd_b200.md import DeviceLangevin
    from ai2bmd_b200.restraints import hydrogen_bond_springs
    from ai2bmd_b200.weights import load_state_dict
    sd = load_state_dict(WEIGHTS)
    fd, pm = load_fragments("chig")
    pos, z, recipe = load_protein("chig")
    springs = hydrogen_bond_springs(load_capped_protein("chig"))
    plain = DeviceLangevin(sd, fd, pm, recipe, pos, z, seed=0)
    restr = DeviceLangevin(sd, fd, pm, recipe, pos, z, seed=0)
    restr.set_restraints(tether_atoms=np.arange(restr.n), tether_k_kcal=10, springs=springs)

    def timed(md, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        md.run(n)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n * 1e6

    for md in (plain, restr):            # warm-up: graph capture
        timed(md, 50)
    us = {"plain": [], "restrained": []}
    for _ in range(a.runs):
        us["plain"].append(timed(plain, a.steps))
        us["restrained"].append(timed(restr, a.steps))
    out = {"card": card(), "steps": a.steps, "us_per_step": {k: [round(x, 2) for x in v] for k, v in us.items()},
           "overhead_pct": round(100.0 * (min(us["restrained"]) / min(us["plain"]) - 1.0), 3)}
    del plain, restr
    if a.protocol > 0:                   # the reference's default run: 5 restrained stages, then production with springs
        md = DeviceLangevin(sd, fd, pm, recipe, pos, z, seed=1)
        timed(md, 20)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        md.preequilibrate(a.protocol)
        md.set_restraints(springs=springs)
        md.run(1000)
        torch.cuda.synchronize()
        out["protocol_s"] = round(time.perf_counter() - t0, 3)
        out["protocol_steps"] = 5 * a.protocol + 1000
        out["protocol_final_T"] = round(md.temperature(), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
