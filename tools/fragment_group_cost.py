#!/usr/bin/env python
"""Host-to-host time of one FragmentCalculator call spread over a group of window engines (``devices=``).

On Chignolin and Trp-cage, with the hydrogen refinement and the MM term on (synthetic amber-like parameters), the cases
  k = 1                 the single-device calculator (``devices=None``);
  k members on cuda:0   ``devices=["cuda:0"] * k``, k = 2, 3: every member places and refines the whole batch and
                        evaluates its block, all on one GPU;
  k distinct GPUs       ``devices=["cuda:0", ..., "cuda:{k-1}"]``, k = 2 .. min(4, device count), when there are several;
each timed as the best of ``--rounds`` alternated rounds of ``--calls`` synchronous ``calculate`` calls after an untimed
warm-up.  The geometry alternates between the PDB positions and a seeded 0.03 A perturbation.  Prints one JSON line with
the device count and the name and power limit of every card, read in the same run.

    python tools/fragment_group_cost.py [--calls 200] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def cards():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return [line.strip() for line in q.stdout.splitlines() if line.strip()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai2bmd_b200 import caph
    from ai2bmd_b200.calculator import FragmentCalculator
    from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
    from ai2bmd_b200.nonbonded import synthetic_parameters

    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("no CUDA device: the group's cost is a GPU measurement")
    cases = {"k1": None, "k2_same": ["cuda:0"] * 2, "k3_same": ["cuda:0"] * 3}
    for k in range(2, min(4, n_dev) + 1):
        cases[f"k{k}_distinct"] = [f"cuda:{i}" for i in range(k)]
    out = {"device_count": n_dev, "cards": cards(), "calls": a.calls, "rounds": a.rounds}
    for name in ("chig", "trpcage"):
        fd, pm = load_fragments(name)
        x0, z, recipe = load_protein(name)
        tables, _ = load_caph_tables(name)
        pr = caph.build_problem(load_capped_protein(name), fd, recipe, tables)
        nb = synthetic_parameters(z, seed=1)
        geoms = [x0, x0 + 0.03 * np.random.default_rng(5).standard_normal(x0.shape)]
        calcs = {key: FragmentCalculator(WEIGHTS, "", fd, pm, recipe, caph=pr, nonbonded=nb, devices=devs)
                 for key, devs in cases.items()}
        atoms = types.SimpleNamespace(numbers=z, positions=x0)

        def timed(calc):
            t = time.perf_counter()
            for i in range(a.calls):
                atoms.positions = geoms[i & 1]
                calc.calculate(atoms)
            return (time.perf_counter() - t) / a.calls * 1e6

        energy = {}
        for key, calc in calcs.items():
            for x in geoms:
                atoms.positions = x
                calc.calculate(atoms)
            energy[key] = calc.results["energy"]
        rounds = {key: [] for key in calcs}
        for _ in range(a.rounds):
            for key, calc in calcs.items():
                rounds[key].append(timed(calc))
        out[name] = {"atoms": len(z), "fragment_atoms": len(fd.z), "fragments": len(fd),
                     "calculate_us": {key: min(v) for key, v in rounds.items()},
                     "energy_eV_at_perturbed": energy, "rounds_us": rounds}
        del calcs
    print(json.dumps(out))


if __name__ == "__main__":
    main()
