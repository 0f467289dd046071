#!/usr/bin/env python
"""Cost of one FragmentCalculator call for the energy alone (``derivative=False``) against the full call.

On Chignolin and Trp-cage, with the hydrogen refinement and the MM term on (synthetic amber-like parameters), host
positions to host result through ``calculate``, timed over ``--rounds`` alternated rounds of ``--calls`` calls each after
an untimed warm-up of each calculator:
  (a) ``FragmentCalculator(derivative=True)``: energy and forces (vb_forward_fragments_host, one graph replay);
  (b) ``FragmentCalculator(derivative=False)``: the energy alone on a forward-only engine
      (vb_forward_fragments_energy_host, one graph replay).
The geometry alternates between the PDB positions and a seeded 0.03 A perturbation, so no call sees the positions of
the call before.  Prints one JSON line with every round, both handles' workspace sizes and the card's name and power
limit, read in the same run.

    python tools/fragment_energy_cost.py [--calls 200] [--rounds 5]
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    from ai2bmd_b200 import caph
    from ai2bmd_b200.calculator import FragmentCalculator
    from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
    from ai2bmd_b200.nonbonded import synthetic_parameters

    out = {"card": card(), "calls": a.calls, "rounds": a.rounds}
    for name in ("chig", "trpcage"):
        fd, pm = load_fragments(name)
        x0, z, recipe = load_protein(name)
        prot = load_capped_protein(name)
        tables, _ = load_caph_tables(name)
        pr = caph.build_problem(prot, fd, recipe, tables)
        nb = synthetic_parameters(z, seed=1)
        geoms = [x0, x0 + 0.03 * np.random.default_rng(5).standard_normal(x0.shape)]
        calcs = {d: FragmentCalculator(WEIGHTS, "", fd, pm, recipe, caph=pr, nonbonded=nb, derivative=d)
                 for d in (True, False)}
        atoms = types.SimpleNamespace(numbers=z, positions=x0)

        def timed(calc):
            t = time.perf_counter()
            for i in range(a.calls):
                atoms.positions = geoms[i & 1]
                calc.calculate(atoms)
            return (time.perf_counter() - t) / a.calls * 1e6

        for calc in calcs.values():
            for x in geoms:
                atoms.positions = x
                calc.calculate(atoms)
        energies = []
        for x in geoms:
            atoms.positions = x
            e = []
            for calc in calcs.values():
                calc.calculate(atoms)
                e.append(float(calc.results["energy"]))
            energies.append(e)
        res = {"full": [], "energy": []}
        for _ in range(a.rounds):
            res["full"].append(timed(calcs[True]))
            res["energy"].append(timed(calcs[False]))
        out[name] = {"atoms": len(z), "fragment_atoms": len(fd.z), "fragments": len(fd),
                     "energies_equal": all(np.float32(f) == np.float32(e) for f, e in energies),
                     "arena_bytes_full": calcs[True].engine.get_option("arena_bytes"),
                     "arena_bytes_energy": calcs[False].engine.get_option("arena_bytes"),
                     "full_us": [min(res["full"]), max(res["full"])],
                     "energy_us": [min(res["energy"]), max(res["energy"])],
                     "ratio": min(res["full"]) / min(res["energy"]), "rounds_us": res}
        del calcs
    print(json.dumps(out))


if __name__ == "__main__":
    main()
