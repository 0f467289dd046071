#!/usr/bin/env python
"""Cost of one FragmentCalculator call on the device against the host composition a drop-in of the model alone implies.

On Chignolin and Trp-cage, with the hydrogen refinement and the MM term on (synthetic amber-like parameters), timed as
the best of ``--rounds`` alternated rounds of ``--calls`` calls each after an untimed warm-up of each path:
  (a) ``FragmentCalculator.calculate``, host positions to host energy and forces (one graph replay, synchronous);
  (b) the composition the reference's loop runs when only the model is on the GPU: ``recipe.positions`` on the host,
      the refinement on the host CPU (the C restatement ``oracle/caph_c.py`` standing in for the reference's torch LBFGS),
      ``ViSNetModel.dl_potential_loader``, the host dipeptide / ACE-NME combination, and ``MMNonBondedCalculator``;
  (c) ``md_eval`` replays alone on a twin of the calculator's handle, timed to a device synchronise: the device work of
      (a) without its copies and host calls.
The geometry alternates between the PDB positions and a seeded 0.03 A perturbation, so no call sees the positions of
the call before.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/fragment_calculator_cost.py [--calls 200] [--rounds 3]
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
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai2bmd_b200 import caph
    from ai2bmd_b200.calculator import DipeptideBondedCombiner, FragmentCalculator, ViSNetModel
    from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
    from ai2bmd_b200.fragment_data import FragmentData
    from ai2bmd_b200.nonbonded import MMNonBondedCalculator, dipeptide_atom_sets, exclusion_table, synthetic_parameters
    from ai2bmd_b200.weights import load_state_dict
    from oracle.caph_c import relax_problem
    sd = load_state_dict(WEIGHTS)

    out = {"card": card(), "calls": a.calls, "rounds": a.rounds}
    for name in ("chig", "trpcage"):
        fd, pm = load_fragments(name)
        x0, z, recipe = load_protein(name)
        prot = load_capped_protein(name)
        tables, _ = load_caph_tables(name)
        pr = caph.build_problem(prot, fd, recipe, tables)
        nb = synthetic_parameters(z, seed=1)
        geoms = [x0, x0 + 0.03 * np.random.default_rng(5).standard_normal(x0.shape)]

        calc = FragmentCalculator(WEIGHTS, "", fd, pm, recipe, caph=pr, nonbonded=nb)
        atoms = types.SimpleNamespace(numbers=z, positions=x0)

        def device_call(x):
            atoms.positions = x
            calc.calculate(atoms, ["energy", "forces"], ["positions"])
            return calc.results["energy"]

        # (b): the model alone on the GPU, everything around it on the host
        model = ViSNetModel(sd, device="cuda:0")
        mm = MMNonBondedCalculator(model.engine)
        mm.set_parameters(*nb, *exclusion_table(pm.n_protein, dipeptide_atom_sets(fd, recipe, pm)))
        dip_g, an_g = fd.scalar_split()
        dip_a, an_a = fd.vector_split()
        at = np.empty(len(fd.z), dtype=np.int64)
        at[dip_a] = np.arange(dip_a.sum())
        at[an_a] = dip_a.sum() + np.arange(an_a.sum())
        select, origin = at[pm.src_atom], pm.dst_atom
        frag = FragmentData(fd.z, fd.pos.copy(), fd.start, fd.end, fd.batch)

        def host_call(x):
            frag.pos = relax_problem(pr, recipe.positions(x))[0]
            e, f = model.dl_potential_loader(frag)
            e_b = DipeptideBondedCombiner.energy_combine(e[dip_g], e[an_g])
            f_b = DipeptideBondedCombiner.forces_combine(pm.n_protein, f[dip_a], f[an_a], select, origin)
            e_mm, f_mm = mm(x)
            return float(e_b) + e_mm, f_b + f_mm

        def timed(fn):
            t = time.perf_counter()
            for i in range(a.calls):
                fn(geoms[i & 1])
            return (time.perf_counter() - t) / a.calls * 1e6

        # (c): the same launches as md_eval replays, on a twin of the calculator's handle (same inputs, same calibration):
        # on an engine with MD set up, the host entry would first wait for the device
        eng = FragmentCalculator(WEIGHTS, "", fd, pm, recipe, caph=pr, nonbonded=nb).engine
        ef = torch.zeros(3 * pm.n_protein + 1, device="cuda")
        stream = torch.cuda.current_stream()

        eng.md_setup(np.ones(pm.n_protein), recipe.real, recipe.acc, recipe.rem, recipe.blen, 0.1, 0.025, 0.0, 0,
                     ef.data_ptr())
        eng.md_set_state(x0, np.zeros_like(x0), 0)

        def md_timed():
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(a.calls):
                eng.md_eval(stream.cuda_stream)
            torch.cuda.synchronize()
            return (time.perf_counter() - t) / a.calls * 1e6

        for fn in (device_call, host_call):
            for x in geoms:
                fn(x)
        md_timed()
        e_dev, e_host = device_call(x0), host_call(x0)[0]
        res = {"a": [], "b": [], "c": []}
        for _ in range(a.rounds):
            res["a"].append(timed(device_call))
            res["b"].append(timed(host_call))
            res["c"].append(md_timed())
        out[name] = {"atoms": len(z), "fragment_atoms": len(fd.z), "fragments": len(fd),
                     "energy_device_eV": e_dev, "energy_host_eV": e_host,
                     "a_calculate_us": min(res["a"]), "b_host_composition_us": min(res["b"]),
                     "c_md_eval_us": min(res["c"]), "rounds_us": res}
        del calc, model, mm, eng
    print(json.dumps(out))


if __name__ == "__main__":
    main()
