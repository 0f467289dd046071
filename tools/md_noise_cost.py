#!/usr/bin/env python
"""Cost of generating the reference's noise stream inside the device MD step (``noise="reference"``) against the
default Philox stream.

Times ``md_run`` with a host clock around work that ends in a device synchronise, ``--steps`` steps per measurement, in
``--rounds`` alternated rounds in one process, on
  * Chignolin and Trp-cage: the whole step (placement, ViSNet, reduction, both kicks);
  * the c4_20k synthetic protein map's atom count (``synth.synthetic_protein_map`` of the >= 20k-atom batch, about 10k
    protein atoms): kicks over that many atoms around Chignolin's evaluation with an empty protein map, so the difference
    is the prologue's cost at that size (the fragment recipe of a synthetic batch places no real protein).
The noise source is switched on one handle between measurements (each switch re-captures the step graph; an untimed
step after it pays the capture).  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/md_noise_cost.py [--steps 1000] [--rounds 3]
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
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai2bmd_b200 import refnoise
    from ai2bmd_b200.engine import Engine
    from ai2bmd_b200.fixtures import WEIGHTS, load_fragments, load_protein
    from ai2bmd_b200.md import FS, KB, MASSES, DeviceLangevin
    from ai2bmd_b200.synth import synthetic_batch, synthetic_protein_map
    from ai2bmd_b200.weights import load_state_dict
    sd = load_state_dict(WEIGHTS)
    tables = refnoise.tables()
    st = torch.cuda.current_stream().cuda_stream

    def handle(name):
        """(engine, atoms, keep-alive) for one workload, seed 0, at 300 K and 0.001 / fs."""
        if name != "c4_20k":
            fd, pm = load_fragments(name)
            pos, z, recipe = load_protein(name)
            md = DeviceLangevin(sd, fd, pm, recipe, pos, z, seed=0)
            return md.engine, md.n, md
        P = synthetic_protein_map(synthetic_batch(512, seed=0, min_atoms=20000)).n_protein
        fd = load_fragments("chig")[0]
        eng = Engine(sd, 0)
        eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
        eng.set_protein_map(P, [], [], [], np.zeros(len(fd), np.float32))
        eng.forward_host(np.asarray(fd.pos, dtype=np.float32))
        ef = torch.zeros(3 * P + 1, dtype=torch.float32, device="cuda")
        n, rng = len(fd.z), np.random.default_rng(1)
        zero = np.zeros(n, np.int32)
        m = np.array([MASSES[int(q)] for q in rng.choice([1, 6, 7, 8, 16], size=P)])
        eng.md_setup(m, np.arange(n) % P, zero, zero, np.zeros(n, np.float32), FS, 300 * KB, 0.001 / FS, 0, ef.data_ptr())
        eng.md_set_state(rng.normal(size=(P, 3)) * 10, rng.normal(size=(P, 3)) * 0.01, 0)
        eng.md_eval(st)
        return eng, P, ef

    out = {"card": card(), "steps": a.steps, "rounds": a.rounds, "us_per_step": {}}
    for name in ("chig", "trpcage", "c4_20k"):
        eng, n, keep = handle(name)
        x0, v0, _, _ = eng.md_get_state()
        s0, inc = refnoise.pcg_state(0)

        def timed(kind):
            eng.md_set_noise(kind, s0, inc, tables)
            eng.md_set_state(x0, v0, 0)       # every measurement starts from the same state
            eng.md_run(1, st)                 # captures the step graph
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.md_run(a.steps, st)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / a.steps * 1e6

        timed(0), timed(1)                    # warm-up
        us = {"philox": [], "reference": []}
        for _ in range(a.rounds):
            us["philox"].append(timed(0))
            us["reference"].append(timed(1))
        best = {k: min(v) for k, v in us.items()}
        out["us_per_step"][name] = {k: [round(x, 1) for x in v] for k, v in us.items()}
        out[f"{name}_atoms"] = int(n)
        out[f"{name}_delta_us"] = round(best["reference"] - best["philox"], 1)
        out[f"{name}_delta_pct"] = round(100.0 * (best["reference"] / best["philox"] - 1.0), 2)
        del keep, eng
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
