#!/usr/bin/env python
"""Device time of one MD step whose evaluation is spread over a group of window engines (``DeviceLangevin.grouped``).

On Chignolin and Trp-cage, with the hydrogen refinement on, the cases
  k1                    the single-handle DeviceLangevin (one engine of the whole batch);
  k members on cuda:0   ``devices=["cuda:0"] * k``, k = 1, 2, 3: every member places and refines the whole batch and
                        evaluates its block, all on one GPU;
  k distinct GPUs       ``devices=["cuda:0", ..., "cuda:{k-1}"]``, k = 2, 3 up to the device count, when there are several;
each timed as the best of ``--rounds`` alternated rounds of ``--steps`` steps (``run``), a host clock around work that
ends in a synchronise, after an untimed warm-up.  Also reports which form the group's step took (option md_group_graph:
1 one graph over every member's stream, 0 per-member replays).  Prints one JSON line with the device count and the name
and power limit of every card, read in the same run.

    python tools/md_group_cost.py [--steps 500] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def cards():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return [line.strip() for line in q.stdout.splitlines() if line.strip()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from ai2bmd_b200 import caph
    from ai2bmd_b200.fixtures import load_capped_protein, load_caph_tables, load_fragments, load_protein
    from ai2bmd_b200.md import DeviceLangevin
    from ai2bmd_b200.weights import load_state_dict

    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("no CUDA device: the step's cost is a GPU measurement")
    sd = load_state_dict(os.path.join(ROOT, "tests", "golden", "weights_2ef43f29.npz"))
    cases = {"k1": None, "g1_same": ["cuda:0"], "g2_same": ["cuda:0"] * 2, "g3_same": ["cuda:0"] * 3}
    for k in range(2, min(3, n_dev) + 1):
        cases[f"g{k}_distinct"] = [f"cuda:{i}" for i in range(k)]
    out = {"device_count": n_dev, "cards": cards(), "steps": a.steps, "rounds": a.rounds}
    for name in ("chig", "trpcage"):
        fd, pm = load_fragments(name)
        x0, z, recipe = load_protein(name)
        tables, _ = load_caph_tables(name)
        pr = caph.build_problem(load_capped_protein(name), fd, recipe, tables)
        runs = {}
        for key, devs in cases.items():
            if devs is None:
                runs[key] = DeviceLangevin(sd, fd, pm, recipe, x0, z, caph=pr, seed=1)
            else:
                runs[key] = DeviceLangevin.grouped(sd, fd, pm, recipe, x0, z, devices=devs, caph=pr, seed=1)

        def timed(md):
            md.stream.synchronize()
            t = time.perf_counter()
            md.run(a.steps)
            md.stream.synchronize()
            return (time.perf_counter() - t) / a.steps * 1e6

        for md in runs.values():
            md.run(20)
            md.stream.synchronize()
        rounds = {key: [] for key in runs}
        for _ in range(a.rounds):
            for key, md in runs.items():
                rounds[key].append(timed(md))
        out[name] = {"atoms": len(z), "fragment_atoms": len(fd.z), "fragments": len(fd),
                     "step_us": {key: min(v) for key, v in rounds.items()},
                     "step_us_rounds": rounds,
                     "md_group_graph": {key: md.engine.get_option("md_group_graph") for key, md in runs.items()},
                     "temperature_K": {key: md.temperature() for key, md in runs.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
