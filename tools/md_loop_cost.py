#!/usr/bin/env python
"""Cost of the device loop (``DeviceLangevin.run_segment``, one launch of a WHILE conditional graph) against one graph
replay per step (``run``), and how long each takes to return after a runaway halt.

On Chignolin (fragment step) and the ACE-ALA-NME input (un-fragmented step), one handle each:
  * us per step: ``run(n)`` + a device synchronise against ``run_segment(n)``, ``--steps`` steps from the same state,
    ``--rounds`` alternated rounds after an untimed warm-up of each (which pays the graph captures); the same again on a
    fresh handle with option ``use_pdl`` = 1 set before its first step, where the tool asserts that both graphs kept
    their programmatic edges (``use_pdl`` still 1, ``md_loop_pdl`` = 1: the conditional body accepted them);
  * halt to return: a 1000 K start at 300 K, so the recorder's runaway guard (1.5 T0) fires on the first record step
    (every ``--record`` steps), then ``run_observed(--steps, --record)`` (the block-wise drain) against ``run_segment``
    with the same recorder; the host time of the whole call minus the halting step's count times the step time.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/md_loop_cost.py [--steps 2000] [--rounds 3] [--record 10]
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
    ap.add_argument("--record", type=int, default=10)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai2bmd_b200.fixtures import GOLDEN, WEIGHTS, load_fragments, load_protein
    from ai2bmd_b200.md import KB, DeviceLangevin, TemperatureRunawayError
    from ai2bmd_b200.weights import load_state_dict
    sd = load_state_dict(WEIGHTS)

    def handle(name):
        if name == "chig":
            fd, pm = load_fragments("chig")
            pos, z, recipe = load_protein("chig")
            return DeviceLangevin(sd, fd, pm, recipe, pos, z, seed=0)
        g = np.load(os.path.join(GOLDEN, "reference_visnet_mode.npz"))
        return DeviceLangevin.unfragmented(sd, g["c1_z"], g["c1_pos"].astype(np.float64), seed=0)

    out = {"card": card(), "steps": a.steps, "rounds": a.rounds, "record_per_steps": a.record}
    for name in ("chig", "ace_ala_nme"):
        res = {}
        for pdl in (1, 0):                        # a fresh handle per setting, the option set before any step or loop
            dev = handle(name)
            eng = dev.engine
            eng.set_option("use_pdl", pdl)
            x0, v0, _, _ = dev.state()

            def timed(fn):
                eng.md_set_state(x0, v0, 0)       # every measurement starts from the same state
                dev._eval()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) / a.steps * 1e6

            def run():
                dev.run(a.steps)

            def seg():
                assert dev.run_segment(a.steps) == a.steps

            c0 = eng.get_option("graph_captures")
            timed(run), timed(seg)                # warm-up: both graphs captured, with this handle's option
            # the step graph and the loop graph (and the start evaluation's graph) were captured under this setting, and
            # neither capture fell back: both keep programmatic edges with use_pdl = 1
            assert eng.get_option("graph_captures") - c0 >= 2
            assert eng.get_option("use_pdl") == pdl and eng.get_option("md_loop_pdl") == pdl
            us = {"run": [], "run_segment": []}
            for _ in range(a.rounds):
                us["run"].append(timed(run))
                us["run_segment"].append(timed(seg))
            best = {k: min(v) for k, v in us.items()}
            key = "use_pdl" if pdl else "default"
            res[key] = {k: [round(t, 1) for t in v] for k, v in us.items()}
            res[key]["loop_minus_run_us"] = round(best["run_segment"] - best["run"], 1)
            res[key]["loop_body_pdl"] = eng.get_option("md_loop_pdl")
            res["atoms"] = dev.n
            if pdl:
                del dev, eng
                torch.cuda.empty_cache()
        step_us = min(res["default"]["run"])

        # halt to return
        v_hot = np.random.default_rng(6).standard_normal(x0.shape) * np.sqrt(1000.0 * KB / dev.masses[:, None])

        def halted(call, recorder):
            eng.md_set_recorder(*recorder)       # run_observed sets its own recorder inside the call
            eng.md_set_state(x0, v_hot, 0)
            dev._eval()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                call()
            except TemperatureRunawayError:
                pass
            t = time.perf_counter() - t0
            halt = eng.get_option("md_halt_step")
            assert halt > 0, "no runaway: raise the start temperature"
            return t * 1e6 - halt * step_us, int(halt)

        def observed():
            dev.run_observed(a.steps, a.record)

        def segment():
            dev.run_segment(a.steps)

        calls = (("run_observed", observed, (0,)), ("run_segment", segment, (a.record, a.steps // a.record + 1, 1.5)))
        for _, call, rec in calls:                # warm-up: captures with the recorder on
            halted(call, rec)
        lat = {"run_observed": [], "run_segment": []}
        halt_step = None
        for _ in range(a.rounds):
            for k, call, rec in calls:
                t, halt_step = halted(call, rec)
                lat[k].append(round(t, 0))
        res["halt_step"] = halt_step
        res["halt_to_return_us"] = lat
        out[name] = res
        eng.md_set_recorder(0)
        del dev, eng
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
