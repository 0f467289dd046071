"""Cost of observing the device MD run every step, on Chignolin and Trp-cage.

Times, with a host clock around work that ends in a device synchronise, 1,000 steps each of
  (a) ``run(n)``: bare graph replays, no observer;
  (b) the per-step polling loop ``run_observed`` used before the frame recorder: ``md_run`` up to the record step, then
      ``md_get_state(n_hist=1)`` (a device synchronise and pageable copies of x, v, the counter and the whole energy
      ring), Ekin and the temperature check in numpy, the observer, and only then the next step -- restated here;
  (c) ``run_observed(n, 1, obs)`` on the frame recorder;
  (d) ``run_observed(n, 100, obs)``;
with a trivial observer, in ``--rounds`` alternated rounds in one process.  (c) and (d) include switching the recorder on
and off (two captures of the step graph per call), as every call pays them; (a) and (b) are preceded by an untimed step
that captures the plain step graph.  Every timed run starts from the same state (Chignolin with the bonded term alone
passes 1.5 T0 after about 3,000 steps in a row, and the guard would end the run).  Prints one JSON line with the card's
name and power limit.

    python tools/md_record_cost.py [--steps 1000] [--rounds 3]
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


def polling(md, n_steps, k, observer):
    """The observed run as it was before the frame recorder (a host round trip per record step)."""
    from ai2bmd_b200.md import KB, TemperatureRunawayError
    _, _, step, _ = md.state()
    end = step + n_steps
    while step < end:
        nxt = min(end, (step // k + 1) * k)
        md.run(nxt - step)
        step = nxt
        if step % k:
            continue
        x, v, _, hist = md.state(n_hist=1)
        ekin = 0.5 * float((md.masses[:, None] * v * v).sum())
        temp = 2.0 * ekin / (3 * md.n) / KB
        if temp > 1.5 * md.kT / KB:
            raise TemperatureRunawayError(f"temperature runaway at step {step}: {temp:.1f} K")
        observer(step, x, v, float(hist[0]), ekin)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from ai2bmd_b200.fixtures import WEIGHTS, load_fragments, load_protein
    from ai2bmd_b200.md import DeviceLangevin
    from ai2bmd_b200.weights import load_state_dict
    sd = load_state_dict(WEIGHTS)
    calls = [0]

    def obs(step, x, v, epot, ekin):
        calls[0] += 1

    def timed(fn, prime):
        prime()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / a.steps * 1e6

    out = {"card": card(), "steps": a.steps, "rounds": a.rounds, "us_per_step": {}}
    for name in ("chig", "trpcage"):
        fd, pm = load_fragments(name)
        pos, z, recipe = load_protein(name)
        md = DeviceLangevin(sd, fd, pm, recipe, pos, z, seed=0)
        x0, v0, _, _ = md.state()

        def restart(capture):
            md.engine.md_set_state(x0, v0, 0)
            md._eval()
            if capture:
                md.run(1)

        modes = {
            "a_run": (lambda: md.run(a.steps), lambda: restart(True)),
            "b_polling_1": (lambda: polling(md, a.steps, 1, obs), lambda: restart(True)),
            "c_recorder_1": (lambda: md.run_observed(a.steps, 1, obs), lambda: restart(False)),
            "d_recorder_100": (lambda: md.run_observed(a.steps, 100, obs), lambda: restart(False)),
        }
        for fn, prime in modes.values():          # warm-up: graph captures, pinned buffers, lazy module loads
            timed(fn, prime)
        us = {m: [] for m in modes}
        for _ in range(a.rounds):
            for m, (fn, prime) in modes.items():
                calls[0] = 0
                us[m].append(timed(fn, prime))
                want = a.steps // 100 if m == "d_recorder_100" else (0 if m == "a_run" else a.steps)
                assert calls[0] == want, (m, calls[0], want)
        best = {m: min(v) for m, v in us.items()}
        out["us_per_step"][name] = {m: [round(x, 1) for x in v] for m, v in us.items()}
        out[f"{name}_c_over_a_pct"] = round(100.0 * (best["c_recorder_1"] / best["a_run"] - 1.0), 2)
        out[f"{name}_b_over_a_pct"] = round(100.0 * (best["b_polling_1"] / best["a_run"] - 1.0), 2)
        out[f"{name}_final_T"] = round(md.temperature(), 1)
        del md
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
