"""Graph-replay time of one evaluation with forces (``vb_forward``) against one without (``vb_forward_energy``), and the
workspace size of both modes of option "derivative".

For each workload one derivative = 1 handle runs both plans and one derivative = 0 handle runs the energy plan, all on the
same device positions, calibrated like the host entry points.  Each timed sample is ``--iters`` back-to-back replays
between CUDA events; the three variants alternate inside every one of ``--rounds`` rounds.  Prints a table and one JSON
line with the card's name and power limit, read in the same run.

    python tools/energy_times.py [--workloads chig,trpcage,abd,c4,c5] [--rounds 3] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

from bench import load_weights, load_workload                            # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="chig,trpcage,abd,c4,c5")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    from ai2bmd_b200.engine import Engine
    sd = load_weights()
    st = torch.cuda.current_stream()
    out = {"card": card(), "rounds": a.rounds, "iters": a.iters, "workloads": {}}
    rows = []
    for name in a.workloads.split(","):
        fd, _, desc = load_workload(name)
        N, G = len(fd.z), len(fd)
        pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
        e = torch.empty(G, device="cuda")
        f = torch.empty(N, 3, device="cuda")
        full, fwd_only = Engine(sd, 0), Engine(sd, 0, derivative=False)
        for eng in (full, fwd_only):
            eng.set_topology(fd.z, fd.batch, n_graphs=G)
        full.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), st.cuda_stream)
        full.set_option("calibrate", 1)
        fwd_only.energy_device(pos.data_ptr(), e.data_ptr(), st.cuda_stream)
        fwd_only.set_option("calibrate", 1)
        variants = {
            "forward (derivative=1)": lambda: full.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), st.cuda_stream),
            "energy (derivative=1)": lambda: full.energy_device(pos.data_ptr(), e.data_ptr(), st.cuda_stream),
            "energy (derivative=0)": lambda: fwd_only.energy_device(pos.data_ptr(), e.data_ptr(), st.cuda_stream),
        }
        for fn in variants.values():                 # graph captures, then a few warm replays
            for _ in range(5):
                fn()
        torch.cuda.synchronize()
        us = {k: [] for k in variants}
        for _ in range(a.rounds):
            for k, fn in variants.items():
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(st)
                for _ in range(a.iters):
                    fn()
                t1.record(st)
                t1.synchronize()
                us[k].append(t0.elapsed_time(t1) / a.iters * 1e3)
        arena = {"derivative=1": full.get_option("arena_bytes"), "derivative=0": fwd_only.get_option("arena_bytes")}
        launches = {"forward": full.launches_per_forward, "energy": fwd_only.launches_per_forward}
        best = {k: min(v) for k, v in us.items()}
        out["workloads"][name] = {"desc": desc, "N": N, "G": G, "us": {k: [round(x, 1) for x in v] for k, v in us.items()},
                                  "speedup_derivative1": round(best["forward (derivative=1)"] / best["energy (derivative=1)"], 2),
                                  "speedup_derivative0": round(best["forward (derivative=1)"] / best["energy (derivative=0)"], 2),
                                  "arena_bytes": arena, "arena_ratio": round(arena["derivative=0"] / arena["derivative=1"], 3),
                                  "launches": launches}
        rows.append(f"{name:8s} N={N:7d} " + "  ".join(f"{k}: {min(v):9.1f} us" for k, v in us.items()) +
                    f"  x{out['workloads'][name]['speedup_derivative0']:.2f}  arena {arena['derivative=1'] / 2**20:8.1f} -> "
                    f"{arena['derivative=0'] / 2**20:7.1f} MiB ({out['workloads'][name]['arena_ratio']:.3f})")
        del full, fwd_only
        torch.cuda.empty_cache()
    print(out["card"])
    print("\n".join(rows))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
