"""What evaluating a batch in fragment chunks (option "chunk_atoms", the reference's --chunk-size) costs and saves: the
workspace size and the graph-replay time of one evaluation, unchunked and in chunks of 9999 / 4000 / 2000 / 1000 atoms,
with forces (derivative = 1, vb_forward) and energies only (derivative = 0, vb_forward_energy).

Per workload and plan, one handle per chunk size runs on the same device positions, calibrated like the host entry
points.  Each timed sample is enough back-to-back replays between CUDA events to fill about 0.2 s; the chunk sizes
alternate inside every one of ``--rounds`` rounds.  Prints a table and one JSON line with the card's name and power
limit, read in the same run.

    python tools/chunk_cost.py [--workloads chig,abd,c4,c5] [--chunks 0,9999,4000,2000,1000] [--rounds 3]
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
    ap.add_argument("--workloads", default="chig,abd,c4,c5")
    ap.add_argument("--chunks", default="0,9999,4000,2000,1000")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from ai2bmd_b200.engine import Engine
    sd = load_weights()
    st = torch.cuda.current_stream()
    chunks = [int(c) for c in a.chunks.split(",")]
    out = {"card": card(), "rounds": a.rounds, "workloads": {}}
    rows = []
    for name in a.workloads.split(","):
        fd, _, desc = load_workload(name)
        N, G = len(fd.z), len(fd)
        pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
        e = torch.empty(G, device="cuda")
        f = torch.empty(N, 3, device="cuda")
        res = out["workloads"][name] = {"desc": desc, "N": N, "G": G}
        for derivative in (1, 0):
            plan = "full" if derivative else "energy"
            engines = {}
            for c in chunks:
                eng = Engine(sd, 0, derivative=bool(derivative), chunk_atoms=c)
                eng.set_topology(fd.z, fd.batch, n_graphs=G)
                engines[c] = eng

            def run(eng, derivative=derivative):
                if derivative:
                    eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), st.cuda_stream)
                else:
                    eng.energy_device(pos.data_ptr(), e.data_ptr(), st.cuda_stream)

            iters = {}
            for c, eng in engines.items():               # calibrate, capture, warm up, size the samples
                run(eng)
                eng.set_option("calibrate", 1)
                for _ in range(3):
                    run(eng)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(st)
                run(eng)
                t1.record(st)
                t1.synchronize()
                iters[c] = max(3, int(200.0 / max(t0.elapsed_time(t1), 1e-3)))
            us = {c: [] for c in chunks}
            for _ in range(a.rounds):
                for c, eng in engines.items():
                    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    t0.record(st)
                    for _ in range(iters[c]):
                        run(eng)
                    t1.record(st)
                    t1.synchronize()
                    us[c].append(t0.elapsed_time(t1) / iters[c] * 1e3)
            res[plan] = {str(c): {"chunks": eng.get_option("chunks"), "arena_bytes": eng.get_option("arena_bytes"),
                                  "launches": eng.launches_per_forward, "us": [round(x, 1) for x in us[c]]}
                         for c, eng in engines.items()}
            base = min(us[0]) if 0 in us else None
            for c, eng in engines.items():
                r = res[plan][str(c)]
                rows.append(f"{name:5s} {plan:6s} chunk {c:5d}: {r['chunks']:4d} chunks  arena {r['arena_bytes'] / 2**20:9.1f} MiB"
                            f"  {min(us[c]):10.1f} us (min of {a.rounds}, spread {max(us[c]) - min(us[c]):.1f})"
                            + (f"  x{min(us[c]) / base:.3f}" if base else ""))
            del engines, eng
            torch.cuda.empty_cache()
    print(out["card"])
    print("\n".join(rows))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
