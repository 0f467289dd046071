#!/usr/bin/env python
"""Where do the tensor-core edge kernels start to pay?  Sweep the fragment count of the synthetic batch and time one
evaluation (CUDA events, L2 flushed) with edge_tc = 0 (SIMT), 1 (TC forward), 3 (TC forward + adjoint) at every tile
length, and with the engine's automatic choice.

    python tools/tc_crossover.py [--fragments 1,2,4,8,12,19,32] [--steps 40]

The engine's automatic policy (engine.cu choose_defaults) is meant to follow this table.
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from ai2bmd_b200.engine import Engine            # noqa: E402
from ai2bmd_b200.fixtures import WEIGHTS         # noqa: E402
from ai2bmd_b200.synth import synthetic_batch    # noqa: E402
from ai2bmd_b200.weights import load_state_dict  # noqa: E402


def time_eval(eng, pos, e, f, flush, steps):
    s = torch.cuda.current_stream()
    for _ in range(5):
        eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), s.cuda_stream)
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(steps):
        flush.fill_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), s.cuda_stream)
        b.record(s)
        b.synchronize()
        tot += a.elapsed_time(b)
    return tot / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fragments", default="1,2,4,8,12,19,32,64")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--stages", type=int, default=0, help="print the per-launch times of a batch of this many fragments")
    args = ap.parse_args()
    sd = load_state_dict(WEIGHTS)
    if args.stages:
        fd = synthetic_batch(args.stages, seed=0)
        pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
        eng = Engine(sd, 0)
        eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
        prof = eng.profile_stages(pos.data_ptr(), n_iter=10)
        for name, ms in prof:
            print(f"{name:<24} {ms * 1e3:8.1f} us")
        print(f"{'sum':<24} {sum(m for _, m in prof) * 1e3:8.1f} us  ({len(prof)} launches, edge_tc={eng.get_option('edge_tc')})")
        return
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    print(f"{'frags':>6} {'atoms':>6} {'tiles':>6} {'simt':>8} {'tc_fwd':>8} {'tc r32':>8} {'tc r64':>8} {'tc r96':>8} {'tc r128':>8} {'auto':>8}   ms per evaluation")
    for g in [int(x) for x in args.fragments.split(",")]:
        fd = synthetic_batch(g, seed=0)
        pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
        e = torch.empty(len(fd), dtype=torch.float32, device="cuda")
        f = torch.empty((len(fd.z), 3), dtype=torch.float32, device="cuda")
        row = []
        for tc, rows in ((0, 0), (1, 0), (3, 32), (3, 64), (3, 96), (3, 128), (-1, 0)):
            eng = Engine(sd, 0)
            if tc >= 0:
                eng.set_option("edge_tc", tc)
            if rows:
                eng.set_option("tc_rows", rows)
            eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
            row.append(time_eval(eng, pos, e, f, flush, args.steps))
            eng.close()
        print(f"{g:>6} {len(fd.z):>6} {len(fd.z) * 17 // 128:>6} " + " ".join(f"{t:>8.3f}" for t in row))


if __name__ == "__main__":
    main()
