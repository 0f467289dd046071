#!/usr/bin/env python
"""Per-launch device times of one evaluation (CUDA events inside the library, eager launches) and the graph-replay time,
for a workload and a set of engine options.  GPU box diagnostic:

    python tools/stage_times.py --workload chig --opts node_tc=1 [--out stages.txt]
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

from ai2bmd_b200.engine import Engine                                   # noqa: E402
from bench import load_weights, load_workload                            # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="chig")
    ap.add_argument("--fragments", type=int, default=512)
    ap.add_argument("--max-frags", type=int, default=0)
    ap.add_argument("--opts", default="")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    fd, pm, desc = load_workload(args.workload, args.fragments)
    if args.max_frags:
        fd = fd[0:args.max_frags]
    eng = Engine(load_weights(), 0)
    for kv in filter(None, args.opts.split(",")):
        k, v = kv.split("=")
        eng.set_option(k, int(v))
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
    e = torch.empty(len(fd), device="cuda")
    f = torch.empty(len(fd.z), 3, device="cuda")
    st = torch.cuda.current_stream()
    eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), st.cuda_stream)
    if "tc_rows" not in args.opts:
        eng.set_option("calibrate", 1)
    prof = eng.profile_stages(pos.data_ptr(), n_iter=args.iters)
    for _ in range(5):
        eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), st.cuda_stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(args.iters):
        eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), st.cuda_stream)
    b.record(st)
    torch.cuda.synchronize()
    lines = [f"workload {args.workload}: {desc}: G={len(fd)} N={len(fd.z)}  options: {args.opts or 'defaults'} "
             f"(node_tc={eng.get_option('node_tc')}, edge_tc={eng.get_option('edge_tc')}, tc_rows={eng.get_option('tc_rows')}, tile_rows={eng.get_option('tile_rows')})"]
    for name, ms in prof:
        lines.append(f"{name:24s} {ms * 1e3:8.1f} us")
    lines.append(f"{'sum (eager, per-launch events)':32s} {sum(ms for _, ms in prof) * 1e3:8.1f} us  ({len(prof)} launches)")
    lines.append(f"{'graph replay, L2 warm':32s} {a.elapsed_time(b) / args.iters * 1e3:8.1f} us per evaluation")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
