#!/usr/bin/env python
"""In-kernel timeline of the tensor-core edge kernels: SM-clock stamps taken by CTA 0 (first tile) at every phase
boundary (engine option "timeline"; slots documented next to TC_TL in csrc/k_edge_tc.cuh).

    python tools/tc_timeline.py [--workload chig] [--layer 2] [--mhz 1920]

Prints, for the forward and the adjoint kernel of one layer, the time of each stamp relative to kernel start and
the delta to the previous stamp -- where a single 128-edge tile spends its ~30-60 us.
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from ai2bmd_b200.engine import Engine            # noqa: E402
from ai2bmd_b200.fixtures import WEIGHTS, load_fragments   # noqa: E402
from ai2bmd_b200.synth import synthetic_batch    # noqa: E402
from ai2bmd_b200.weights import load_state_dict  # noqa: E402

# Slots marked "96/128 rows" are stamped only by the two-buffer schedule of 96- and 128-row tiles; a tile of <= 64 rows
# copies no A operand and gathers no row set twice (its s1/s2, g_Pdk/g_q and g_Pf/g_wdot rows are written in one pass).
# The forward of a tile of <= 64 rows is warp-specialised: FWD_WS are the stamps of the MMA warps (thread 0), slots
# 32.. those of the gather warps (thread 128); both are printed in time order.
FWD_WS = {0: "kernel start", 1: "setup done (barriers)", 2: "f rows (= A) landed", 4: "dk -> tile",
          7: "dv MMAs done", 8: "dv -> tc_aux (attention done)", 11: "f -> tile", 3: "m complete (A of s1, s2)",
          13: "s1 -> abuf", 16: "s2 MMAs done", 17: "s2 -> tile (edge update done)", 18: "CTA barrier: s1/s2 sums start",
          19: "s1 sums done", 20: "s2 sums done", 31: "teardown done"}
FWD_WS_GATHER = {32: "q*k rows -> tc_aux", 33: "dk seen", 34: "attention weights done", 35: "dv seen",
                 36: "messages m done", 37: "xa aggregation done", 38: "f seen", 39: "edge update done"}
FWD = {0: "kernel start", 1: "setup done (barriers)", 2: "f rows (= A) + meta loaded",
       4: "dk MMAs done", 5: "dk -> tile", 6: "attention weights done", 7: "dv MMAs done", 8: "dv -> tile",
       9: "messages m done", 10: "xa aggregation done", 11: "f MMAs done (96/128 rows: + A=m copy)",
       12: "edge update (f) done", 13: "s1 MMAs done", 14: "s1 -> buffer", 15: "s1 aggregation done",
       16: "s2 MMAs done", 17: "s2 -> buffer", 18: "s2 aggregation done", 31: "teardown done"}
BWD = {0: "kernel start", 1: "setup done", 2: "meta loaded", 3: "s1-half SIMT done (<=64 rows: s1+s2)",
       5: "s2-half SIMT done (96/128 rows)", 6: "g3a MMAs done", 7: "A copied for g3b (96/128 rows)", 8: "g3b MMAs done",
       9: "g_m -> tile", 10: "g_m / g_Pdv SIMT done (= A of g4dv)", 12: "g_Pdk SIMT done (<=64 rows: + g_q)",
       13: "g4dv MMAs done", 14: "A copied for g4dk (96/128 rows)", 15: "g_q aggregation done",
       16: "g_Pf SIMT done (<=64 rows: + g_wdot)", 17: "g4dk MMAs done", 18: "A copied for g4f (96/128 rows)",
       19: "g_wdot aggregation done", 20: "last job MMAs done", 21: "g_f -> tile", 22: "g_f written", 31: "teardown done"}


NFWD = {0: "start", 1: "xa rows staged", 2: "o_proj unit done", 4: "K-quarters summed", 5: "per-node phase done",
        7: "projection unit done", 9: "results written", 11: "vec_dot done"}
NBWD = {0: "start", 1: "A rows staged", 3: "adjoint unit done", 5: "per-node phase done", 7: "o_proj adjoint unit done", 9: "g_xa written"}


def show(title, tl, names, mhz):
    t0 = int(tl[0])
    print(f"--- {title} ---")
    prev = t0
    for k in sorted(names):
        if tl[k] == 0:
            continue
        t = int(tl[k])
        print(f"  [{k:2d}] {names[k]:<36} {(t - t0) / mhz:8.2f} us   (+{(t - prev) / mhz:6.2f})")
        prev = t


def show_roles(title, tl, mma, gather, mhz):
    t0 = int(tl[0])
    print(f"--- {title} (M: MMA warps, G: gather warps) ---")
    stamps = sorted([(int(tl[k]), "M", n) for k, n in mma.items() if tl[k]] + [(int(tl[k]), "G", n) for k, n in gather.items() if tl[k]])
    last = {"M": t0, "G": t0}
    for t, role, name in stamps:
        print(f"  {role} {name:<36} {(t - t0) / mhz:8.2f} us   (+{(t - last[role]) / mhz:6.2f} on {role})")
        last[role] = t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="chig")
    ap.add_argument("--layer", type=int, default=2)
    ap.add_argument("--mhz", type=float, default=0.0)
    ap.add_argument("--opts", default="", help="comma list key=value for vb_set_option")
    args = ap.parse_args()
    mhz = args.mhz
    if not mhz:
        try:
            mhz = float(subprocess.check_output(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"]).split()[0])
        except Exception:
            mhz = 1920.0
    if args.workload.isdigit():
        fd = synthetic_batch(int(args.workload), seed=0)
    else:
        fd, _ = load_fragments(args.workload)
    sd = load_state_dict(WEIGHTS)
    eng = Engine(sd, 0)
    eng.set_option("edge_tc", 3)
    eng.set_option("timeline", 1)
    for kv in filter(None, args.opts.split(",")):
        kk, vv = kv.split("=")
        eng.set_option(kk, int(vv))
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    pos = np.ascontiguousarray(fd.pos, dtype=np.float32)
    for _ in range(3):
        eng.forward_host(pos)
    torch.cuda.synchronize()
    print(f"workload {args.workload}: {len(fd.z)} atoms, SM clock assumed {mhz:.0f} MHz, layer {args.layer}")
    nl = 6
    tf = eng.debug_read("TL", args.layer, (64,), dtype=np.uint64)
    tb = eng.debug_read("TL", nl + args.layer, (64,), dtype=np.uint64)
    if tf[32:].any():
        show_roles("edge_fwd_tc", tf, FWD_WS, FWD_WS_GATHER, mhz)
    else:
        show("edge_fwd_tc", tf, FWD, mhz)
    show("edge_bwd_tc", tb, BWD, mhz)
    if eng.get_option("node_tc") == 0:
        EMB = {0: "start", 1: "previous kernel complete (pdl)", 2: "loads issued, rows staged", 3: "aggregation done", 4: "combine done", 5: "x written"}
        for title, idx, names in ((f"node_fwd2 stage {args.layer}", args.layer, NFWD), (f"node_bwd2 stage {args.layer}", nl + 1 + args.layer, NBWD),
                                  ("embed_node_small", 2 * nl + 2, EMB)):
            tl = eng.debug_read("TLN", idx, (16, 16), dtype=np.uint64).astype(np.int64)     # [stamp][warp]
            t0 = tl[0][tl[0] > 0].min()
            print(f"--- {title} (nodes per CTA {eng.get_option('node_nb')}): per stamp, first / last warp to pass it ---")
            for i in sorted(names):
                row = tl[i][tl[i] > 0]
                if len(row):
                    per = " ".join(f"{(x - t0) / mhz:5.1f}" if x > 0 else "    -" for x in tl[i])
                    print(f"  [{i:2d}] {names[i]:<34} {(row.min() - t0) / mhz:7.2f} .. {(row.max() - t0) / mhz:7.2f} us   | {per}")

if __name__ == "__main__":
    main()
