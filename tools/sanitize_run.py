#!/usr/bin/env python
"""Tiny evaluation for compute-sanitizer (memcheck / racecheck / synccheck): a few fragments, chosen kernels.

    compute-sanitizer --tool memcheck python tools/sanitize_run.py [edge_tc] [n_fragments] [key=value ...]

Extra ``key=value`` pairs are engine options (``node_tc=1``, ``node_nb=4``); ``caph=1`` also runs the hydrogen refinement
and the whole-protein reduction of the first n_fragments through the device MD entry points."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from ai2bmd_b200.engine import Engine                    # noqa: E402
from ai2bmd_b200.fixtures import WEIGHTS, load_fragments  # noqa: E402
from ai2bmd_b200.weights import load_state_dict          # noqa: E402

edge_tc = int(sys.argv[1]) if len(sys.argv) > 1 else 3
nfrag = int(sys.argv[2]) if len(sys.argv) > 2 else 6
opts = dict(kv.split("=") for kv in sys.argv[3:])
fd, pm = load_fragments("chig")
sub = fd[0:nfrag] if not opts.get("caph") else fd
eng = Engine(load_state_dict(WEIGHTS), 0)
eng.set_topology(sub.z, sub.batch)
eng.set_option("use_graph", 0)
eng.set_option("edge_tc", edge_tc)
for k, v in opts.items():
    if k != "caph":
        eng.set_option(k, int(v))
e, f = eng.forward_host(sub.pos)
e2, f2 = eng.forward_host(sub.pos)
print("edge_tc", edge_tc, opts, "E0", e[0], "|F|max", np.abs(f).max(), "repeat diff", np.abs(f - f2).max())
if opts.get("caph"):
    from ai2bmd_b200 import caph
    from ai2bmd_b200.fixtures import load_capped_protein, load_caph_tables, load_protein
    from ai2bmd_b200.md import DeviceLangevin
    prot_pos, prot_z, recipe = load_protein("chig")
    pr = caph.build_problem(load_capped_protein("chig"), fd, recipe, load_caph_tables("chig")[0])
    md = DeviceLangevin(load_state_dict(WEIGHTS), fd, pm, recipe, prot_pos, prot_z, seed=1, caph=pr)
    md.engine.set_option("use_graph", 0)
    md.run(2)
    x, v, step, _ = md.state()
    print("device MD with refinement: step", step, "max |dx|", np.abs(x - prot_pos).max(), "evals", md.engine.get_option("caph_evals"))
