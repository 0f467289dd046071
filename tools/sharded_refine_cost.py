#!/usr/bin/env python
"""Cost of refining the cap hydrogens of the whole batch on every rank of a sharded step.

On Chignolin and Trp-cage, with the MM term on (synthetic amber-like parameters), the device time of one
``vb_forward_fragments`` replay (placement, hydrogen refinement, evaluation with its signed reduction, MM term) of:
  (a) the unwindowed handle: the whole batch with the refinement;
  (b) each W = 2 window handle (DeviceShard.set_window) with the whole batch's refinement;
  (c) the same windows without the refinement.
Each is timed with CUDA events over ``--calls`` back-to-back replays on the same positions, best of ``--rounds``
alternated rounds after an untimed warm-up.  With two or more GPUs it also times the sharded MD step
(DeviceLangevin.sharded, refinement and MM on, the engine's own all-reduce) on Chignolin over ``--steps`` steps; with
one GPU that number is reported as not measured.  Prints one JSON line with the card's name and power limit, read in
the same run.

    python tools/sharded_refine_cost.py [--calls 200] [--rounds 5] [--steps 500]
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _case(name):
    import numpy as np
    from ai2bmd_b200 import caph
    from ai2bmd_b200.fixtures import load_capped_protein, load_caph_tables, load_fragments, load_protein
    from ai2bmd_b200.nonbonded import synthetic_parameters
    fd, pm = load_fragments(name)
    x0, z, recipe = load_protein(name)
    tables, _ = load_caph_tables(name)
    pr = caph.build_problem(load_capped_protein(name), fd, recipe, tables)
    return fd, pm, np.ascontiguousarray(x0), z, recipe, pr, synthetic_parameters(z, seed=1)


def _md_worker(rank, world, port, steps, out):
    import time
    import torch
    import torch.distributed as dist
    from ai2bmd_b200.fixtures import WEIGHTS
    from ai2bmd_b200.md import DeviceLangevin
    from ai2bmd_b200.weights import load_state_dict
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    fd, pm, x0, z, recipe, pr, nb = _case("chig")
    md = DeviceLangevin.sharded(load_state_dict(WEIGHTS), fd, pm, recipe, x0, z, dist.group.WORLD, caph=pr, nonbonded=nb,
                                device=rank, seed=0)
    md.run(50)
    torch.cuda.synchronize()
    dist.barrier()
    t = time.perf_counter()
    md.run(steps)
    torch.cuda.synchronize()
    us = (time.perf_counter() - t) / steps * 1e6
    if rank == 0:
        with open(out, "w") as fh:
            json.dump({"ranks": world, "step_us": us, "one_graph": bool(md._native_comm)}, fh)
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=500)
    a = ap.parse_args()
    import torch
    from ai2bmd_b200.calculator import FragmentCalculator
    from ai2bmd_b200.fixtures import WEIGHTS
    from ai2bmd_b200.parallel import DeviceShard
    from ai2bmd_b200.weights import load_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    sd = load_state_dict(WEIGHTS)
    stream = torch.cuda.current_stream()
    out = {"card": card(), "calls": a.calls, "rounds": a.rounds}
    for name in ("chig", "trpcage"):
        fd, pm, x0, z, recipe, pr, nb = _case(name)
        xd = torch.from_numpy(x0).cuda()
        handles = {"a_unwindowed": FragmentCalculator(WEIGHTS, "", fd, pm, recipe, caph=pr, nonbonded=nb).engine}
        for refine in (True, False):
            for r in range(2):
                sh = DeviceShard(sd, fd, pm, r, 2, 0, native_comm=False)
                sh.set_window(fd, pm, recipe, caph=pr if refine else None, nonbonded=nb)
                handles[f"{'b' if refine else 'c'}_window{r}{'' if refine else '_no_refinement'}"] = sh.engine
        bufs = {k: torch.zeros(3 * pm.n_protein + 1, device="cuda") for k in handles}

        def timed(key):
            eng, ef = handles[key], bufs[key]
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(stream)
            for _ in range(a.calls):
                eng.forward_fragments_device(xd.data_ptr(), ef.data_ptr(), stream.cuda_stream)
            t1.record(stream)
            t1.synchronize()
            return t0.elapsed_time(t1) / a.calls * 1e3

        for k in handles:            # graph capture and warm-up
            timed(k)
        res = {k: [] for k in handles}
        for _ in range(a.rounds):
            for k in handles:
                res[k].append(timed(k))
        out[name] = {"atoms": len(z), "fragment_atoms": len(fd.z), "fragments": len(fd),
                     **{f"{k}_us": min(v) for k, v in res.items()}, "rounds_us": res}
        del handles, bufs
    if torch.cuda.device_count() >= 2:
        import torch.multiprocessing as mp
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "md.json")
            mp.spawn(_md_worker, args=(torch.cuda.device_count(), port, a.steps, path), nprocs=torch.cuda.device_count(),
                     join=True)
            with open(path) as fh:
                out["chig_sharded_md"] = json.load(fh)
    else:
        out["chig_sharded_md"] = "not measured: one GPU"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
