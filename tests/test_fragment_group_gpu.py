"""One FragmentCalculator call spread over a group of window engines in one process (vb_group_*, EngineGroup,
``FragmentCalculator(devices=...)``), and the reference's multi-device DLBondedCalculator.

Every case runs with k = 2 and 3 members on cuda:0 and again on k distinct GPUs when that many are visible (skipped
otherwise), on Chignolin and Trp-cage:

1. the join: the group's buffer equals, bit for bit, the rank-order float32 sum from +0.0f of the members' partials of
   the same call (vb_debug_read "ef"); each partial's energy equals the member's own vb_forward_fragments_host bit for
   bit and its forces to the bar (the forces are fp32 atomic sums in no fixed order, so two evaluations of the same
   launches differ in the last bits);
2. every member's placed and refined batch is bit-identical to the single handle's;
3. energy and forces agree with the single-handle FragmentCalculator within test_fragment_calculator_gpu.py's bars, at
   the PDB and a perturbed geometry, with refinement and MM on, with each off, and in chunks;
4. a k = 1 group against the single handle, the device entry against the host entry, no capture on a second call;
5. NaN partials left by a member's own call do not reach the next group call;
6. a call from a worker thread (AsyncQMMM's shape) gives the same result and leaves the thread's device as it was;
7. every refusal of vb_group_create, and a member reconfigured after it, name the member;
8. launch lists: the un-grouped Chignolin plan is the golden one, and a member launches what a DeviceShard window does;
9. DLBondedCalculator(devices=["cuda:0", "cuda:0"]) against the single-device calculator (per fragment, within the
   oracle bars) and against one model per block (the same launch plan: energies bit for bit)."""
import ctypes as C
import json
import os
import types
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.calculator import DLBondedCalculator, FragmentCalculator
from ai2bmd_b200.engine import Engine, EngineGroup, load_library
from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.md import DeviceLangevin
from ai2bmd_b200.nonbonded import synthetic_parameters
from ai2bmd_b200.parallel import DeviceShard, mm_rows

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NAMES = ["chig", "trpcage"]
F_TIE = 5e-2          # forces of protein atoms fed by a fragment on a VecLayerNorm tie: bounded jump only (DESIGN §2)


def e_tol(e, ulps=2):
    return np.maximum(4e-3, ulps * np.spacing(np.abs(e).astype(np.float32)))


def f_tol(f):
    return 5e-5 + 2e-5 * np.abs(f).max()


class _Case:
    def __init__(self, name):
        self.name = name
        self.fd, self.pm = load_fragments(name)
        self.x0, self.z, self.recipe = load_protein(name)
        tables, _ = load_caph_tables(name)
        self.prot = load_capped_protein(name)
        self.pr = caph.build_problem(self.prot, self.fd, self.recipe, tables)
        self.nb = synthetic_parameters(self.z, seed=1)
        self.geoms = {"pdb": self.x0,
                      "perturbed": self.x0 + 0.03 * np.random.default_rng(5).standard_normal(self.x0.shape)}

    def calc(self, refine=True, mm=True, **kw):
        return FragmentCalculator(WEIGHTS, "", self.fd, self.pm, self.recipe, caph=self.pr if refine else None,
                                  nonbonded=self.nb if mm else None, **kw)


_CASES = {}


def _case(name):
    if name not in _CASES:
        _CASES[name] = _Case(name)
    return _CASES[name]


def _layouts():
    out = []
    for k in (2, 3):
        out.append(pytest.param(["cuda:0"] * k, id=f"k{k}-cuda0"))
        out.append(pytest.param([f"cuda:{i}" for i in range(k)], id=f"k{k}-distinct",
                                marks=pytest.mark.skipif(torch.cuda.device_count() < k,
                                                         reason=f"{k} distinct GPUs are not visible")))
    return out


LAYOUTS = _layouts()


def _partials(calc):
    P = calc.n_protein
    return [sh.engine.debug_read("ef", 0, (3 * P + 1,)) for sh in calc.shards]


def _rank_sum(parts):
    s = np.zeros_like(parts[0])                       # +0.0f
    for p in parts:
        s = (s + p).astype(np.float32)
    return s


def _tied(c, sd, pos):
    """Protein atoms fed by a fragment on a VecLayerNorm tie at the placed positions `pos` (an unchunked evaluation)."""
    eng = Engine(sd, 0)
    eng.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd))
    eng.forward_host(pos)
    tie_frag = np.unique(c.fd.batch[eng.vecln_near_ties()])
    tie_atoms = np.isin(c.fd.batch, tie_frag)
    tied = np.zeros(c.pm.n_protein, bool)
    tied[c.pm.dst_atom[tie_atoms[c.pm.src_atom]]] = True
    return tied


# ---- 1-3. the join, the placed batch, and the single handle -----------------------------------------------------------
@pytest.mark.parametrize("variant", ["full", "no_refinement", "no_mm", "chunks"])
@pytest.mark.parametrize("devices", LAYOUTS)
@pytest.mark.parametrize("name", NAMES)
def test_group_against_its_partials_and_the_single_handle(real_weights, name, devices, variant):
    c = _case(name)
    refine, mm = variant != "no_refinement", variant != "no_mm"
    chunk = 60 if variant == "chunks" else None
    single = c.calc(refine, mm, chunk_size=chunk)
    group = c.calc(refine, mm, chunk_size=chunk, devices=devices)
    if chunk:
        assert all(sh.engine.get_option("chunks") >= 2 for sh in group.shards)
    N = len(c.fd.z)
    for geom, x in c.geoms.items():
        atoms = types.SimpleNamespace(numbers=c.z, positions=x)
        group.calculate(atoms)
        E, F = group.results["energy"], group.results["forces"]
        ef = np.r_[F.reshape(-1), np.float32(E)].astype(np.float32)
        parts = _partials(group)
        assert np.array_equal(_rank_sum(parts).view(np.uint32), ef.view(np.uint32)), geom       # 1. the join, bitwise
        E1, F1 = single.engine.forward_fragments_host(x)
        pos = single.engine.debug_read("pos", 0, (N, 3))
        tied = _tied(c, real_weights, pos)
        for r, sh in enumerate(group.shards):
            assert np.array_equal(sh.engine.debug_read("pos", 0, (N, 3)), pos), (geom, r)       # 2. the placed batch
            e_own, f_own = sh.engine.forward_fragments_host(x)
            assert np.float32(e_own) == parts[r][-1], (geom, r)
            assert np.abs(f_own.reshape(-1) - parts[r][:-1]).max() <= f_tol(f_own), (geom, r)
        df = np.abs(F - F1).max(1)                                                              # 3. the single handle
        bar_e = 4e-3 * len(c.fd)
        print(f"\n{name} {variant} {devices} {geom}: |dE| {abs(E - E1):.2e} eV (bar {bar_e:.2e}), "
              f"|dF| {df[~tied].max():.2e} eV/A (bar {f_tol(F1):.2e}), {tied.sum()} tie atoms")
        assert np.isfinite(F).all() and np.isfinite(E)
        assert abs(E - E1) <= bar_e
        assert df[~tied].max() <= f_tol(F1)
        assert (df[tied] <= F_TIE).all()


# ---- 4. k = 1, the device entry, the graph cache ----------------------------------------------------------------------
def test_one_member_group_is_the_single_handle():
    c = _case("chig")
    single, one = c.calc(), c.calc(devices=["cuda:0"])
    assert one.shards[0].engine.get_option("batch_atoms") == len(c.fd.z)          # the whole batch: no window
    for x in c.geoms.values():
        E1, F1 = single.engine.forward_fragments_host(x)
        E, F = one.group.forward_fragments_host(x)
        part = _partials(one)[0]
        assert np.array_equal((np.float32(0) + part).view(np.uint32), np.r_[F.reshape(-1), np.float32(E)].astype(np.float32).view(np.uint32))
        assert E == E1                                   # the energy sums run in a fixed order: bit for bit
        assert np.abs(F - F1).max() <= f_tol(F1)         # the forces are fp32 atomic sums: to the bar


@pytest.mark.parametrize("devices", LAYOUTS)
def test_device_entry_and_graph_cache(devices):
    c = _case("chig")
    calc = c.calc(devices=devices)
    g, P = calc.group, c.pm.n_protein
    x = c.geoms["perturbed"]
    E, F = g.forward_fragments_host(x)
    captures = [sh.engine.get_option("graph_captures") for sh in calc.shards]
    E2, F2 = g.forward_fragments_host(c.geoms["pdb"])
    E3, F3 = g.forward_fragments_host(x)
    assert [sh.engine.get_option("graph_captures") for sh in calc.shards] == captures     # same buffers: no capture
    assert E3 == E and np.abs(F3 - F).max() <= f_tol(F)
    dev = torch.device(devices[0])
    xd = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    out = torch.full((3 * P + 1,), float("nan"), device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev)
        g.forward_fragments_device(xd.data_ptr(), out.data_ptr(), stream.cuda_stream)
        captures = [sh.engine.get_option("graph_captures") for sh in calc.shards]
        g.forward_fragments_device(xd.data_ptr(), out.data_ptr(), stream.cuda_stream)
        assert [sh.engine.get_option("graph_captures") for sh in calc.shards] == captures
        stream.synchronize()
    ef = out.cpu().numpy()
    assert np.array_equal(_rank_sum(_partials(calc)).view(np.uint32), ef.view(np.uint32))
    assert np.float32(ef[-1]) == np.float32(E) and np.abs(ef[:-1] - F.reshape(-1)).max() <= f_tol(F)


# ---- 5. stale partials ------------------------------------------------------------------------------------------------
def _nan_decoy(c):
    """test_fragment_calculator_gpu.py's decoy: the first HA atom of every residue on its CA, so every buffer after the
    edge geometry is NaN."""
    x = c.x0 + 0.2 * np.random.default_rng(9).standard_normal(c.x0.shape)
    for r in np.unique(c.prot.resnums):
        at = [i for i in range(len(c.prot)) if c.prot.resnums[i] == r]
        ca = [i for i in at if c.prot.names[i] == "CA"]
        ha = [i for i in at if c.prot.names[i].startswith("HA")]
        if ca and ha:
            x[ha[0]] = x[ca[0]]
    return x


@pytest.mark.parametrize("devices", LAYOUTS)
@pytest.mark.parametrize("name", NAMES)
def test_stale_partials(name, devices):
    c = _case(name)
    calc = c.calc(devices=devices)
    clean = {g: calc.group.forward_fragments_host(x) for g, x in c.geoms.items()}
    for sh in calc.shards:
        sh.engine.forward_fragments_host(_nan_decoy(c))
    assert all(not np.isfinite(p).all() for p in _partials(calc))
    for g, x in c.geoms.items():
        E, F = calc.group.forward_fragments_host(x)
        assert np.isfinite(F).all() and E == clean[g][0], g
        assert np.abs(F - clean[g][1]).max() <= f_tol(F), g


# ---- 6. a worker thread -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("devices", LAYOUTS)
def test_worker_thread(devices):
    c = _case("chig")
    calc = c.calc(devices=devices)
    x = c.geoms["perturbed"]
    E, F = calc.group.forward_fragments_host(x)

    def work():
        torch.cuda.set_device(0)
        atoms = types.SimpleNamespace(numbers=c.z, positions=x)
        calc.calculate(atoms)
        return calc.results["energy"], calc.results["forces"], torch.cuda.current_device()

    with ThreadPoolExecutor(1) as pool:
        E_t, F_t, dev_after = pool.submit(work).result()
    assert E_t == E and np.abs(F_t - F).max() <= f_tol(F) and dev_after == 0
    torch.cuda.set_device(0)
    calc.group.forward_fragments_host(x)
    assert torch.cuda.current_device() == 0


# ---- 7. refusals ------------------------------------------------------------------------------------------------------
def _create(engines):
    lib = load_library()
    arr = (C.c_void_p * len(engines))(*[None if e is None else e.h for e in engines])
    out = C.c_void_p()
    rc = lib.vb_group_create(arr, len(engines), C.byref(out))
    if rc == 0:
        lib.vb_group_destroy(out)
    return rc, lib.vb_group_last_error(None).decode()


def _windows(c, sd, k, nonbonded=True, ranks=None):
    shards = [DeviceShard(sd, c.fd, c.pm, r, k, 0, native_comm=False) for r in (ranks or range(k))]
    for sh in shards:
        sh.set_window(c.fd, c.pm, c.recipe, caph=c.pr, nonbonded=c.nb if nonbonded else None)
    return shards


def test_refusals(real_weights):
    c = _case("chig")
    P = c.pm.n_protein
    w = _windows(c, real_weights, 2)
    e0, e1 = w[0].engine, w[1].engine
    assert _create([e0, e1])[0] == 0
    rc, msg = _create([e0, None])
    assert rc == -1 and "member 1 is null" in msg
    rc, msg = _create([e0, e1, e0])
    assert rc == -1 and "member 2" in msg
    rc, msg = _create([e1, e0])                                                     # windows out of rank order
    assert rc == -1 and "member 0" in msg and "tile" in msg
    rc, msg = _create([e0])                                                         # the batch not covered
    assert rc == -1 and "member 0" in msg and "ends at" in msg
    # MM rows on some members only, and rows that do not tile the protein
    mixed = _windows(c, real_weights, 2, nonbonded=False)
    rc, msg = _create([e0, mixed[1].engine])
    assert rc == -1 and "member 1" in msg and "MM rows" in msg
    rc, msg = _create([mixed[0].engine, e1])
    assert rc == -1 and "member 0" in msg and "MM rows" in msg
    assert _create([mixed[0].engine, mixed[1].engine])[0] == 0                      # no MM rows anywhere
    from ai2bmd_b200.nonbonded import dipeptide_atom_sets, exclusion_table
    excl = exclusion_table(P, dipeptide_atom_sets(c.fd, c.recipe, c.pm))
    whole_rows = _windows(c, real_weights, 2, nonbonded=False)
    for sh in whole_rows:
        sh.engine.set_nonbonded(*c.nb, *excl, 0, P)
    rc, msg = _create([whole_rows[0].engine, whole_rows[1].engine])
    assert rc == -1 and "member 1" in msg and "MM rows" in msg
    # another protein, another batch
    t = _case("trpcage")
    other = DeviceShard(real_weights, t.fd, t.pm, 1, 2, 0, native_comm=False)
    other.set_window(t.fd, t.pm, t.recipe)
    rc, msg = _create([e0, other.engine])
    assert rc == -1 and "member 1" in msg and "protein atoms" in msg
    block = DeviceShard(real_weights, c.fd, c.pm, 1, 2, 0, native_comm=False)         # block 1 without a window
    a0, a1 = block.plan.atom_lo, block.plan.atom_hi
    r = c.recipe
    block.engine.set_fragment_recipe(r.real[a0:a1], r.acc[a0:a1], r.rem[a0:a1], r.blen[a0:a1])
    rc, msg = _create([e0, block.engine])
    assert rc == -1 and "member 1" in msg and "batch" in msg
    # members that cannot evaluate fragments
    bare = Engine(real_weights, 0)
    bare.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd))
    rc, msg = _create([bare])
    assert rc == -3 and "member 0" in msg and "protein map" in msg
    bare.set_protein_map(P, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)
    rc, msg = _create([bare])
    assert rc == -3 and "member 0" in msg and "recipe" in msg
    fwd = Engine(real_weights, 0, derivative=False)
    fwd.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd))
    fwd.set_protein_map(P, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)
    fwd.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
    rc, msg = _create([fwd])
    assert rc == -3 and "member 0" in msg and "derivative" in msg
    un = DeviceLangevin.unfragmented(real_weights, c.z, c.x0, seed=1)
    rc, msg = _create([un.engine])
    assert rc == -3 and "member 0" in msg and "un-fragmented" in msg
    conn = _windows(c, real_weights, 2)
    conn[1].engine.comm_connect([conn[1].engine.comm_init(0, 1, 4 * P)])
    rc, msg = _create([conn[0].engine, conn[1].engine])
    assert rc == -3 and "member 1" in msg and "vb_comm_connect" in msg
    # a member reconfigured after vb_group_create
    for change in ("option", "caph", "recipe", "nonbonded", "topology"):
        w = _windows(c, real_weights, 2)
        g = EngineGroup([sh.engine for sh in w])
        E, _ = g.forward_fragments_host(c.x0)
        eng = w[1].engine
        if change == "option":
            eng.set_option("calibrate", 1)
        elif change == "caph":
            eng.set_caph(c.pr)
        elif change == "recipe":
            eng.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
        elif change == "nonbonded":
            eng.set_nonbonded(*c.nb, *excl, *mm_rows(P, 1, 2))
        else:                                    # the same block again: the window, recipe and map are gone
            a0, a1 = w[1].plan.atom_lo, w[1].plan.atom_hi
            eng.set_topology(c.fd.z[a0:a1], c.fd.batch[a0:a1] - c.fd.batch[a0])
        with pytest.raises(RuntimeError, match="member 1 was reconfigured"):
            g.forward_fragments_host(c.x0)
        xd = torch.from_numpy(np.ascontiguousarray(c.x0)).cuda()
        out = torch.zeros(3 * P + 1, device="cuda")
        with pytest.raises(RuntimeError, match="member 1 was reconfigured"):
            g.forward_fragments_device(xd.data_ptr(), out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        g.close()
    # null buffers
    g = EngineGroup([sh.engine for sh in _windows(c, real_weights, 2)])
    assert g.lib.vb_group_forward_fragments_host(g.g, None, None) == -1 and "null buffer" in g.last_error()
    assert g.lib.vb_group_forward_fragments(g.g, None, None, None) == -1 and "null buffer" in g.last_error()


# ---- 8. launch lists --------------------------------------------------------------------------------------------------
def test_launch_lists(real_weights):
    with open(os.path.join(ROOT, "tests", "golden", "chig_fragment_plan.json")) as fh:
        want = json.load(fh)
    c = _case("chig")
    grouped = c.calc(devices=["cuda:0"] * 2)
    grouped.group.forward_fragments_host(c.x0)
    whole = DeviceLangevin(real_weights, c.fd, c.pm, c.recipe, c.x0, c.z, seed=1).engine     # un-grouped, as before
    got = [list(k) for k in whole.stage_kernels()]
    assert [(s, k) for s, k, _ in got] == [(s, k) for s, k, _ in want["stage_kernels"]]
    if torch.cuda.get_device_properties(0).multi_processor_count == want["sm_count"]:
        assert got == want["stage_kernels"]
    assert whole.launches_per_forward == want["launches_per_forward"]
    for k in (2, 3):
        calc = c.calc(devices=["cuda:0"] * k)
        calc.group.forward_fragments_host(c.x0)
        for sh, ref in zip(calc.shards, _windows(c, real_weights, k)):
            assert sh.engine.stage_kernels() == ref.engine.stage_kernels()
            assert sh.engine.launches_per_forward == ref.engine.launches_per_forward


# ---- 9. the reference's multi-device DLBondedCalculator ---------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_bonded_calculator_on_two_devices(real_weights, name):
    c = _case(name)
    one = DLBondedCalculator(WEIGHTS)
    two = DLBondedCalculator(WEIGHTS, devices=["cuda:0", "cuda:0"])
    assert len(two.models) == 2 and two.models[0].engine is not two.models[1].engine
    fd = c.fd
    for calc in (one, two):              # the first call of a topology plans the tiles from its real edge count
        calc._evaluate(fd)
    e1, f1 = one._evaluate(fd)
    e2, f2 = two._evaluate(fd)
    assert e2.shape == e1.shape and f2.shape == f1.shape
    from ai2bmd_b200.calculator import ViSNetModel
    from ai2bmd_b200.parallel import partition_fragments
    for m, (lo, hi) in zip(two.models, partition_fragments(fd.start, fd.end, 2)):
        a0, a1 = int(fd.start[lo]), int(fd.end[hi - 1])
        assert np.all(np.abs(e2[lo:hi] - e1[lo:hi]) <= e_tol(e1[lo:hi])), (lo, hi)
        assert np.abs(f2[a0:a1] - f1[a0:a1]).max() <= f_tol(f1[a0:a1]), (lo, hi)
        # a block's launch plan follows its size, so it is not the whole batch's; against a single-device model of the
        # same block (the same plan) the energies are bit for bit, the forces (fp32 atomic sums) to the bar
        block = ViSNetModel(real_weights, device="cuda:0")
        block.dl_potential_loader(fd[lo:hi])
        e_b, f_b = block.dl_potential_loader(fd[lo:hi])
        assert block.engine.stage_kernels() == m.engine.stage_kernels()
        assert np.array_equal(e2[lo:hi], e_b), (lo, hi)
        assert np.abs(f2[a0:a1] - f_b).max() <= f_tol(f_b), (lo, hi)
    dip_e, dip_f, an_e, an_f = two.calculate(fd)
    d1 = one.calculate(fd)
    assert dip_e.shape == d1[0].shape and dip_f.shape == d1[1].shape and an_e.shape == d1[2].shape
    assert an_f.shape == d1[3].shape
