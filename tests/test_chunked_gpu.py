"""Evaluation in fragment chunks (option "chunk_atoms", the reference's --chunk-size) on the GPU.

a. Every fragment's energy and forces against the fp64 oracle, with bars and VecLayerNorm-tie handling of
   test_kernel_variants_gpu.py (c): Chignolin in chunks of 40 (one to three fragments each) and 100, Trp-cage,
   ABD, and c160 (4,265 atoms) with full chunks above 600 atoms and a tail below, so that the full chunks run the
   tensor-core node stage and the tail the SIMT one; the dry-run list shows each chunk's own variant.
b. A chunk at least as large as the batch: energies bit-identical to an unchunked handle, forces within the adjoint's
   run-to-run jitter (the bar of test_stale_workspace_gpu.py).
c. The energy plan: chunked derivative = 0 energies bit-identical to a chunked derivative = 1 handle's.
d. The whole-protein reduction after the last chunk against the unchunked one.
e. Isolation: NaN-decoy fragments in the first chunk, the targets in a later, smaller one.
f. Memory: the 512-fragment batch in chunks of 2000 atoms.
g. The device MD step with chunks follows the unchunked one; recorder frames still arrive.
h. Calibration per chunk, and an edge overflow names its chunk.
i. The stage diagnostics refuse a chunked handle.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from stage_check import decoy_positions                                     # noqa: E402
from test_kernel_variants_gpu import e_tol                                  # noqa: E402


def _fd(name):
    from ai2bmd_b200.fixtures import load_fragments
    from ai2bmd_b200.synth import synthetic_batch
    if name[0] == "c" and name[1:].isdigit():
        return synthetic_batch(int(name[1:]), seed=5)
    return load_fragments(name)[0]


def _engine(weights, fd, chunk_atoms=0, derivative=True, max_edges=0):
    from ai2bmd_b200.engine import Engine
    eng = Engine(weights, 0, derivative=derivative, chunk_atoms=chunk_atoms)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd), max_edges=max_edges)
    return eng


def _chunks(eng):
    return [(eng.get_option(f"c{k}/first_graph"), eng.get_option(f"c{k}/graphs"), eng.get_option(f"c{k}/atoms"))
            for k in range(eng.get_option("chunks"))]


def c160_chunk_size(fd):
    """The smallest chunk size from 650 atoms on whose full chunks all hold >= 600 atoms and whose tail < 600."""
    from ai2bmd_b200.parallel import chunk_fragments
    start, end = np.asarray(fd.start), np.asarray(fd.end)
    for c in range(650, 900):
        ch = chunk_fragments(start, end, c)
        atoms = [int(end[hi - 1] - start[lo]) for lo, hi in ch]
        if len(ch) >= 3 and min(atoms[:-1]) >= 600 and atoms[-1] < 600:
            return c
    raise AssertionError("no chunk size splits c160 as wanted")


# ---- a. per fragment against the fp64 oracle -----------------------------------------------------------------------
ORACLE_CASES = [("chig", 40), ("chig", 100), ("trpcage", 250), ("abd", 1000), ("c160", None)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,chunk", ORACLE_CASES, ids=[f"{n}-{c or 'mixed'}" for n, c in ORACLE_CASES])
def test_every_fragment_against_the_fp64_oracle(real_weights, name, chunk):
    import torch
    from ai2bmd_b200.parallel import chunk_fragments
    from oracle import visnet_ref as O
    fd = _fd(name)
    chunk = chunk or c160_chunk_size(fd)
    eng = _engine(real_weights, fd, chunk)
    want = chunk_fragments(fd.start, fd.end, chunk)
    got = _chunks(eng)
    assert [(lo, hi - lo) for lo, hi in want] == [(g0, g) for g0, g, _ in got]
    assert len(got) >= 2
    sizes = np.asarray(fd.end) - np.asarray(fd.start)
    assert all(abs(atoms - chunk) <= sizes.max() / 2 + 1 for _, _, atoms in got[:-1])   # cut at the nearest boundary
    if chunk == 40:
        assert max(g for _, g, _ in got) <= 3 and len(got) > len(fd) // 3
    # each chunk runs the node-stage variant its own size selects, in the dry-run list too
    ks = eng.stage_kernels()
    assert eng.launches_per_forward == len(ks)
    for k, (_, _, atoms) in enumerate(got):
        mine = [kern for s, kern, _ in ks if s.startswith(f"c{k}/")]
        assert mine and any("finalize_kernel" in x for x in mine)
        tc = atoms >= 600
        assert eng.get_option(f"c{k}/node_tc") == int(tc)
        assert any("node_tc_kernel" in x for x in mine) == tc, (k, atoms)
        assert any("node_fwd2_kernel" in x for x in mine) == (not tc), (k, atoms)
    if name == "c160":
        assert {eng.get_option(f"c{k}/node_tc") for k in range(len(got))} == {0, 1}
    eng.forward_host(fd.pos)
    eng.set_option("calibrate", 1)
    e, f = eng.forward_host(fd.pos)
    ties = np.unique(fd.batch[_engine(real_weights, fd).vecln_near_ties()])   # the tie scan reads an unchunked handle
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64, device="cuda")
    G = len(fd)
    de, df, fbar = np.zeros(G), np.zeros(G), np.zeros(G)
    for g0 in range(0, G, 64):
        sub = fd[g0:min(G, g0 + 64)]
        e_ref, f_ref = oracle.energy_and_forces(sub.z, sub.pos, sub.batch)
        e_ref, f_ref = e_ref.cpu().numpy()[:, 0], f_ref.cpu().numpy()
        a0 = fd.start[g0]
        for j in range(len(sub)):
            g, s, t = g0 + j, int(sub.start[j]), int(sub.end[j])
            de[g] = abs(float(e[g]) - e_ref[j]) / e_tol(e_ref[j])
            df[g] = np.abs(f[a0 + s:a0 + t] - f_ref[s:t]).max()
            fbar[g] = 5e-5 + 2e-5 * np.abs(f_ref[s:t]).max()
    del oracle
    torch.cuda.empty_cache()
    assert (de <= 1).all(), f"energy: fragments {np.flatnonzero(de > 1)[:8]} (|dE| / e_tol up to {de.max():.2f})"
    assert len(ties) <= max(1, G // 20)
    keep = ~np.isin(np.arange(G), ties)
    bad = np.flatnonzero(keep & (df > fbar))
    assert not len(bad), f"forces: fragments {bad[:8]}, |dF| {df[bad[:8]]} over {fbar[bad[:8]]}"
    assert df.max() <= 5e-2
    print(f"\n{name} chunk {chunk}: {len(got)} chunks, |dE|/e_tol {de.max():.2f}, |dF|/bar {(df / fbar)[keep].max():.2f}")


# ---- b. one chunk as large as the batch ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chig", "abd"])
def test_a_chunk_as_large_as_the_batch_equals_the_unchunked_handle(real_weights, name):
    fd = _fd(name)
    a, b = _engine(real_weights, fd), _engine(real_weights, fd, chunk_atoms=10 ** 6)
    assert b.get_option("chunks") == 1 and a.get_option("chunks") == 1
    assert [s for s, _, _ in b.stage_kernels()] == ["c0/" + s for s, _, _ in a.stage_kernels()]
    assert [k for _, k, _ in b.stage_kernels()] == [k for _, k, _ in a.stage_kernels()]
    ea, fa = a.forward_host(fd.pos)
    eb, fb = b.forward_host(fd.pos)
    assert np.array_equal(ea, eb)
    ties = np.isin(fd.batch, np.unique(fd.batch[a.vecln_near_ties()]))
    df = np.abs(fa - fb).max(1)
    assert df[~ties].max(initial=0.0) <= 1e-5 + 1e-6 * np.abs(fa).max() and df.max() <= 5e-2


# ---- c. the energy plan -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,chunk", [("chig", 100), ("c160", None)])
def test_chunked_energy_plan_equals_chunked_full_plan(real_weights, name, chunk):
    fd = _fd(name)
    chunk = chunk or c160_chunk_size(fd)
    full, en = _engine(real_weights, fd, chunk), _engine(real_weights, fd, chunk, derivative=False)
    assert _chunks(full) == _chunks(en)
    assert en.get_option("arena_bytes") < full.get_option("arena_bytes")
    e1, _ = full.forward_host(fd.pos)
    e0 = en.energy_host(fd.pos)
    assert np.array_equal(e0, e1)
    e1d = full.energy_host(fd.pos)              # the energy entries of a derivative = 1 handle
    assert np.array_equal(e1d, e1)


# ---- d. whole-protein reduction --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,chunk", [("chig", 100), ("abd", 250)])
def test_whole_protein_reduction_after_the_last_chunk(real_weights, name, chunk):
    import torch
    from ai2bmd_b200.fixtures import load_fragments
    fd, pm = load_fragments(name)
    out = []
    for c in (0, chunk):
        eng = _engine(real_weights, fd, c)
        eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
        pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
        ef = torch.full((3 * pm.n_protein + 1,), -1.0, device="cuda")
        eng.forward_protein_device(pos.data_ptr(), ef.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        e, _ = eng.forward_host(fd.pos)
        out.append((ef.cpu().numpy().astype(np.float64), e, eng))
    (ef0, e0, eng0), (ef1, e1, eng1) = out
    assert eng1.get_option("chunks") >= 2 and np.isfinite(ef1).all()
    assert eng1.launches_per_forward == len(eng1.stage_names())
    # energy: within the sum of the fragments' energy bars
    assert abs(ef1[-1] - ef0[-1]) <= float(np.sum(e_tol(e0)))
    assert abs(ef1[-1] - float(np.sum(pm.frag_sign.astype(np.float64) * e1))) <= float(np.sum(e_tol(e1)))
    # forces: the end-to-end force bar; protein atoms fed by a fragment on a VecLayerNorm tie only bounded
    f0, f1 = ef0[:-1].reshape(-1, 3), ef1[:-1].reshape(-1, 3)
    tie_frag = np.unique(fd.batch[eng0.vecln_near_ties()])
    tie_atoms = np.isin(np.arange(len(fd.z)), np.flatnonzero(np.isin(fd.batch, tie_frag)))
    tied = np.zeros(pm.n_protein, bool)
    tied[pm.dst_atom[tie_atoms[pm.src_atom]]] = True
    df = np.abs(f1 - f0).max(1)
    bar = 5e-5 + 2e-5 * np.abs(f0).max()
    assert df[~tied].max(initial=0.0) <= bar, f"|dF| {df[~tied].max():.2e} over {bar:.2e}"
    assert df.max() <= 5e-2


# ---- e. isolation -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_nan_decoys_in_the_first_chunk_leave_later_chunks_alone(real_weights):
    import torch
    from ai2bmd_b200.fragment_data import FragmentData
    dec, tgt = _fd("trpcage"), _fd("chig")
    n_dec = len(dec.z)
    z = np.concatenate([dec.z, tgt.z])
    batch = np.concatenate([dec.batch, tgt.batch + len(dec)])
    target = np.ascontiguousarray(tgt.pos, dtype=np.float32)
    pos = np.concatenate([decoy_positions(dec.pos, dec.batch, "nan"), target]).astype(np.float32)
    start = np.concatenate([dec.start, tgt.start + n_dec])
    end = np.concatenate([dec.end, tgt.end + n_dec])
    both = FragmentData(z, pos, start, end, batch)
    chunk = n_dec                                   # the first chunk ends where the decoys end
    a = _engine(real_weights, both, chunk)
    got = _chunks(a)
    assert got[0] == (0, len(dec), n_dec) and all(n < n_dec for _, _, n in got[1:])
    b = _engine(real_weights, tgt)
    ties = np.isin(tgt.batch, np.unique(tgt.batch[b.vecln_near_ties()]))
    G, N = len(both), len(z)
    for entry in ("host", "device"):
        for use_graph in (0, 1):
            a.set_option("use_graph", use_graph)
            b.set_option("use_graph", use_graph)
            if entry == "host":
                e, f = a.forward_host(pos)
                e_b, f_b = b.forward_host(target)
            else:
                st = torch.cuda.current_stream().cuda_stream
                p = torch.from_numpy(pos).cuda()
                eo, fo = torch.full((G,), -1.0, device="cuda"), torch.full((N, 3), -1.0, device="cuda")
                a.forward_device(p.data_ptr(), eo.data_ptr(), fo.data_ptr(), st)
                pb = torch.from_numpy(target).cuda()
                ebo, fbo = torch.empty(len(tgt), device="cuda"), torch.empty((len(tgt.z), 3), device="cuda")
                b.forward_device(pb.data_ptr(), ebo.data_ptr(), fbo.data_ptr(), st)
                torch.cuda.synchronize()
                e, f, e_b, f_b = eo.cpu().numpy(), fo.cpu().numpy(), ebo.cpu().numpy(), fbo.cpu().numpy()
            label = f"{entry} use_graph={use_graph}"
            assert not np.isfinite(e[:len(dec)][np.bincount(dec.batch) >= 2]).any(), f"{label}: the decoys did not poison"
            e_t, f_t = e[len(dec):], f[n_dec:]
            assert np.isfinite(e_t).all() and np.isfinite(f_t).all(), label
            assert np.abs(e_t - e_b).max() <= e_tol(e_b).min(), label
            df = np.abs(f_t - f_b).max(1)
            assert df[~ties].max(initial=0.0) <= 1e-5 + 1e-6 * np.abs(f_b).max() and df.max() <= 5e-2, label


# ---- f. memory ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_chunked_arena_is_bounded_by_the_largest_chunk(real_weights):
    from ai2bmd_b200.synth import synthetic_batch
    fd = synthetic_batch(512, seed=0)
    N = len(fd.z)
    c = _engine(real_weights, fd, 2000)
    chunked = c.get_option("arena_bytes")
    g0, g, atoms = max(_chunks(c), key=lambda t: t[2])
    largest = _engine(real_weights, fd[g0:g0 + g]).get_option("arena_bytes")
    del c
    whole = _engine(real_weights, fd).get_option("arena_bytes")
    print(f"\n512-fragment batch, {N} atoms: arena {whole / 2**20:.1f} MiB unchunked, {chunked / 2**20:.1f} MiB in chunks "
          f"of 2000 atoms (largest {atoms} atoms: {largest / 2**20:.1f} MiB alone)")
    assert chunked <= largest + 256 * N
    assert 5 * chunked <= whole


# ---- g. device MD step --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_md_with_chunks_follows_the_unchunked_step(real_weights):
    from ai2bmd_b200.fixtures import load_fragments, load_protein
    from ai2bmd_b200.md import DeviceLangevin
    from test_md_gpu import V_TOL, X_TOL
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    n = 50
    pool = np.random.default_rng(3).standard_normal((n, 2, pm.n_protein, 3))
    runs = []
    for chunk in (0, 100):
        dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, friction_per_fs=0.01, seed=3,
                             chunk_atoms=chunk)
        dev.set_normals(pool)
        dev.run(n)
        runs.append(dev)
    assert runs[1].engine.get_option("chunks") >= 2
    (x0, v0, s0, h0), (x1, v1, s1, h1) = (r.state(n_hist=n) for r in runs)
    assert s0 == s1 == n
    assert np.abs(x1 - x0).max() <= X_TOL and np.abs(v1 - v0).max() <= V_TOL
    assert np.abs(h1 - h0).max() <= 1e-2
    seen = []
    runs[1].run_observed(10, 5, lambda step, x, v, epot, ekin: seen.append(step))
    assert seen == [n + 5, n + 10]


# ---- h. calibration and overflow ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_calibration_plans_each_chunk_from_its_own_edges(real_weights):
    fd = _fd("trpcage")
    eng = _engine(real_weights, fd, 250)
    nc = eng.get_option("chunks")
    eng.forward_host(fd.pos)
    eng.set_option("calibrate", 1)
    edges = [eng.get_option(f"c{k}/edges") for k in range(nc)]
    assert all(e > 0 for e in edges) and len(set(edges)) > 1
    assert [eng.get_option(f"c{k}/edges_plan") for k in range(nc)] == edges
    # the real count of every chunk, from the neighbour list of the whole batch, which vb_get_edges reports in batch
    # atom indices as an unchunked handle does
    slots, deg = eng.get_edges()
    ref = _engine(real_weights, fd)
    ref.forward_host(fd.pos)
    slots_u, deg_u = ref.get_edges()
    assert np.array_equal(slots, slots_u) and np.array_equal(deg, deg_u)
    for k, (g0, g, _) in enumerate(_chunks(eng)):
        a0, a1 = int(fd.start[g0]), int(fd.end[g0 + g - 1])
        assert edges[k] == int(deg[a0:a1].sum())


@pytest.mark.gpu
def test_an_edge_overflow_names_its_chunk(real_weights):
    fd = _fd("trpcage")
    probe = _engine(real_weights, fd, 250)
    probe.forward_host(fd.pos)
    edges = [probe.get_option(f"c{k}/edges") for k in range(probe.get_option("chunks"))]
    cap = sorted(edges)[-2] if sorted(edges)[-2] < max(edges) else max(edges) - 1
    over = next(k for k, e in enumerate(edges) if e > cap)
    eng = _engine(real_weights, fd, 250, max_edges=cap)
    assert eng.get_option("n_edges_capacity") == cap
    with pytest.raises(RuntimeError, match=rf"chunk {over} \(fragments"):
        eng.forward_host(fd.pos)
    ok = _engine(real_weights, fd, 250, max_edges=max(edges))
    e, f = ok.forward_host(fd.pos)
    assert np.isfinite(e).all() and np.isfinite(f).all()


# ---- i. refusals --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stage_diagnostics_refuse_a_chunked_handle(real_weights):
    import torch
    fd = _fd("chig")
    eng = _engine(real_weights, fd, 100)
    pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
    for call in (lambda: eng.debug_run(pos.data_ptr(), 3), lambda: eng.profile_stages(pos.data_ptr(), 1),
                 lambda: eng.set_option("timeline", 1), lambda: eng.debug_read("X", 1, (len(fd.z), 128))):
        with pytest.raises(RuntimeError, match=r"\(-3\)"):
            call()
    e, _ = eng.forward_host(fd.pos)                # still usable
    assert np.isfinite(e).all()
    assert eng.debug_read("energy", 0, (len(fd),)).tolist() == e.tolist()
