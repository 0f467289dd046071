"""Multi-GPU evaluation: fragments sharded over ranks, one all-reduce of the whole-protein buffer per step.

The reference spreads fragments over devices as contiguous, atom-balanced blocks of the interleaved
fragment list (``/root/reference/src/Calculators/device_strategy.py:83-127``), runs one Python thread /
sub-process per device, concatenates the results on the host and re-uploads them
(``src/Calculators/bonded.py:65-89``) before the signed scatter of ``combiner.py:38-39``.

Here every rank (one process per GPU, ``torch.distributed``) owns a static shard of fragments, evaluates it
with its own engine, scatters the signed fragment forces into a local whole-protein buffer
``[3*N_prot + 1]`` (last slot = sum of signed fragment energies) on the device, and a single
``all_reduce(SUM)`` (NCCL over NVLink / NVSwitch; gloo in the CPU tests of the host logic) combines the
shards.  Fragments are independent, so this is the only collective on the path.
"""
from __future__ import annotations

from typing import Callable, List, Sequence, Tuple

import numpy as np

from .fragment_data import FragmentData
from .pdbfrag import ProteinMap


def partition_fragments(start: Sequence[int], end: Sequence[int], n_parts: int) -> List[Tuple[int, int]]:
    """Contiguous fragment ranges [lo, hi) per part, balanced by atom count.

    Same rule as the reference: walk the parts in order, give each an equal share of the *remaining*
    atoms, and cut at the fragment boundary nearest to that share (ties towards the earlier boundary);
    the last part takes the rest.  Parts may be empty when there are fewer fragments than parts."""
    start = np.asarray(start, dtype=np.int64)
    end = np.asarray(end, dtype=np.int64)
    n_frag = len(start)
    out: List[Tuple[int, int]] = []
    lo = 0
    for p in range(n_parts):
        if lo >= n_frag:
            out.append((n_frag, n_frag))
            continue
        if p == n_parts - 1:
            out.append((lo, n_frag))
            lo = n_frag
            continue
        remaining = int(end[-1] - start[lo])
        target = int(start[lo]) + remaining // (n_parts - p)
        hi = int(np.searchsorted(start, target, side="right"))      # first fragment starting after the target
        last = hi - 1                                                 # fragment containing the target
        if last >= lo and (target - int(start[last])) < (int(end[last]) - target):
            hi = last                                                 # target nearer to its start: leave it to the next part
        hi = max(hi, lo)
        hi = min(hi, n_frag)
        out.append((lo, hi))
        lo = hi
    return out


def chunk_fragments(start: Sequence[int], end: Sequence[int], chunk_atoms: int) -> List[Tuple[int, int]]:
    """Contiguous fragment ranges [lo, hi) of about ``chunk_atoms`` atoms each: the chunk loop of the reference's
    ``_set_combined_work_partitions`` (``--chunk-size``), applied to one block of packed fragments.

    The rule is the engine's own (``vb_chunk_fragments`` of the C library, which ``Engine(chunk_atoms=...)`` runs): each
    chunk ends at the fragment boundary nearest to ``start[lo] + chunk_atoms``.  Every chunk takes at least one fragment
    and one atom, where the reference would loop forever; fragments without atoms go with the chunk they fall in.
    ``chunk_atoms = 0`` is one chunk.  The fragments must be packed (``end[g] == start[g + 1]``)."""
    import ctypes as C
    from .engine import load_library
    start = np.asarray(start, dtype=np.int64)
    end = np.asarray(end, dtype=np.int64)
    if int(chunk_atoms) < 0:
        raise ValueError(f"chunk_atoms must be >= 0, not {chunk_atoms}")
    if len(start) == 0 or len(start) != len(end) or (start[1:] != end[:-1]).any():
        raise ValueError("start / end must describe a non-empty run of packed fragments")
    offsets = np.ascontiguousarray(np.append(start, end[-1]) - start[0])
    bounds = np.zeros(len(start) + 1, dtype=np.int64)
    lib = load_library()
    n = lib.vb_chunk_fragments(len(start), offsets.ctypes.data_as(C.c_void_p), int(chunk_atoms),
                               bounds.ctypes.data_as(C.c_void_p))
    if n < 1:
        raise ValueError(f"vb_chunk_fragments rejected the fragments ({n})")
    return [(int(bounds[c]), int(bounds[c + 1])) for c in range(n)]


def mm_rows(n_protein: int, rank: int, world_size: int) -> Tuple[int, int]:
    """The destination atoms [lo, hi) of the MM term one rank computes: an even split of the protein atoms."""
    return n_protein * rank // world_size, n_protein * (rank + 1) // world_size


def check_shardable(frags: FragmentData, world_size: int):
    """Every rank needs a block of fragments to hold an engine; raises ``ValueError`` when
    :func:`partition_fragments` leaves a rank without one."""
    parts = partition_fragments(frags.start, frags.end, world_size)
    empty = [r for r, (lo, hi) in enumerate(parts) if hi <= lo]
    if empty:
        raise ValueError(f"{len(frags)} fragments over {world_size} ranks leave rank(s) {empty} without a block")


def shard_protein_map(pm: ProteinMap, frags: FragmentData, lo: int, hi: int) -> ProteinMap:
    """Restrict the signed force map to fragments [lo, hi), re-basing fragment-atom indices to the shard."""
    if hi <= lo:
        return ProteinMap(pm.n_protein, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32),
                          np.zeros(0, np.float32))
    a0, a1 = int(frags.start[lo]), int(frags.end[hi - 1])
    keep = (pm.src_atom >= a0) & (pm.src_atom < a1)
    return ProteinMap(pm.n_protein, (pm.src_atom[keep] - a0).astype(np.int32), pm.dst_atom[keep].astype(np.int32),
                      pm.sign[keep].astype(np.float32), pm.frag_sign[lo:hi].astype(np.float32))


def combine_local(pm: ProteinMap, energy: np.ndarray, forces: np.ndarray) -> np.ndarray:
    """Host restatement of the device epilogue: local [3*N_prot + 1] buffer of one shard."""
    ef = np.zeros(3 * pm.n_protein + 1, dtype=np.float64)
    if len(pm.src_atom):
        np.add.at(ef[:-1].reshape(-1, 3), pm.dst_atom, pm.sign[:, None].astype(np.float64) * forces[pm.src_atom])
    ef[-1] = float(np.sum(pm.frag_sign.astype(np.float64) * np.asarray(energy, dtype=np.float64).reshape(-1)))
    return ef.astype(np.float32)


class ShardedBondedCalculator:
    """Whole-protein bonded energy/forces from a sharded fragment batch.

    ``evaluate_shard(frag_shard) -> (e[G_local], f[N_local,3])`` is the per-rank evaluator; on GPUs it is
    the engine (see :func:`make_engine_evaluator`), in the gloo CPU tests a stand-in.  ``all_reduce`` is
    ``torch.distributed.all_reduce`` when a process group is initialised, identity otherwise."""

    def __init__(self, frags: FragmentData, pm: ProteinMap, rank: int, world_size: int):
        self.rank, self.world_size = rank, world_size
        self.parts = partition_fragments(frags.start, frags.end, world_size)
        self.lo, self.hi = self.parts[rank]
        self.n_protein = pm.n_protein
        self.local_map = shard_protein_map(pm, frags, self.lo, self.hi)
        self.atom_lo = int(frags.start[self.lo]) if self.hi > self.lo else 0
        self.atom_hi = int(frags.end[self.hi - 1]) if self.hi > self.lo else 0

    def local_fragments(self, frags: FragmentData):
        return frags[self.lo:self.hi] if self.hi > self.lo else None

    def reduce_host(self, ef_local: np.ndarray) -> np.ndarray:
        import torch
        import torch.distributed as dist
        t = torch.from_numpy(np.ascontiguousarray(ef_local))
        if dist.is_available() and dist.is_initialized() and self.world_size > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return t.numpy()

    def evaluate_host(self, frags: FragmentData, evaluate_shard: Callable) -> Tuple[float, np.ndarray]:
        local = self.local_fragments(frags)
        if local is None:
            ef = np.zeros(3 * self.n_protein + 1, dtype=np.float32)
        else:
            e, f = evaluate_shard(local)
            ef = combine_local(self.local_map, np.asarray(e).reshape(-1), np.asarray(f).reshape(-1, 3))
        ef = self.reduce_host(ef)
        return float(ef[-1]), ef[:-1].reshape(-1, 3)


class DeviceShard:
    """Device-resident shard: engine + protein map + persistent torch buffers; one all-reduce per step.

    With ``native_comm`` (default) the ranks exchange CUDA IPC handles once (``torch.distributed`` is only the host
    transport for those 64 bytes) and every evaluation then ends with the engine's own one-shot all-reduce over NVLink
    peer memory, captured in the step's CUDA graph (``csrc/k_comm.cuh``).  If peer mapping is not possible on this box
    the ranks fall back -- together -- to ``torch.distributed.all_reduce`` (NCCL) enqueued after the evaluation.

    ``chunk_atoms`` > 0 evaluates the rank's block in chunks of about that many atoms (``Engine(chunk_atoms=...)``): the
    reference's order, blocks per device first, then chunks inside each block."""

    def __init__(self, state_dict, frags: FragmentData, pm: ProteinMap, rank: int, world_size: int, device: int,
                 native_comm: bool = True, chunk_atoms: int = 0):
        import torch
        from .engine import Engine
        self.torch = torch
        self.plan = ShardedBondedCalculator(frags, pm, rank, world_size)
        self.device = torch.device("cuda", device)
        self.ef = torch.zeros(3 * pm.n_protein + 1, dtype=torch.float32, device=self.device)
        self.engine = None
        self.comm_engine = None
        self.native = False
        local = self.plan.local_fragments(frags)
        if local is not None:
            self.engine = Engine(state_dict, device, chunk_atoms=chunk_atoms)
            self.engine.set_topology(local.z, local.batch, n_graphs=len(local))
            m = self.plan.local_map
            self.engine.set_protein_map(m.n_protein, m.src_atom, m.dst_atom, m.sign, m.frag_sign)
            self.pos = torch.from_numpy(np.ascontiguousarray(local.pos, dtype=np.float32)).to(self.device)
            # one evaluation of the start geometry, then plan the edge-tile length from its real edge count
            e0 = torch.empty(len(local), dtype=torch.float32, device=self.device)
            f0 = torch.empty((len(local.z), 3), dtype=torch.float32, device=self.device)
            self.engine.forward_device(self.pos.data_ptr(), e0.data_ptr(), f0.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
            self.engine.set_option("calibrate", 1)
        if world_size > 1 and native_comm:
            import torch.distributed as dist
            self.comm_engine = self.engine if self.engine is not None else Engine(state_dict, device)   # empty shard: comm only
            ok = 1
            try:
                handle = self.comm_engine.comm_init(rank, world_size, 3 * pm.n_protein + 1)
            except RuntimeError:
                handle, ok = b"\0" * 64, 0
            handles = [None] * world_size
            dist.all_gather_object(handles, handle)
            if ok:
                try:
                    self.comm_engine.comm_connect(handles)
                except RuntimeError:
                    ok = 0
            flag = torch.tensor([ok], dtype=torch.int32, device=self.device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)          # all ranks use the peer-memory path, or none does
            self.native = bool(int(flag.item()))
            if not self.native:
                self.comm_engine.set_option("comm_auto", 0)

    def set_window(self, frags: FragmentData, pm: ProteinMap, recipe, caph=None, nonbonded=None):
        """Make this rank place and refine the WHOLE batch, as the reference does on one device before it splits the
        fragments (``bonded.py:64-110``), and evaluate its own block of it (``vb_set_batch_window``): the window, then the
        whole placement ``recipe`` and the whole :class:`ai2bmd_b200.caph.CapHProblem` ``caph`` (optional).  Every rank's
        placed and refined batch is bit-identical to a single-GPU handle's.  ``nonbonded = (charges, sigmas, epsilons)``
        (optional) sets this rank's rows of the MM term, :func:`mm_rows`, with the exclusions ``FragmentCalculator`` uses.
        A rank without fragments has no engine and cannot take part: :func:`check_shardable` refuses that case."""
        from .nonbonded import check_parameters, dipeptide_atom_sets, exclusion_table
        eng = self.engine
        eng.set_batch_window(len(frags.z), self.plan.atom_lo)
        eng.set_fragment_recipe(recipe.real, recipe.acc, recipe.rem, recipe.blen)
        if caph is not None:
            eng.set_caph(caph)
        if nonbonded is not None:
            q, sg, ep = check_parameters(nonbonded, pm.n_protein)
            rowptr, col = exclusion_table(pm.n_protein, dipeptide_atom_sets(frags, recipe, pm))
            eng.set_nonbonded(q, sg, ep, rowptr, col, *mm_rows(pm.n_protein, self.plan.rank, self.plan.world_size))

    @property
    def collective(self) -> str:
        if self.plan.world_size == 1:
            return "none (single GPU)"
        return ("one-shot all-reduce over NVLink peer memory, last kernel of the step graph (k_comm.cuh)" if self.native
                else "torch.distributed.all_reduce (NCCL), enqueued by the host after the step graph")

    def set_positions(self, frag_pos_host: np.ndarray):
        """Upload this rank's slice of the packed fragment positions (pinned -> device)."""
        if self.engine is not None:
            sl = frag_pos_host[self.plan.atom_lo:self.plan.atom_hi]
            self.pos.copy_(self.torch.from_numpy(np.ascontiguousarray(sl, dtype=np.float32)), non_blocking=True)

    def step(self, all_reduce: bool = True):
        """Evaluate the local shard and all-reduce the whole-protein buffer (asynchronous on the current stream)."""
        torch = self.torch
        stream = torch.cuda.current_stream(self.device).cuda_stream
        if self.engine is not None:
            self.engine.forward_protein_device(self.pos.data_ptr(), self.ef.data_ptr(), stream)   # native: reduces too
        else:
            self.ef.zero_()
            if self.native and all_reduce:
                self.comm_engine.comm_allreduce(self.ef.data_ptr(), self.ef.numel(), stream)
        if all_reduce and self.plan.world_size > 1 and not self.native:
            import torch.distributed as dist
            dist.all_reduce(self.ef, op=dist.ReduceOp.SUM)
        return self.ef
