"""The reference's Calculator surface over the H100 engine.

Mirrors, name for name, the classes of ``/root/reference/src/Calculators`` that sit on the hot path:

* :class:`ViSNetModel`        <- ``visnet_calculator.py:22-75``  (``dl_potential_loader``, ``from_file``)
* :func:`get_visnet_model`    <- ``visnet_calculator.py:184-204``
* :class:`ViSNetCalculator`   <- ``visnet_calculator.py:121-155`` (un-fragmented ``--mode visnet``)
* :class:`DipeptideBondedCombiner` <- ``combiner.py:11-41``
* :class:`DLBondedCalculator` <- ``bonded.py:19-123`` (fragment-batch evaluation + combine)
* :class:`FragmentCalculator` <- ``fragment.py:16-68`` (placement, hydrogen refinement, bonded + MM term in one device call,
  on one GPU or, with ``devices``, on a group of them: ``bonded.py:64-89``; energies alone with ``derivative=False``)

ASE is not a dependency: calculators expose ``calculate(atoms, ...)`` / ``get_potential_energy`` /
``get_forces`` with ASE semantics (results cached while positions are unchanged,
``src/Calculators/calculator.py:9-23``) for any ``atoms`` object with ``.numbers`` and ``.positions``.
All compute goes through the C-ABI library; nothing here falls back to PyTorch or the CPU.
"""
from __future__ import annotations

import os.path as osp
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Optional, Tuple

import numpy as np

from .engine import Engine
from .fragment_data import FragmentData
from .weights import load_checkpoint, resolve_derivative


def _device_index(device: str) -> int:
    if device == "cpu":
        raise RuntimeError("the engine has no CPU path (device='cpu' requested)")
    if not device.startswith("cuda"):
        raise ValueError(f"Unrecognized device {device!r}")   # device_strategy.py:24-35
    return int(device.split(":")[1]) if ":" in device else 0


def _device_list(devices) -> Optional[List[str]]:
    """The ``devices`` argument of the multi-device calculators: a list or tuple of devices (duplicates allowed, e.g.
    ``["cuda:0", "cuda:0"]``; the reference's ``DeviceStrategy.get_bonded_devices()``) is returned as a list of strings,
    each checked as a device; None or one device is None, the single-device path."""
    if devices is None or not isinstance(devices, (list, tuple)):
        return None
    devs = [str(d) for d in devices]
    if not devs:
        raise ValueError("devices must name at least one device")
    for d in devs:
        _device_index(d)
    return devs


class ViSNetModel:
    """Energy and forces of a packed fragment batch with the ViSNet potential on one H100.

    ``derivative=False`` is the reference's ``ViSNet(derivative=False)``: energies only, on a forward-only engine
    (``dl_potential_loader`` returns ``(e, None)``).  ``chunk_size`` is the reference's ``--chunk-size``: the batch is
    evaluated in contiguous fragment chunks of about that many atoms on one workspace sized for the largest chunk
    (``Engine(chunk_atoms=...)``); None or 0 evaluates it in one pass."""

    implemented_properties = ["energy", "forces"]

    def __init__(self, state_dict: Dict[str, np.ndarray], device: str = "cuda:0", derivative: bool = True,
                 chunk_size: Optional[int] = None):
        self.device = device
        self.derivative = bool(derivative)
        self.engine = Engine(state_dict, _device_index(device), derivative=self.derivative, chunk_atoms=int(chunk_size or 0))
        self._topo_key = None
        if not self.derivative:
            self.implemented_properties = ["energy"]

    @classmethod
    def from_file(cls, **kwargs):
        """``from_file(model_path=..., device=..., derivative=None, chunk_size=None)``: ``derivative`` follows the
        reference's ``load_model(path, derivative=...)`` -- the checkpoint's hyper-parameter unless given (an ``.npz``
        counts as True)."""
        if "model_path" not in kwargs:
            raise ValueError("model_path must be provided")
        sd, ckpt_derivative = load_checkpoint(kwargs["model_path"])
        return cls(sd, device=kwargs.get("device", "cuda:0"),
                   derivative=resolve_derivative(ckpt_derivative, kwargs.get("derivative")),
                   chunk_size=kwargs.get("chunk_size"))

    @classmethod
    def from_engine(cls, engine: Engine, device: str, frag: FragmentData):
        """Wrap an engine whose topology is already ``frag``'s (e.g. a shard's engine with its protein map set)."""
        self = cls.__new__(cls)
        self.device, self.engine = device, engine
        self.derivative = engine.derivative
        if not self.derivative:
            self.implemented_properties = ["energy"]
        self._topo_key = self._key(frag)[0]
        self._calibrated = True
        return self

    @staticmethod
    def _key(frag: FragmentData):
        z = np.ascontiguousarray(frag.z, dtype=np.int64)
        batch = np.ascontiguousarray(frag.batch, dtype=np.int64)
        return (z.size, hash(z.tobytes()), hash(batch.tobytes())), z, batch

    def _ensure_topology(self, frag: FragmentData):
        # the same READ-ONLY z / batch arrays as last time cannot have changed: identity short-cuts the hash.  Writable arrays
        # are hashed every call (the reference re-uploads z and batch every call, so in-place edits must keep working)
        seen = getattr(self, "_topo_arrays", None)
        if seen is not None and seen[0] is frag.z and seen[1] is frag.batch:
            return
        key, z, batch = self._key(frag)
        if key != self._topo_key:
            self.engine.set_topology(z, batch, n_graphs=len(frag))
            self._topo_key = key
            self._calibrated = False
        frozen = (isinstance(frag.z, np.ndarray) and isinstance(frag.batch, np.ndarray)
                  and not frag.z.flags.writeable and not frag.batch.flags.writeable)
        self._topo_arrays = (frag.z, frag.batch) if frozen else None

    def dl_potential_loader(self, frag_data: FragmentData) -> Tuple[np.ndarray, Optional[np.ndarray]]:
        """``FragmentData -> (e[G,1] float32 eV, f[N,3] float32 eV/A)`` as numpy arrays; ``f`` is None on a
        ``derivative=False`` model (``visnet.py:166``)."""
        self._ensure_topology(frag_data)
        if self.derivative:
            e, f = self.engine.forward_host(frag_data.pos)
        else:
            e, f = self.engine.energy_host(frag_data.pos), None
        if not getattr(self, "_calibrated", True):      # once per topology: tile length from the real edge count
            self.engine.set_option("calibrate", 1)
            self._calibrated = True
        return e.reshape(-1, 1), f


_local_calc: Dict[str, ViSNetModel] = {}


def get_visnet_model(model_path: str, device: str, derivative: Optional[bool] = None,
                     chunk_size: Optional[int] = None) -> ViSNetModel:
    """One engine per (device, checkpoint[, derivative][, chunk size]); the reference's sub-process proxies
    (``ViSNetAsyncModel``) are unnecessary because every engine is in-process and asynchronous."""
    signature = f"{device}-{model_path}" if derivative is None else f"{device}-{model_path}-derivative={bool(derivative)}"
    if chunk_size:
        signature += f"-chunk_size={int(chunk_size)}"
    if signature not in _local_calc:
        _local_calc[signature] = ViSNetModel.from_file(model_path=model_path, device=device, derivative=derivative,
                                                       chunk_size=chunk_size)
    return _local_calc[signature]


class _CalculatorBase:
    """Minimal ASE-style result cache (``Calculator.get_property`` + patched ``check_state``)."""

    implemented_properties = ["energy", "forces"]

    def __init__(self):
        self.results: Dict[str, np.ndarray] = {}
        self._cached_pos: Optional[np.ndarray] = None

    def _changed(self, atoms) -> bool:
        pos = np.asarray(atoms.positions)
        return self._cached_pos is None or pos.shape != self._cached_pos.shape or not np.array_equal(pos, self._cached_pos)

    def get_property(self, name, atoms):
        if name not in self.implemented_properties:
            raise NotImplementedError(name)
        if self._changed(atoms) or name not in self.results:
            self.calculate(atoms, [name], ["positions"])
            self._cached_pos = np.array(atoms.positions, copy=True)
        return self.results[name]

    def get_potential_energy(self, atoms):
        return self.get_property("energy", atoms)

    def get_forces(self, atoms):
        return self.get_property("forces", atoms)


class ViSNetCalculator(_CalculatorBase):
    """Feed the input through the ViSNet model without fragmentation (one graph).

    ``derivative`` as in :meth:`ViSNetModel.from_file`; with ``derivative=False`` the calculator serves
    ``get_potential_energy`` only and ``get_forces`` raises ``NotImplementedError``."""

    def __init__(self, ckpt_path: str, ckpt_type: str, device: str = "cuda:0", is_root_calc=True,
                 derivative: Optional[bool] = None, chunk_size: Optional[int] = None, **kwargs):
        super().__init__()
        self.ckpt_path, self.ckpt_type, self.is_root_calc = ckpt_path, ckpt_type, is_root_calc
        model_path = osp.join(ckpt_path, f"visnet-uni-{ckpt_type}.ckpt")
        if not osp.exists(model_path) and osp.exists(ckpt_path) and osp.isfile(ckpt_path):
            model_path = ckpt_path
        self.device = device
        self.model = get_visnet_model(model_path, device, derivative, chunk_size)
        self.implemented_properties = list(self.model.implemented_properties)

    def calculate(self, atoms, properties, system_changes):
        n = len(atoms.numbers)
        data = FragmentData(np.asarray(atoms.numbers), np.asarray(atoms.positions).astype(np.float32),
                            np.array([0], dtype=int), np.array([n], dtype=int), np.zeros((n,), dtype=int))
        e, f = self.model.dl_potential_loader(data)
        self.results = {"energy": e} if f is None else {"energy": e, "forces": f}


class DipeptideBondedCombiner:
    """E = sum E_dipeptide - sum E_ACE-NME ; F = scatter_sum(cat[F_dip, -F_AN][select], origin)."""

    @staticmethod
    def energy_combine(dipeptides_energies: np.ndarray, acenmes_energies: np.ndarray) -> np.ndarray:
        return np.asarray(np.sum(dipeptides_energies, dtype=np.float32) - np.sum(acenmes_energies, dtype=np.float32))

    @staticmethod
    def forces_combine(num_atoms: int, dipeptides_forces, acenmes_forces, select_index, origin_index) -> np.ndarray:
        forces = np.concatenate([dipeptides_forces, -acenmes_forces])[select_index]
        out = np.zeros((num_atoms, 3), dtype=np.float32)
        np.add.at(out, origin_index, forces)
        return out


class DLBondedCalculator:
    """Fragment batch -> per-fragment (E, F) -> whole-protein (E, F).

    ``calculate(fragments)`` keeps the reference's return signature (``bonded.py:51-100``).  The
    whole-protein reduction can also run on the device through ``Engine.set_protein_map`` /
    ``forward_protein_device`` (used by ``parallel.ShardedBondedCalculator`` for the multi-GPU path).
    ``chunk_size`` is the reference's ``--chunk-size`` (``DeviceStrategy._chunk_size``): the engine evaluates the batch
    in fragment chunks of about that many atoms, one after the other on one bounded workspace (None: one pass).
    ``devices`` is the reference's multi-device ``calculate`` (``bonded.py:64-89``): a list of devices (duplicates
    allowed) gets one engine per entry, each evaluates its block of :func:`ai2bmd_b200.parallel.partition_fragments`
    from a thread pool (the engine calls release the GIL), and the results are concatenated in fragment order.  None or
    one device is the single-device path."""

    def __init__(self, ckpt_path: str, ckpt_type: str = "", device: str = "cuda:0", chunk_size: Optional[int] = None,
                 devices=None, **kwargs):
        model_path = osp.join(ckpt_path, f"visnet-uni-{ckpt_type}.ckpt") if ckpt_type else ckpt_path
        devs = _device_list(devices)
        if devs is None:
            self.models = [get_visnet_model(model_path, device if devices is None else str(devices), chunk_size=chunk_size)]
        else:            # one engine per entry, also for a device named twice: each keeps its own block's topology
            sd, ckpt_derivative = load_checkpoint(model_path)
            derivative = resolve_derivative(ckpt_derivative, None)
            self.models = [ViSNetModel(sd, device=d, derivative=derivative, chunk_size=chunk_size) for d in devs]
        if not self.models[0].derivative:
            raise ValueError(f"{model_path}: the bonded calculator needs forces, and the checkpoint has derivative=False")
        self.combiner = DipeptideBondedCombiner()

    def _evaluate(self, fragments: FragmentData):
        if len(self.models) == 1:
            return self.models[0].dl_potential_loader(fragments)
        from .parallel import partition_fragments
        parts = partition_fragments(fragments.start, fragments.end, len(self.models))
        jobs = [(m, fragments[lo:hi]) for m, (lo, hi) in zip(self.models, parts) if hi > lo]
        with ThreadPoolExecutor(len(jobs)) as pool:
            out = list(pool.map(lambda job: job[0].dl_potential_loader(job[1]), jobs))
        return np.concatenate([e for e, _ in out]), np.concatenate([f for _, f in out])

    def calculate(self, fragments: FragmentData):
        energy, forces = self._evaluate(fragments)
        dip_e, an_e = (energy[s] for s in fragments.scalar_split())
        dip_f, an_f = (forces[s] for s in fragments.vector_split())
        return dip_e, dip_f, an_e, an_f

    def combine(self, fragments: FragmentData, num_atoms: int, select_index, origin_index):
        dip_e, dip_f, an_e, an_f = self.calculate(fragments)
        return (self.combiner.energy_combine(dip_e, an_e),
                self.combiner.forces_combine(num_atoms, dip_f, an_f, select_index, origin_index))


def _check_nbcalc_type(nbcalc_type: str):
    if nbcalc_type == "pme":
        raise NotImplementedError("nbcalc_type='pme': the smooth-PME non-bonded term is not implemented on the device "
                                  "(DESIGN.md section 9); use 'mm'")
    if nbcalc_type != "mm":
        raise ValueError(f"nbcalc_type must be 'mm' or 'pme', not {nbcalc_type!r}")


def _check_derivative(derivative):
    if derivative is not None and not isinstance(derivative, (bool, np.bool_)):
        raise TypeError(f"derivative must be None, True or False, not {derivative!r}")


class FragmentCalculator(_CalculatorBase):
    """The reference's whole per-step calculator call (``FragmentCalculator.calculate``, ``src/Calculators/fragment.py:50-68``)
    as ONE engine call: protein positions in, the bonded (fragment) energy and forces plus the non-bonded MM term out,
    in eV and eV/A.  Everything between runs on the device in one graph replay (``vb_forward_fragments_host``): the
    fragment placement with the cap hydrogens (``DistanceFragment.get_fragments``), their LBFGS refinement, the model on
    every fragment, the signed dipeptide / ACE-NME combination (``DLBondedCalculator.__call__``) and
    ``MMNonBondedCalculator``, added as ``DipeptideCombiner`` does.  For any loop that keeps its own integrator: ASE's
    ``Langevin``, the QM/MM solvent mode (``AsyncQMMM``'s ``qmcalc``), or :class:`ai2bmd_b200.md.Langevin`.

    ``frags``, ``pm``, ``recipe``: the fragment batch, protein map and placement recipe of
    :func:`ai2bmd_b200.pdbfrag.fragment_protein` (``with_recipe=True``); :meth:`from_protein` builds them.  ``caph``: a
    :class:`ai2bmd_b200.caph.CapHProblem` turns the hydrogen refinement on.  ``nonbonded = (charges [e], sigmas [nm],
    epsilons [kJ/mol])`` per protein atom turns the MM term on, with the reference's exclusions (atoms sharing a
    dipeptide); without it the calculator is the reference's ``DLBondedCalculator.__call__``.  ``nbcalc_type`` is the
    reference's ``--fragment-longrange-calc``: ``"mm"`` only, ``"pme"`` raises ``NotImplementedError``.  ``chunk_size`` is
    the reference's ``--chunk-size`` (``Engine(chunk_atoms=...)``).  Arguments are checked before any engine is made.

    ``devices`` spreads the call over several GPUs of this process, as the reference's bonded devices do
    (``DeviceStrategy.get_bonded_devices()``, ``bonded.py:64-89``; the default ``--solvent`` run calls it from
    ``AsyncQMMM``'s worker thread): a list of devices (duplicates allowed, e.g. ``["cuda:0", "cuda:0"]``) builds one
    window engine per entry on its block of :func:`ai2bmd_b200.parallel.partition_fragments`, set up as a rank of the
    sharded path (:meth:`ai2bmd_b200.parallel.DeviceShard.set_window`: the whole placement and refinement, its own
    fragments, its rows of the MM term) and calibrated on the start geometry, joined by an
    :class:`ai2bmd_b200.engine.EngineGroup` that sums their buffers on the first device.  A list that leaves an entry
    without fragments is refused (:func:`ai2bmd_b200.parallel.check_shardable`).  None or one device is the
    single-device path; ``calculate`` is the same either way.

    ``derivative`` follows the reference's ``load_model(path, derivative=...)``: the checkpoint's hyper-parameter unless
    given (an ``.npz`` counts as True).  With ``derivative=False`` the calculator serves ``get_potential_energy`` only
    (``get_forces`` raises ``NotImplementedError``): every ``calculate`` runs the energy plan of the same call
    (``vb_forward_fragments_energy_host``), whose energy equals the full call's bit for bit, for conformer ranking,
    energy scans and Monte-Carlo acceptance tests.  On one device the engine is a forward-only one, with the smaller
    workspace; with ``devices`` the group's window engines stay full ones (so the workspace is not reduced there) and
    run the energy plan alone."""

    def __init__(self, ckpt_path: str, ckpt_type: str, frags: FragmentData, pm, recipe, caph=None, nonbonded=None,
                 nbcalc_type: str = "mm", device: str = "cuda:0", chunk_size: Optional[int] = None, devices=None,
                 derivative: Optional[bool] = None, **kwargs):
        super().__init__()
        _check_nbcalc_type(nbcalc_type)
        _check_derivative(derivative)
        from .engine import check_recipe
        real, acc, rem, blen = check_recipe(recipe.real, recipe.acc, recipe.rem, recipe.blen, len(frags.z))
        devs = _device_list(devices)
        if devs is None:
            device = device if devices is None else str(devices)
        else:
            from .parallel import check_shardable
            check_shardable(frags, len(devs))
        if nonbonded is not None:
            from .nonbonded import check_parameters, dipeptide_atom_sets, exclusion_table
            nonbonded = check_parameters(nonbonded, pm.n_protein)
            excl = exclusion_table(pm.n_protein, dipeptide_atom_sets(frags, recipe, pm)) if devs is None else None
        model_path = osp.join(ckpt_path, f"visnet-uni-{ckpt_type}.ckpt") if ckpt_type else ckpt_path
        sd, ckpt_derivative = load_checkpoint(model_path)
        self.derivative = resolve_derivative(ckpt_derivative, derivative)
        if not self.derivative:
            self.implemented_properties = ["energy"]
        self.n_protein = int(pm.n_protein)
        self.devices, self.shards, self.group = devs, None, None
        if devs is not None:
            from .engine import EngineGroup
            from .parallel import DeviceShard
            self.device, self.engine = devs[0], None
            self.shards = [DeviceShard(sd, frags, pm, r, len(devs), _device_index(d), native_comm=False,
                                       chunk_atoms=int(chunk_size or 0)) for r, d in enumerate(devs)]
            for sh in self.shards:
                sh.set_window(frags, pm, recipe, caph=caph, nonbonded=nonbonded)
            self.group = EngineGroup([sh.engine for sh in self.shards])
            self._target = self.group
            return
        self.device = device
        self.engine = eng = Engine(sd, _device_index(device), derivative=self.derivative, chunk_atoms=int(chunk_size or 0))
        eng.set_topology(frags.z, frags.batch, n_graphs=len(frags))
        eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
        start = np.asarray(frags.pos, dtype=np.float32)             # start geometry: real edge count for the tile plan
        if self.derivative:
            eng.forward_host(start)
        else:
            eng.energy_host(start)
        eng.set_option("calibrate", 1)
        eng.set_fragment_recipe(real, acc, rem, blen)
        if caph is not None:
            eng.set_caph(caph)
        if nonbonded is not None:
            eng.set_nonbonded(*nonbonded, *excl)
        self._target = eng

    @classmethod
    def from_protein(cls, ckpt_path: str, ckpt_type: str, prot, caph_tables=None, nonbonded=None, nbcalc_type: str = "mm",
                     device: str = "cuda:0", chunk_size: Optional[int] = None, devices=None,
                     derivative: Optional[bool] = None, **kwargs):
        """From a :class:`ai2bmd_b200.pdbfrag.CappedProtein`: fragmentation, protein map and recipe
        (``fragment_protein``), and with ``caph_tables`` (the per-dipeptide prmtop tables of
        :func:`ai2bmd_b200.caph.build_problem`) the hydrogen refinement; ``devices`` and ``derivative`` as in the
        constructor."""
        _check_nbcalc_type(nbcalc_type)
        _check_derivative(derivative)
        _device_list(devices)
        from .pdbfrag import fragment_protein
        frags, pm, recipe = fragment_protein(prot, with_recipe=True)
        caph = None
        if caph_tables is not None:
            from .caph import build_problem
            caph = build_problem(prot, frags, recipe, caph_tables)
        return cls(ckpt_path, ckpt_type, frags, pm, recipe, caph=caph, nonbonded=nonbonded, nbcalc_type=nbcalc_type,
                   device=device, chunk_size=chunk_size, devices=devices, derivative=derivative, **kwargs)

    def calculate(self, atoms, properties=("energy", "forces"), system_changes=("positions",)):
        if not self.derivative:
            self.results = {"energy": self._target.forward_fragments_energy_host(atoms.positions)}
            return None
        energy, forces = self._target.forward_fragments_host(atoms.positions)
        self.results = {"energy": energy, "forces": forces}
        return forces
