"""Minimal MD driver for the bonded (ViSNet fragment) potential -- the loop that drives the hot path.

The reference runs ASE's ``Langevin`` (``/root/reference/src/AIMD/simulator.py:96-137``: dt = 1 fs, 300 K,
friction 0.001 / fs, Maxwell-Boltzmann start) and asks ``FragmentCalculator`` for forces once per step.  ASE is
not available here, so this module restates that integrator (ASE 3.22 ``ase/md/langevin.py``, recalled; SURVEY
App. C) in numpy around :class:`BondedForceField`, which performs per step exactly what
``DLBondedCalculator.__call__`` does (``src/Calculators/bonded.py:102-123``) minus the cap-hydrogen LBFGS:

  protein positions -> fragment positions (cap hydrogens on the acceptor->removed ray, ``distancefrag.py:34-54``)
  -> engine (energies/forces of every fragment) -> signed reduction to whole-protein energy / forces.

friction = 0 gives velocity Verlet; its energy conservation is a physics check of the analytic forces
(``tests/test_md_gpu.py``).  Units follow ASE: eV, Angstrom, amu, time in Angstrom*sqrt(amu/eV).
"""
from __future__ import annotations

import numpy as np

from .elements import MASSES, masses_of   # noqa: F401  (MASSES: z -> amu, every z the model accepts)
from .engine import Engine
from .fragment_data import FragmentData
from .pdbfrag import FragmentRecipe, ProteinMap
from .restraints import KCALMOL_EV, PREEQ_SCHEDULE

FS = 0.09822694788464063        # 1 fs in ASE time units
KB = 8.617330337217213e-05      # eV / K


class BondedForceField:
    """Whole-protein bonded energy/forces from the fragment batch (device-side reduction)."""

    def __init__(self, state_dict, frags: FragmentData, pm: ProteinMap, recipe: FragmentRecipe, device: int = 0, refine=None):
        """``refine(frag_pos) -> frag_pos``: optional host-side refinement of the placed fragment coordinates (the parity
        tests pass the CPU restatement of the cap-hydrogen LBFGS here to check the device loop that runs it in-kernel)."""
        import torch
        self.torch = torch
        self.recipe, self.pm, self.refine = recipe, pm, refine
        self.engine = Engine(state_dict, device)
        self.engine.set_topology(frags.z, frags.batch, n_graphs=len(frags))
        self.engine.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
        self.engine.forward_host(np.asarray(frags.pos, dtype=np.float32))       # start geometry: real edge count for the tile plan
        self.engine.set_option("calibrate", 1)
        dev = torch.device("cuda", device)
        self.pos_host = torch.empty((len(frags.z), 3), dtype=torch.float32).pin_memory()
        self.pos_dev = torch.empty((len(frags.z), 3), dtype=torch.float32, device=dev)
        self.ef_dev = torch.empty(3 * pm.n_protein + 1, dtype=torch.float32, device=dev)
        self.ef_host = torch.empty(3 * pm.n_protein + 1, dtype=torch.float32).pin_memory()
        self.stream = torch.cuda.current_stream(dev)

    def __call__(self, prot_pos: np.ndarray):
        """(E [eV], F [n_protein,3] eV/A) for the given protein coordinates."""
        frag_pos = self.recipe.positions(prot_pos)
        if getattr(self, "refine", None) is not None:
            frag_pos = self.refine(frag_pos)
        self.pos_host.numpy()[:] = frag_pos
        self.pos_dev.copy_(self.pos_host, non_blocking=True)
        self.engine.forward_protein_device(self.pos_dev.data_ptr(), self.ef_dev.data_ptr(), self.stream.cuda_stream)
        self.ef_host.copy_(self.ef_dev, non_blocking=True)
        self.stream.synchronize()
        ef = self.ef_host.numpy()
        return float(ef[-1]), ef[:-1].reshape(-1, 3).astype(np.float64)


class Langevin:
    """ASE-style Langevin integrator, restating ``ase/md/langevin.py`` ``Langevin.step`` of ASE 3.22 with
    ``fixcm=True`` (recalled; ASE is not in the image): half-kick, drift, centre of mass put back where it was,
    velocities recomputed from the positions, forces, half-kick, centre-of-mass velocity removed.
    ``friction=0`` reduces to velocity Verlet (no random numbers, no centre-of-mass handling)."""

    def __init__(self, positions, numbers, force_fn, dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.001, seed=0,
                 normal_source=None, zero_com_momentum=False, noise="numpy"):
        """``normal_source(step) -> (xi, eta)`` overrides the numpy generator for the per-step normals (used to
        drive this host integrator with the device's Philox stream in the parity tests).  ``zero_com_momentum``
        removes the centre-of-mass momentum of the Maxwell-Boltzmann draw; the reference does not
        (``simulator.py:96`` calls ``MaxwellBoltzmannDistribution`` only, no ``Stationary``).

        ``noise="reference"`` draws as the reference does: the start velocities from ``np.random.RandomState(seed)``
        (:func:`reference_velocities`) and every step's xi, eta from ``np.random.default_rng(seed)`` in ``RNGPool``
        order, at friction 0 too (ASE's step draws regardless).  The default ``"numpy"`` takes both from one
        ``default_rng(seed)`` and draws nothing at friction 0."""
        if noise not in ("numpy", "reference"):
            raise ValueError(f"noise must be 'numpy' or 'reference', not {noise!r}")
        self.normal_source, self.noise = normal_source, noise
        self.nsteps = 0
        self.x = np.array(positions, dtype=np.float64)
        self.m = masses_of(numbers)[:, None]
        self.force_fn = force_fn
        self.dt = dt_fs * FS
        self.T = temperature_K * KB
        self.fr = friction_per_fs / FS
        self.rng = np.random.default_rng(seed)
        # Maxwell-Boltzmann start (simulator.py:96)
        if noise == "reference":
            self.v = reference_velocities(seed, self.m[:, 0], self.T)
        else:
            self.v = self.rng.standard_normal(self.x.shape) * np.sqrt(self.T / self.m)
        if zero_com_momentum:
            self.v -= (self.v * self.m).sum(0) / self.m.sum()
        self.energy, self.f = force_fn(self.x)
        dt, fr = self.dt, self.fr
        sigma = np.sqrt(2 * self.T * fr / self.m)
        self.c1 = dt / 2.0 - dt * dt * fr / 8.0
        self.c2 = dt * fr / 2 - dt * dt * fr * fr / 8.0
        self.c3 = np.sqrt(dt) * sigma / 2.0 - dt ** 1.5 * fr * sigma / 8.0
        self.c5 = dt ** 1.5 * sigma / (2 * np.sqrt(3))
        self.c4 = fr / 2.0 * self.c5

    def kinetic_energy(self):
        return 0.5 * float((self.m * self.v * self.v).sum())

    def temperature(self):
        return 2.0 * self.kinetic_energy() / (3 * len(self.x)) / KB

    def normals(self):
        """(xi, eta) of the current step: from ``normal_source``, else two draws of the numpy generator (0 at friction 0)."""
        if self.fr > 0 and self.normal_source is not None:
            return self.normal_source(self.nsteps)
        if self.noise == "reference":
            return self.rng.standard_normal(self.x.shape), self.rng.standard_normal(self.x.shape)
        xi = self.rng.standard_normal(self.x.shape) if self.fr > 0 else 0.0
        eta = self.rng.standard_normal(self.x.shape) if self.fr > 0 else 0.0
        return xi, eta

    def first_half(self, xi, eta):
        """Half-kick with the current forces, drift, centre of mass put back, velocities from the positions
        (the device's ``md_kick1_kernel``)."""
        self.v = self.v + (self.c1 * self.f / self.m - self.c2 * self.v + self.c3 * xi - self.c4 * eta)
        x_old = self.x
        self.x = self.x + self.dt * self.v + self.c5 * eta
        if self.fr > 0:     # fix_com: the centre of mass stays where it was before the drift (atoms.set_center_of_mass(old_com))
            msum = self.m.sum()
            self.x = self.x + ((self.m * x_old).sum(0) / msum - (self.m * self.x).sum(0) / msum)
        self.v = (self.x - x_old - self.c5 * eta) / self.dt

    def second_half(self, xi, eta):
        """Half-kick with the forces of the new positions, centre-of-mass velocity removed, step counter advanced
        (the device's ``md_kick2_kernel``)."""
        self.v = self.v + (self.c1 * self.f / self.m - self.c2 * self.v + self.c3 * xi - self.c4 * eta)
        if self.fr > 0:
            self.v -= (self.v * self.m).sum(0) / self.m.sum()
        self.nsteps += 1

    def step(self):
        xi, eta = self.normals()
        self.first_half(xi, eta)
        self.energy, self.f = self.force_fn(self.x)
        self.second_half(xi, eta)
        return self.energy

    def run(self, n_steps):
        for _ in range(n_steps):
            self.step()


def reference_velocities(seed: int, masses, kT: float):
    """The reference's start velocities: ASE's ``MaxwellBoltzmannDistribution(atoms, temperature_K,
    rng=np.random.RandomState(seed))`` (``simulator.py:96``; ASE 3.22, recalled, not pinned), i.e. one
    ``standard_normal((n, 3))`` of the legacy generator scaled by sqrt(kT / m)."""
    m = np.asarray(masses, dtype=np.float64)[:, None]
    return np.random.RandomState(seed).standard_normal((len(m), 3)) * np.sqrt(kT / m)


# ---------------------------------------------------------------------------------------------------------
# device-resident integrator (csrc/k_md.cuh behind include/visnet_b200.h vb_md_*)
# ---------------------------------------------------------------------------------------------------------
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on arrays of 32-bit words held in uint64; returns the four output words."""
    m32 = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = (np.atleast_1d(np.asarray(c, dtype=np.uint64)) for c in np.broadcast_arrays(c0, c1, c2, c3))
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & m32, p1 & m32, ((p0 >> np.uint64(32)) ^ c3 ^ k1) & m32, p0 & m32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m32, (k1 + np.uint64(0xBB67AE85)) & m32
    return c0, c1, c2, c3


def philox_normals(seed: int, step: int, n_components: int):
    """Host restatement of the device's per-step normals (k_md.cuh ``md_normals``): Philox4x32-10 with counter
    (component, step_lo, step_hi, 0) and key (seed_lo, seed_hi), two 53-bit uniforms in (0, 1], Box-Muller.
    Returns (xi, eta), each ``[n_components]`` float64."""
    c0, c1, c2, c3 = philox4x32_10(np.arange(n_components, dtype=np.uint64), step & 0xFFFFFFFF, (step >> 32) & 0xFFFFFFFF, 0,
                                   seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    u1 = ((((c0 << np.uint64(32)) | c1) >> np.uint64(11)).astype(np.float64) + 1.0) / 9007199254740992.0
    u2 = ((((c2 << np.uint64(32)) | c3) >> np.uint64(11)).astype(np.float64) + 1.0) / 9007199254740992.0
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2.0 * np.pi * u2), r * np.sin(2.0 * np.pi * u2)


class DeviceLangevin:
    """The same integrator with positions, velocities, cap-hydrogen placement and the force evaluation all on the
    GPU: ``run(n)`` enqueues n replays of one captured CUDA graph and never touches the host.

    With ``group`` (a ``torch.distributed`` process group, one rank per GPU) every rank holds the whole-protein state
    and its own shard of fragments; the per-step exchange is the one all-reduce of the force/energy buffer.
    :meth:`grouped` runs the step over several GPUs of ONE process instead (an :class:`ai2bmd_b200.engine.EngineGroup`)."""

    engine_group = None      # grouped(): the EngineGroup whose members evaluate every step of this engine's state

    def __init__(self, state_dict, frags: FragmentData, pm: ProteinMap, recipe: FragmentRecipe, positions, numbers,
                 dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.001, seed=0, device: int = 0, velocities=None,
                 group=None, engine: Engine = None, zero_com_momentum=False, caph=None, step: int = 0,
                 chunk_atoms: int = 0, noise: str = "philox", noise_state: int = None):
        """``caph``: an :class:`ai2bmd_b200.caph.CapHProblem` -- the added hydrogens are then refined every step on the
        device (one LBFGS call on the Amber terms, ``csrc/k_caph.cuh``) between their placement and the evaluation.
        ``step``: the step counter to start from; with ``positions`` / ``velocities`` of a frame that ``run_observed``
        recorded at step s, the run continues with the random numbers the original run drew after s.
        ``chunk_atoms``: the engine this creates evaluates the fragments in chunks of about that many atoms
        (``Engine(chunk_atoms=...)``); the step stays one graph replay.
        ``noise``: ``"philox"`` (default) draws the step's normals from the counter-based Philox stream keyed by
        (seed, step); ``"reference"`` draws exactly the numbers the reference's ``RNGPool(seed)`` hands ASE's Langevin
        (numpy's ``default_rng(seed)``, generated on the device, :mod:`ai2bmd_b200.refnoise`), and the default start
        velocities are the reference's (:func:`reference_velocities`).  Its stream starts from ``PCG64(seed)`` unless
        ``noise_state`` (a 128-bit state from :meth:`noise_state`) is given: like the reference's ``--restart``, which
        builds a fresh ``RNGPool(seed)``, a run started from a recorded frame reseeds unless it is handed the saved
        state.  Every rank of a sharded run generates the same stream."""
        if noise not in ("philox", "reference"):
            raise ValueError(f"noise must be 'philox' or 'reference', not {noise!r}")
        import torch
        self.torch, self.group = torch, group
        self.n = pm.n_protein
        self.masses = masses_of(numbers)
        self.kT = temperature_K * KB
        self.fr = friction_per_fs / FS
        dev = torch.device("cuda", device)
        if engine is None:
            engine = Engine(state_dict, device, chunk_atoms=chunk_atoms)
            engine.set_topology(frags.z, frags.batch, n_graphs=len(frags))
            engine.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
            engine.forward_host(np.asarray(frags.pos, dtype=np.float32))
            engine.set_option("calibrate", 1)
        self.engine = engine
        if caph is not None:
            engine.set_caph(caph)
        self.ef = torch.zeros(3 * self.n + 1, dtype=torch.float32, device=dev)
        self.stream = torch.cuda.current_stream(dev)
        engine.md_setup(self.masses, recipe.real, recipe.acc, recipe.rem, recipe.blen, dt_fs * FS, self.kT, self.fr,
                        seed, self.ef.data_ptr())
        self._start(positions, velocities, seed, step, noise, noise_state, zero_com_momentum)

    @classmethod
    def sharded(cls, state_dict, frags: FragmentData, pm: ProteinMap, recipe: FragmentRecipe, positions, numbers, group, *,
                caph=None, nonbonded=None, chunk_atoms: int = 0, native_comm: bool = True, device: int = None, **kwargs):
        """This rank's part of a step sharded over ``group`` (one rank per GPU) with the hydrogen refinement and the MM
        term: the reference's step on several devices.  The rank's :class:`ai2bmd_b200.parallel.DeviceShard` evaluates
        its block of fragments (``partition_fragments``), but places and refines the WHOLE batch first
        (``DeviceShard.set_window``), so every rank refines exactly what one GPU would; ``caph`` is the whole batch's
        :class:`ai2bmd_b200.caph.CapHProblem` and ``recipe`` the whole batch's.  ``nonbonded = (charges, sigmas,
        epsilons)`` adds the MM term, each rank computing an even split of its rows (``parallel.mm_rows``).  The ranks
        combine the force buffer with the engine's own all-reduce inside the step graph (``native_comm``; NCCL between
        the kicks where peer memory is unavailable).  ``device`` defaults to the current CUDA device; the other keyword
        arguments are the constructor's.  A recipe or MM parameters of the wrong length, or more ranks than blocks,
        raise ``ValueError`` before any engine is made."""
        from .engine import check_recipe
        from .nonbonded import check_parameters
        from .parallel import DeviceShard, check_shardable
        check_recipe(recipe.real, recipe.acc, recipe.rem, recipe.blen, len(frags.z))
        if nonbonded is not None:
            check_parameters(nonbonded, pm.n_protein)
        import torch
        import torch.distributed as dist
        world = dist.get_world_size(group)
        check_shardable(frags, world)
        device = torch.cuda.current_device() if device is None else int(device)
        sh = DeviceShard(state_dict, frags, pm, dist.get_rank(group), world, device, native_comm=native_comm,
                         chunk_atoms=chunk_atoms)
        sh.set_window(frags, pm, recipe, caph=caph, nonbonded=nonbonded)
        self = cls(None, None, pm, recipe, positions, numbers, device=device, group=group, engine=sh.engine, **kwargs)
        self.shard = sh
        return self

    @classmethod
    def grouped(cls, state_dict, frags: FragmentData, pm: ProteinMap, recipe: FragmentRecipe, positions, numbers, *,
                devices, caph=None, nonbonded=None, chunk_atoms: int = 0, dt_fs=1.0, temperature_K=300.0,
                friction_per_fs=0.001, seed=0, velocities=None, zero_com_momentum=False, step: int = 0,
                noise: str = "philox", noise_state: int = None):
        """The step over several GPUs of this process, as the reference's single-process run spreads each step's
        fragments over its bonded devices (``DLBondedCalculator.calculate``, ``src/Calculators/bonded.py:64-89``).
        ``devices`` is the list ``FragmentCalculator(devices=...)`` takes (duplicates allowed, e.g. ``["cuda:0"] * 2``),
        and the window engines are built as it builds them: one per entry on its block of
        :func:`ai2bmd_b200.parallel.partition_fragments`, each placing and refining the whole batch (``caph``, the whole
        :class:`ai2bmd_b200.caph.CapHProblem`) and evaluating its block and its rows of the MM term (``nonbonded``).
        Member 0 (``devices[0]``) holds the MD state and integrates; every step is one launch of the group's step graph
        (``vb_group_md_run``).  The other keyword arguments are the constructor's.

        ``run``, ``run_observed``, ``preequilibrate``, ``set_restraints``, ``set_normals``, ``state``, ``energy``,
        ``temperature`` and ``noise_state`` work as on one GPU, on member 0's engine (``self.engine``; the members are
        ``self.shards``).  ``run_segment`` raises: its device loop runs one engine's step."""
        from .calculator import _device_index, _device_list
        from .engine import EngineGroup, check_recipe
        from .nonbonded import check_parameters
        from .parallel import DeviceShard, check_shardable
        if noise not in ("philox", "reference"):
            raise ValueError(f"noise must be 'philox' or 'reference', not {noise!r}")
        devs = _device_list(devices)
        if devs is None:
            raise ValueError("devices must be a list of devices, e.g. ['cuda:0', 'cuda:1']")
        check_recipe(recipe.real, recipe.acc, recipe.rem, recipe.blen, len(frags.z))
        check_shardable(frags, len(devs))
        if nonbonded is not None:
            check_parameters(nonbonded, pm.n_protein)
        import torch
        self = cls.__new__(cls)
        self.torch, self.group = torch, None
        self.n = pm.n_protein
        self.masses = masses_of(numbers)
        self.kT = temperature_K * KB
        self.fr = friction_per_fs / FS
        self.shards = [DeviceShard(state_dict, frags, pm, r, len(devs), _device_index(d), native_comm=False,
                                   chunk_atoms=chunk_atoms) for r, d in enumerate(devs)]
        for sh in self.shards:
            sh.set_window(frags, pm, recipe, caph=caph, nonbonded=nonbonded)
        self.engine = self.shards[0].engine
        dev = torch.device("cuda", self.engine.device)
        self.ef = torch.zeros(3 * self.n + 1, dtype=torch.float32, device=dev)
        self.stream = torch.cuda.current_stream(dev)
        self.engine.md_setup(self.masses, recipe.real, recipe.acc, recipe.rem, recipe.blen, dt_fs * FS, self.kT, self.fr,
                             seed, self.ef.data_ptr())
        self.engine_group = EngineGroup([sh.engine for sh in self.shards])     # after md_setup: it replaces the recipe
        self._start(positions, velocities, seed, step, noise, noise_state, zero_com_momentum)
        return self

    @classmethod
    def unfragmented(cls, state_dict, numbers, positions, *, dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.001,
                     seed=0, device: int = 0, velocities=None, step: int = 0, noise: str = "philox",
                     noise_state: int = None, chunk_atoms: int = 0, zero_com_momentum=False, group=None):
        """The reference's ``--mode visnet`` run on the device: the whole input is ONE ViSNet graph
        (``ViSNetCalculator``, ``src/Calculators/visnet_calculator.py:138-155``) -- no fragments, no cap hydrogens, no
        protein map, no MM term -- inside the same device step (``vb_md_setup`` with no placement recipe).  The
        reference sends every input of three or fewer residues (caps counted) here, e.g. an ACE-X-NME dipeptide.

        ``numbers`` / ``positions`` are the input's atoms in file order (:func:`ai2bmd_b200.pdbfrag.whole_input`).  The
        other arguments and the run protocol (``run``, ``run_observed``, ``preequilibrate``, ``set_restraints``,
        ``state``, ``noise_state``, ``temperature``, ``set_normals``) are those of the fragment step.  One graph is not
        sharded: ``group`` raises."""
        if group is not None:
            raise ValueError("DeviceLangevin.unfragmented runs one graph on one GPU: it cannot be sharded over a process group")
        if noise not in ("philox", "reference"):
            raise ValueError(f"noise must be 'philox' or 'reference', not {noise!r}")
        z = np.asarray(numbers, dtype=np.int64).reshape(-1)
        x = np.asarray(positions, dtype=np.float64)
        if x.shape != (len(z), 3):
            raise ValueError(f"positions must be [{len(z)}, 3], one row per atom of numbers")
        import torch
        self = cls.__new__(cls)
        self.torch, self.group = torch, None
        self.n = len(z)
        self.masses = masses_of(z)
        self.kT = temperature_K * KB
        self.fr = friction_per_fs / FS
        dev = torch.device("cuda", device)
        engine = Engine(state_dict, device, chunk_atoms=chunk_atoms)
        engine.set_topology(z, np.zeros(len(z), dtype=np.int64), n_graphs=1)
        engine.forward_host(x.astype(np.float32))           # start geometry: real edge count for the tile plan
        engine.set_option("calibrate", 1)
        self.engine = engine
        self.ef = torch.zeros(3 * self.n + 1, dtype=torch.float32, device=dev)
        self.stream = torch.cuda.current_stream(dev)
        engine.md_setup_unfragmented(self.masses, dt_fs * FS, self.kT, self.fr, seed, self.ef.data_ptr())
        self._start(x, velocities, seed, step, noise, noise_state, zero_com_momentum)
        return self

    def _start(self, positions, velocities, seed, step, noise, noise_state, zero_com_momentum):
        """Noise source, start state and the forces of the start positions (after ``md_setup``)."""
        engine = self.engine
        if noise == "reference":
            from . import refnoise
            s0, inc = refnoise.pcg_state(seed)
            engine.md_set_noise(1, s0 if noise_state is None else int(noise_state), inc, refnoise.tables())
        x = np.array(positions, dtype=np.float64)
        if velocities is None:      # Maxwell-Boltzmann start, as Langevin above (simulator.py:96)
            m = self.masses[:, None]
            if noise == "reference":
                velocities = reference_velocities(seed, self.masses, self.kT)
            else:
                velocities = np.random.default_rng(seed).standard_normal(x.shape) * np.sqrt(self.kT / m)
            if zero_com_momentum:
                velocities -= (velocities * m).sum(0) / m.sum()
        engine.md_set_state(x, velocities, step)
        self._eval()
        self._copy_stream = None
        self._frame_bufs = {}

    @property
    def _native_comm(self):
        """True when the engine all-reduces the force buffer itself (peer-memory all-reduce inside the step graph)."""
        return self.group is not None and self.engine.get_option("comm_ready") == 1 and self.engine.get_option("comm_auto") == 1

    def _eval(self):
        sp = self.stream.cuda_stream
        if self.engine_group is not None:
            self.engine_group.md_eval(sp)
            return
        self.engine.md_eval(sp)
        if self.group is not None and not self._native_comm:
            self.torch.distributed.all_reduce(self.ef, group=self.group)

    def set_normals(self, pool):
        """Externally supplied normals ``[steps, 2, n, 3]`` (float64) instead of the Philox stream (tests)."""
        if pool is None:
            self._pool = None
            self.engine.md_set_normals(0, 0)
            return
        self._pool = self.torch.as_tensor(np.ascontiguousarray(pool, dtype=np.float64)).to(self.ef.device)
        self.engine.md_set_normals(self._pool.data_ptr(), self._pool.shape[0])

    def noise_state(self) -> int:
        """The 128-bit PCG64 state of the reference noise stream after the last step (``noise="reference"``;
        synchronises).  Hand it to a new ``DeviceLangevin(noise_state=...)`` to continue the stream."""
        return self.engine.md_get_noise_state()

    def run(self, n_steps: int):
        sp = self.stream.cuda_stream
        if self.engine_group is not None:                # every member's evaluation inside the group's step graph
            self.engine_group.md_run(n_steps, sp)
            return
        if self.group is None or self._native_comm:      # whole step (incl. the all-reduce) = one graph replay
            self.engine.md_run(n_steps, sp)
            return
        for _ in range(n_steps):
            self.engine.md_kick1(sp)
            self._eval()
            self.engine.md_kick2(sp)

    def run_segment(self, n_steps: int) -> int:
        """Up to ``n_steps`` steps as ONE launch of the device loop (``vb_md_run_loop``), waited for; returns the steps
        actually run.  The loop ends by itself at the step the recorder's runaway guard halts on (a recorder set with
        ``engine.md_set_recorder``), which raises :class:`TemperatureRunawayError` as ``run_observed`` does, and at the
        next step boundary after :meth:`request_stop`.  While the engine stays halted (until ``engine.md_set_state``)
        every call runs no step and raises again.  A ``KeyboardInterrupt`` during the wait asks the loop to stop, waits
        for it and re-raises, so the state is that of a whole step; in a sharded run, where the ranks could not agree on
        a stop step, it only waits for the launch to end (at ``n_steps`` or a halt) and re-raises.  Frames are not drained during the launch: read them
        afterwards with ``engine.md_read_frames``.  A sharded run needs the engine's own all-reduce: with the
        ``torch.distributed`` all-reduce between the kicks the step cannot loop on the device."""
        n_steps = int(n_steps)
        if n_steps < 0:
            raise ValueError(f"n_steps must be >= 0, not {n_steps}")
        if self.engine_group is not None:
            raise ValueError("run_segment's device loop runs one engine's step, and this step spans the members of an "
                             "EngineGroup; use run_observed (or run)")
        if self.group is not None and not self._native_comm:
            raise ValueError("run_segment needs the engine's own all-reduce inside the step graph: this run all-reduces "
                             "with torch.distributed between the kicks, which cannot run inside a device loop; use run()")
        import time
        torch = self.torch
        done = torch.cuda.Event()
        try:
            self.engine.md_run_loop(n_steps, self.stream.cuda_stream)
            done.record(self.stream)
            while not done.query():              # a sleep-poll, not synchronize(): a KeyboardInterrupt gets through
                time.sleep(2e-4)
        except KeyboardInterrupt:
            if self.group is None:               # a launch already enqueued ends at its next step boundary
                self.request_stop()
            self.stream.synchronize()            # sharded: no stop step is agreed between ranks, the launch runs out
            raise
        ran = self.engine.md_loop_iterations()
        halt = self.engine.get_option("md_halt_step")
        if halt >= 0:
            raise TemperatureRunawayError(f"temperature runaway at step {halt}: {self.temperature():.1f} K")
        return ran

    def request_stop(self):
        """Stop a running :meth:`run_segment` (or ``engine.md_run_loop``) at its next step boundary.  Safe to call from
        another thread while it waits; a sharded run refuses it (the ranks would stop at different steps)."""
        self.engine.md_request_stop()

    def state(self, n_hist: int = 0):
        """(positions, velocities, step, potential energies of the last n_hist steps); synchronises."""
        return self.engine.md_get_state(n_hist)

    @property
    def energy(self):
        self.stream.synchronize()
        return float(self.ef[-1].item())

    def kinetic_energy(self):
        _, v, _, _ = self.state()
        return 0.5 * float((self.masses[:, None] * v * v).sum())

    def temperature(self):
        return 2.0 * self.kinetic_energy() / (3 * self.n) / KB

    # ---- restraints and the reference's run protocol (simulator.py:139-180) ----
    def set_restraints(self, tether_atoms=None, tether_k_kcal=0.0, springs=None):
        """Hookean restraints inside the device step, replacing any set before: ``tether_atoms`` tied to where they stand
        now with ``tether_k_kcal`` kcal/mol/A^2, and ``springs = (ij [n,2], k [n] eV/A^2, rt [n] A)`` (e.g.
        :func:`ai2bmd_b200.restraints.hydrogen_bond_springs`).  No argument removes them.  Every rank of a sharded run
        makes the same call."""
        ij, k, rt = springs if springs is not None else (None, (), ())
        self.engine.md_set_restraints(() if tether_atoms is None else tether_atoms, tether_k_kcal * KCALMOL_EV, ij, k, rt)

    def run_observed(self, n_steps: int, record_per_steps=None, observer=None):
        """``run(n_steps)`` observed at every step number divisible by ``record_per_steps``: there, like the reference's
        ``MDObserver.printenergy`` (utils.py:143-159), the temperature is checked -- above 1.5 T0 raises
        :class:`TemperatureRunawayError` -- and ``observer(step, x, v, epot, ekin)`` is called, in step order, with the
        restrained potential energy of that step.

        The device records the frames and makes the runaway decision itself (``vb_md_set_recorder``); this loop only
        drains them.  It keeps at most ``max(2 record_per_steps, 64)`` steps enqueued beyond the last frame it handed to
        the observer, in blocks that each end with one asynchronous copy of their frames into pinned memory on a side
        stream, so the GPU steps on while the observer runs.  On a runaway the device stops at the halting step by
        itself, the observer is not called for it, and the engine stays halted (``state()`` is that step, ``run`` changes
        nothing) until ``engine.md_set_state``; otherwise the recorder is switched off again at the end."""
        if not record_per_steps:
            self.run(n_steps)
            return
        torch, k = self.torch, int(record_per_steps)
        _, _, step, _ = self.state()
        end = step + n_steps
        ahead = max(2 * k, 64)                       # steps enqueued beyond the last drained block, at most
        block = max(k, ahead // 2 // k * k)          # blocks end at multiples of `block` (itself a multiple of k) and at `end`
        # a block's frames are copied out before the lookahead lets later steps reuse their slots
        self.engine.md_set_recorder(k, (ahead + block) // k + 2, RUNAWAY_FACTOR)
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(self.ef.device)
        copy, free = self._copy_stream, self._frame_bufs.setdefault(block // k, [])
        inflight, frame, enq, drained, halted = [], 0, step, step, False
        try:
            while drained < end:
                while enq < end and (not inflight or min(end, (enq // block + 1) * block) - drained <= ahead):
                    nxt = min(end, (enq // block + 1) * block)
                    self.run(nxt - enq)
                    nf = nxt // k - enq // k
                    enq = nxt
                    buf = free.pop() if free else _FrameBuffers(torch, block // k, self.n)
                    ran = torch.cuda.Event()
                    ran.record(self.stream)
                    copy.wait_event(ran)
                    if nf:
                        self.engine.md_read_frames_async(frame, nf, *buf.ptrs, copy.cuda_stream)
                    copied = torch.cuda.Event()
                    copied.record(copy)
                    inflight.append((copied, nf, nxt, buf))
                    frame += nf
                copied, nf, nxt, buf = inflight.pop(0)
                copied.synchronize()
                for i in range(nf):
                    if buf.halted[i]:
                        temp = 2.0 * buf.ekin[i] / (3 * self.n) / KB
                        halted = True
                        raise TemperatureRunawayError(f"temperature runaway at step {int(buf.step[i])}: {temp:.1f} K")
                    if observer is not None:
                        x, v = buf.x[i].copy(), buf.v[i].copy()
                        observer(int(buf.step[i]), x, v, float(buf.epot[i]), 0.5 * float((self.masses[:, None] * v * v).sum()))
                drained = nxt
                free.append(buf)
        finally:
            copy.synchronize()                       # no copy may still write a buffer that goes back to the pool
            free.extend(b for _, _, _, b in inflight)
            if not halted:
                self.engine.md_set_recorder(0)

    def preequilibrate(self, steps_per_stage: int, schedule=PREEQ_SCHEDULE, atoms=None, record_per_steps=None, observer=None):
        """The reference's pre-equilibration: for each force constant of ``schedule`` (kcal/mol/A^2, the reference's
        :data:`ai2bmd_b200.restraints.PREEQ_SCHEDULE`) tether ``atoms`` (default: every protein atom) to where they stand
        at the start of the stage, run ``steps_per_stage`` steps (``run_observed``), and remove the restraints.  The
        step counter, and with it the random stream, runs on through the stages."""
        atoms = np.arange(self.n) if atoms is None else atoms
        for k in schedule:
            self.set_restraints(tether_atoms=atoms, tether_k_kcal=k)
            try:
                self.run_observed(steps_per_stage, record_per_steps, observer)
            finally:
                self.set_restraints()


class _FrameBuffers:
    """Pinned host buffers for ``n_frames`` recorder frames (``vb_md_read_frames``) and numpy views of them."""

    def __init__(self, torch, n_frames: int, n_atoms: int):
        f64, pin = torch.float64, dict(pin_memory=True)
        t = [torch.empty(n_frames, dtype=torch.int64, **pin), torch.empty((n_frames, n_atoms, 3), dtype=f64, **pin),
             torch.empty((n_frames, n_atoms, 3), dtype=f64, **pin), torch.empty(n_frames, dtype=f64, **pin),
             torch.empty(n_frames, dtype=f64, **pin), torch.empty(n_frames, dtype=torch.int32, **pin)]
        self._keep = t
        self.ptrs = [a.data_ptr() for a in t]
        self.step, self.x, self.v, self.epot, self.ekin, self.halted = (a.numpy() for a in t)


RUNAWAY_FACTOR = 1.5        # the reference's guard: T > 1.5 T0 (src/utils/utils.py:154)


class TemperatureRunawayError(RuntimeError):
    """The temperature left 1.5 x the thermostat's target (the reference's guard, ``src/utils/utils.py:153-155``)."""
