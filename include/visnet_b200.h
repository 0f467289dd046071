/* visnet_b200.h -- C ABI of the H100-native ViSNet energy/force engine.
 *
 * Drop-in boundary for the one hot path of microsoft/AI2BMD: the per-MD-step ViSNet evaluation over a
 * packed batch of protein fragments.  Each entry point names the reference interface it replaces
 * (paths relative to the reference tree).  Plain pointers and sizes only -- no torch types.  Every
 * function returns 0 on success or a negative vb_status; the message is available from vb_last_error().
 * There is no CPU fallback: every compute entry fails with VB_ERR_CUDA when no sm_90 device is usable.
 *
 * Units/dtypes are the reference's: positions in Angstrom, energies in eV, forces in eV/Angstrom, fp32.
 */
#ifndef VISNET_B200_H
#define VISNET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vb_handle vb_handle;

typedef enum {
    VB_OK = 0,
    VB_ERR_ARG = -1,      /* bad argument / hyper-parameter mismatch */
    VB_ERR_CUDA = -2,     /* CUDA runtime error (no device, launch failure, ...) */
    VB_ERR_STATE = -3,    /* call order (e.g. forward before set_topology) */
    VB_ERR_ALLOC = -4
} vb_status;

/* Hyper-parameters of the checkpoint (src/ViSNet/model/visnet.py:14-30; both shipped checkpoints:
 * embedding_dimension 128, num_layers 6, num_heads 8, num_rbf 32, lmax 1, cutoff 5.0,
 * max_num_neighbors 32).  The kernels are specialised for exactly these; vb_create() rejects others. */
typedef struct {
    int32_t hidden_channels;
    int32_t num_layers;
    int32_t num_heads;
    int32_t num_rbf;
    int32_t max_num_neighbors;
    float cutoff;
} vb_hparams;

/* Order and element counts ("name:count;...") of the flat fp32 weight blob vb_create() expects.
 * Replaces: ViSNet.load_state_dict in load_model(), src/ViSNet/model/visnet.py:73-93. */
const char* vb_weight_manifest(void);

/* Create an engine on CUDA device `device` from a host weight blob laid out per vb_weight_manifest().
 * Replaces: get_visnet_model(model_path, device) / ViSNetModel.__init__,
 *           src/Calculators/visnet_calculator.py:36-45,184-204. */
int vb_create(const float* weights_host, size_t n_floats, const vb_hparams* hp, int device, vb_handle** out);
void vb_destroy(vb_handle* h);
const char* vb_last_error(const vb_handle* h);   /* h may be NULL: last creation error */

/* Static topology of the packed batch: atomic numbers and graph ids (sorted, contiguous) of N atoms in
 * G fragments -- host pointers, copied.  max_edges <= 0 selects the worst case N*32 (always safe); a smaller value
 * trims the workspace and is a promise by the caller that no step produces more directed edges (incl. self-loops):
 * vb_forward_host verifies it after the fact and fails, the asynchronous entry points cannot.
 * Replaces: the z / batch members of FragmentData (src/AIMD/fragment.py:7-13) that
 *           ViSNetModel.collate() uploads every step (visnet_calculator.py:47-52). */
int vb_set_topology(vb_handle* h, int64_t n_atoms, int64_t n_graphs, const int64_t* z_host,
                    const int64_t* batch_host, int64_t max_edges);

/* One evaluation, device buffers, asynchronous on `stream` (a cudaStream_t passed as void*).
 *   pos_dev[N*3] -> energy_dev[G], forces_dev[N*3].
 * Replaces: ViSNet.forward, src/ViSNet/model/visnet.py:135-166 (energy + autograd force). */
int vb_forward(vb_handle* h, const float* pos_dev, float* energy_dev, float* forces_dev, void* stream);

/* One evaluation with HOST buffers (pinned staging + H2D/D2H inside), synchronous.
 * Replaces: ViSNetModel.dl_potential_loader(FragmentData) -> (e[G,1], f[N,3]),
 *           src/Calculators/visnet_calculator.py:54-63. */
int vb_forward_host(vb_handle* h, const float* pos_host, float* energy_host, float* forces_host);

/* Whole-protein reduction map: F_prot[dst_atom[m]] += sign[m] * F[src_atom[m]], E_prot = sum_g frag_sign[g]*E_g.
 * Replaces: DipeptideBondedCombiner.energy_combine / forces_combine, src/Calculators/combiner.py:11-41
 *           (select_index / origin_index built at src/Fragmentation/distancefrag.py:335-353) and the
 *           dipeptide / ACE-NME split of src/Calculators/bonded.py:91-93. */
int vb_set_protein_map(vb_handle* h, int64_t n_protein_atoms, int64_t n_map, const int32_t* src_atom_host,
                       const int32_t* dst_atom_host, const float* sign_host, const float* frag_sign_host);

/* Evaluation + signed scatter into ef_prot_dev[3*n_protein_atoms + 1] (forces, then the energy in the last
 * slot); the buffer is overwritten.  With several GPUs each rank calls this on its shard of fragments and
 * the caller all-reduces ef_prot_dev (NCCL sum).  Replaces: DLBondedCalculator.__call__, bonded.py:102-123. */
int vb_forward_protein(vb_handle* h, const float* pos_dev, float* ef_prot_dev, void* stream);

/* ---- Energies without forces -------------------------------------------------------------------------------
 * Option "derivative" (vb_set_option, 0 or 1, default 1) selects the workspace vb_set_topology lays out:
 *   1  the full one: vb_forward* evaluate energies and forces; the energy entries below run on it too.
 *   0  a forward-only one of about a fifth of the size (no adjoint buffers, the per-layer node and edge tensors in two
 *      slots by layer parity): only the energy entries below evaluate; vb_forward, vb_forward_host, vb_forward_protein,
 *      vb_md_setup and vb_debug_read of an adjoint buffer fail with VB_ERR_STATE, and the diagnostics (vb_num_stages,
 *      vb_stage_name, vb_stage_kernel, vb_debug_run, vb_profile_stages, vb_launches_per_forward) describe and run the
 *      energy plan.
 * Setting the option drops the topology (and the protein map, MD and hydrogen-refinement state): call vb_set_topology
 * again.  vb_get_option("derivative") answers the setting, vb_get_option("arena_bytes") the workspace size in bytes of
 * the current topology.
 *
 * The energy plan runs the full plan's forward launches with the same kernel choices (node / edge stage variants, tile
 * plan, calibration), so its energies equal vb_forward's bit for bit, then writes the fragment energies; no adjoint.
 * Replaces: ViSNet.forward with derivative=False, src/ViSNet/model/visnet.py:135-166 (returns (E, None)). */

/* pos_dev[N*3] -> energy_dev[G], device buffers, asynchronous on `stream` (one replay of a cached CUDA graph). */
int vb_forward_energy(vb_handle* h, const float* pos_dev, float* energy_dev, void* stream);
/* The same with HOST buffers (pinned staging, one H2D and one D2H inside), synchronous; like vb_forward_host it fails
 * with VB_ERR_STATE when a step produced more edges than a trimmed max_edges holds. */
int vb_forward_energy_host(vb_handle* h, const float* pos_host, float* energy_host);

/* ---- Evaluation in fragment chunks (the reference's --chunk-size) -------------------------------------------------
 * Option "chunk_atoms" (vb_set_option, >= 0, default 0) is read by vb_set_topology, like "derivative", and setting it
 * drops the topology.  With C > 0 the batch is evaluated as a sequence of contiguous fragment chunks of about C atoms
 * (vb_chunk_fragments), one after the other on one workspace sized for the largest chunk, so the workspace no longer
 * grows with the batch: about 700 B per atom of the largest chunk with forces (155 B energy-only), plus about 170 B per
 * batch atom for the arrays that span the batch (topology, neighbour slots, positions, forces, energies).  Every entry
 * evaluates the same way -- vb_forward*, vb_forward_energy*, vb_forward_protein (the whole-protein reduction runs once,
 * after the last chunk) and the MD step -- and all chunks of one evaluation are one CUDA graph replay.  Each chunk gets
 * its own launch plan from its own size (node / edge stage variants, tile plan; "calibrate" plans each chunk from its
 * own edge count), and a trimmed max_edges of vb_set_topology is the edge capacity of every chunk (an overflow names
 * the chunk).  vb_get_option answers "chunk_atoms", "chunks" (the chunk count; 1 without chunks) and, per chunk k,
 * "c<k>/<key>" with key atoms, graphs, first_atom, first_graph, n_edges_capacity, node_tc, npw, te_fwd, edge_tc,
 * tc_rows, tile_rows, gxa_parts, edges_plan, or edges (the chunk's edge count in the last evaluation; synchronises).
 * vb_stage_name / vb_stage_kernel / vb_launches_per_forward list the chunked sequence, stage names prefixed "c<k>/".
 * A chunked handle refuses vb_debug_run, vb_profile_stages, option "timeline" and vb_debug_read of anything but
 * "energy", "forces", "pos" and "RF" with VB_ERR_STATE.  C = 0 is exactly the unchunked engine.
 * Replaces: the chunk loop of DeviceStrategy._set_combined_work_partitions (src/Calculators/device_strategy.py:83-125,
 *           --chunk-size of src/AIMD/arguments.py:189-197) and the per-chunk dl_potential_loader calls of
 *           DLBondedCalculator._inference_impl (src/Calculators/bonded.py:46-49,65-77). */

/* The chunk rule, a pure host function (no handle, no device): fragments [0, n_graphs) with atom offsets
 * frag_start_host[n_graphs + 1] are cut into contiguous chunks; out_bounds[0 .. n] (n_graphs + 1 entries of room)
 * receives the fragment boundaries of the n chunks, and n is returned (VB_ERR_ARG for a negative chunk_atoms or offsets
 * that decrease).  Each chunk ends at the fragment boundary nearest to frag_start[first] + chunk_atoms, a tie keeping
 * the straddling fragment, as the reference does.  Unlike the reference, whose loop never ends once chunk_atoms is
 * below about half a fragment, every chunk takes at least one fragment and at least one atom: fragments without atoms
 * go with the chunk they fall in.  chunk_atoms = 0 is one chunk. */
int vb_chunk_fragments(int64_t n_graphs, const int64_t* frag_start_host, int64_t chunk_atoms, int64_t* out_bounds);

/* ---- Device-resident MD step (SURVEY section 8f, rank 3 and the first half of rank 1) ------------------------
 * State (protein positions / velocities, fp64) stays on the GPU; one step is
 *   kick1 (half-kick + drift) -> eval (place fragment atoms, ViSNet, signed reduction into ef) -> kick2.
 * Replaces: the ASE Langevin loop the reference runs (src/AIMD/simulator.py:96-137: Langevin(dt = 1 fs, 300 K,
 *           friction 0.001/fs), MaxwellBoltzmannDistribution start; ASE 3.22 ase/md/langevin.py step()) and the
 *           per-step fragment coordinate rebuild with cap hydrogens on the acceptor->removed ray
 *           (src/Fragmentation/distancefrag.py:34-54), without the Amber-term LBFGS refinement.
 * Units as ASE: eV, Angstrom, amu; dt in Angstrom*sqrt(amu/eV), friction in 1/that; kT in eV.  friction = 0 is
 * velocity Verlet (no random numbers, no centre-of-mass correction).  Normals come from Philox4x32-10 keyed by
 * (seed; step, component): every rank of a sharded run draws the same numbers.
 *
 * vb_md_setup: recipe per FRAGMENT atom a (arrays of length N): real[a] = protein index, or -1 for an added
 * hydrogen placed at P[acc[a]] + unit(P[rem[a]] - P[acc[a]]) * blen[a].  ef_prot_dev[3*n_protein + 1] is the
 * caller-owned force/energy buffer (must hold forces of the current positions before the first kick1: call
 * vb_md_eval after vb_md_set_state).  Requires vb_set_protein_map with the same n_protein_atoms. */
int vb_md_setup(vb_handle* h, int64_t n_protein_atoms, const double* masses_host, const int32_t* real_host,
                const int32_t* acc_host, const int32_t* rem_host, const float* blen_host, double dt, double kT,
                double friction, uint64_t seed, float* ef_prot_dev);
/* Optional externally supplied normals, device array [pool_steps][2][3*n_protein] (xi, eta), step s reads row
 * s % pool_steps; (NULL, 0) returns to Philox.  For parity tests against a host integrator.  VB_ERR_STATE while the
 * reference noise stream is on (a NULL pool is then accepted and changes nothing). */
int vb_md_set_normals(vb_handle* h, const double* pool_dev, int64_t pool_steps);
/* Noise source of the step.  kind 0: the Philox stream above (the default).  kind 1: the reference's stream -- numpy's
 * np.random.default_rng: PCG64 with the 128-bit state (state_hi, state_lo) and increment (inc_hi, inc_lo, odd) under
 * numpy's ziggurat with its tables wi[256], ki[256], fi[256] (ai2bmd_b200/refnoise.py recovers them) -- generated on the
 * device, 2 * 3 * n_protein normals per step (xi, then eta, C order), advancing the state by exactly the draws numpy
 * consumes; it advances at friction 0 too, and not on a step the frame recorder halted.  Synchronises, drops the
 * captured step graph; the stream survives vb_md_set_state and is freed with the MD state.  VB_ERR_STATE with a
 * normals pool set. */
int vb_md_set_noise(vb_handle* h, int32_t kind, uint64_t state_hi, uint64_t state_lo, uint64_t inc_hi, uint64_t inc_lo,
                    const double* wi, const uint64_t* ki, const double* fi);
/* kind 1 only (else VB_ERR_STATE); synchronise.  state_out[2] = (hi, lo) of the PCG64 state after the last step;
 * normals_host[2 * 3 * n_protein] = the last step's xi, eta. */
int vb_md_get_noise_state(vb_handle* h, uint64_t* state_out);
int vb_md_get_noise(vb_handle* h, double* normals_host);
/* Positions, velocities and the step counter (the normals of step s follow from (seed, s) alone, so a run restarted from
 * a recorded frame draws the random stream the original run drew); synchronises and lifts a halt of the frame recorder. */
int vb_md_set_state(vb_handle* h, const double* x_host, const double* v_host, int64_t step);
/* The three phases, asynchronous on `stream`.  With several GPUs every rank holds the whole-protein state and its
 * own shard of fragments: kick1; eval; all-reduce ef_prot_dev (NCCL sum, by the caller); kick2. */
int vb_md_kick1(vb_handle* h, void* stream);
int vb_md_eval(vb_handle* h, void* stream);
int vb_md_kick2(vb_handle* h, void* stream);
/* Hookean restraints on top of the forces of ef_prot_dev (ASE 3.22 Hookean, the kicks use ef + rf; the energy history
 * records ASE's restrained potential energy ef[3n] + rf[3n]).  Units eV/Angstrom^2 and Angstrom.
 *   tethers: atom tether_atom[t] to the point where it stands NOW (the device positions at this call), spring tether_k,
 *            rt = 0 -- the reference's pre-equilibration stage (src/AIMD/simulator.py:139-166, re-anchored per stage);
 *   springs: atoms spring_ij[s][0..1], spring_k[s], spring_rt[s], pulling only when the pair is farther apart than rt --
 *            the hydrogen bond constraints of --constraints (simulator.py:168-180, pairs from
 *            PDBAnalyzer.find_bonded_atoms, src/utils/utils.py:201-221).
 * Host arrays, copied; replaces the whole previous set; (0, ..., 0, ...) removes all restraints and the step is the
 * unrestrained one again.  Synchronises, then evaluates rf at the current positions so the next kick1 sees the new set
 * (vb_md_eval re-evaluates it, e.g. after vb_md_set_state).  VB_ERR_ARG: atom out of range, an atom tethered twice, a
 * spring with i == j, negative or non-finite k or rt.  Requires vb_md_setup. */
int vb_md_set_restraints(vb_handle* h, int64_t n_tether, const int32_t* tether_atom, double tether_k,
                         int64_t n_spring, const int32_t* spring_ij /* [n][2] */, const double* spring_k,
                         const double* spring_rt);
/* Single GPU: n_steps whole steps, each one replay of a captured CUDA graph, no host synchronisation. */
int vb_md_run(vb_handle* h, int64_t n_steps, void* stream);
/* Synchronises; any of x_host / v_host / step_out may be NULL.  epot_hist_host[n_hist] receives the potential
 * energies recorded at the end of the last n_hist steps (oldest first). */
int vb_md_get_state(vb_handle* h, double* x_host, double* v_host, int64_t* step_out, double* epot_hist_host,
                    int64_t n_hist);
/* Frame recorder: the reference's observed run (MDObserver, src/utils/utils.py:114-166, attached every
 * --record-per-steps steps at src/AIMD/simulator.py:125-137) without a host round trip per frame.  After every step whose
 * counter ends a multiple of `every`, the step itself writes a frame into a device ring of `capacity` slots: the step,
 * the restrained Epot (as the energy history), Ekin = sum m v^2 / 2 (fixed-order sum), a halt mark, and x, v [3n] fp64.
 * With runaway_factor > 0 the frame's temperature T = 2 Ekin / (3 n k_B) is checked against runaway_factor * T0,
 * T0 = kT / k_B of vb_md_setup; above it the frame is marked halted and the device stops integrating: every later step
 * leaves x, v, the counter and the ring as they are, until vb_md_set_state (which lifts the halt) or vb_md_set_recorder.
 * Synchronises; resets the frame count and the halt; drops the cached step graphs.  every = 0 turns the recorder off and
 * frees the ring (the step is then exactly the one without it).  vb_md_kick2 records too, so the sharded phase-by-phase
 * path writes the same frames.  "md_frames" / "md_halt_step" of vb_get_option read the device counters. */
int vb_md_set_recorder(vb_handle* h, int64_t every, int64_t capacity, double runaway_factor);
/* Frames [first, first + n) (frame f = the f-th record step since vb_md_set_recorder) into host arrays step[n],
 * x[n][3n], v[n][3n], epot[n], ekin[n], halted[n] -- any may be NULL -- as asynchronous copies on `stream`; the caller
 * pins the buffers and waits for the stream.  VB_ERR_ARG for frames overwritten or not yet enqueued, as far as the host
 * knows (frames behind a halt are never written: read up to the first halted frame). */
int vb_md_read_frames(vb_handle* h, int64_t first, int64_t n, int64_t* step_host, double* x_host, double* v_host,
                      double* epot_host, double* ekin_host, int32_t* halted_host, void* stream);

/* ---- Non-bonded MM term (SURVEY section 8f, rank 2) ---------------------------------------------------------------
 * All ordered pairs (src j, dst i), j != i, except pairs listed in the exclusion table (atoms sharing a dipeptide,
 * src/Fragmentation/distancefrag.py:355-363; pair list src/AIMD/protein.py:133-151): Lennard-Jones with
 * sigma_ij = (sigma_i + sigma_j)/2 [nm], eps_ij = sqrt(eps_i eps_j) [kJ/mol], plus Coulomb; forces summed on dst,
 * energy halved; results in eV and eV/Angstrom.  Replaces: MMNonBondedCalculator.set_parameters / __call__,
 * src/Calculators/nonbonded.py:24-63.  The exclusion table is CSR over protein atoms, each row strictly ascending.
 * [atom_lo, atom_hi) are the destination atoms this handle computes (a sharded run gives every rank a slice and
 * all-reduces the buffer). */
int vb_set_nonbonded(vb_handle* h, int64_t n_protein_atoms, const float* charges_host, const float* sigmas_nm_host,
                     const float* epsilons_kj_host, const int32_t* excl_rowptr_host, const int32_t* excl_col_host,
                     int64_t atom_lo, int64_t atom_hi);
/* ef_prot_dev[3*n + 1] += non-bonded forces / energy at prot_pos_dev[n*3] (fp32 positions as the reference casts
 * them, nonbonded.py:39).  Accumulates: zero the buffer for the bare term, or call after vb_forward_protein for
 * bonded + non-bonded (FragmentCalculator.calculate, src/Calculators/fragment.py:50-68).  Once set, vb_md_eval
 * adds the term too. */
int vb_nonbonded(vb_handle* h, const float* prot_pos_dev, float* ef_prot_dev, void* stream);

/* ---- Per-step refinement of the added (cap) hydrogens (SURVEY section 8f, rank 1) -----------------------------------
 * One LBFGS call (lr, max_iter, tolerance_grad, tolerance_change; no line search, fresh state) on the Amber energy of all
 * dipeptides, moving only the added hydrogens -- what the reference runs every MD step between placing them and the
 * ViSNet evaluation.  The problem is given as flat term arrays whose atom indices address the PACKED FRAGMENT position
 * buffer [N][3] of vb_set_topology: every term that contains an optimised hydrogen, with its own parameters (Amber
 * units: kcal/mol, Angstrom, radians; qq = product of prmtop charges).  mirror_dst/mirror_src: fragment atoms that are
 * copies of relaxed ones (the ACE-NME fragments take their hydrogens from the neighbouring dipeptides,
 * src/Fragmentation/distancefrag.py:286-307) and are re-copied after the relaxation.
 * Replaces: HydrogenOptimizer.optimize_hydrogen + the five energy terms, src/Fragmentation/hydrogen/energies.py:9-60,
 *           211-242 (tables: hydrogen/ctable.py:58-240), called from DistanceFragment.get_fragments,
 *           src/Fragmentation/distancefrag.py:56-92.  Host helper that builds the arrays from prmtop tables:
 *           ai2bmd_b200/caph.py.  Once set, vb_md_eval / vb_md_run refine after placing the fragment atoms. */
typedef struct {
    int64_t n_h;      const int32_t* h_idx;                                              /* optimised hydrogens        */
    int64_t n_bonds;  const int32_t* bond_ij;   const float* bond_k;  const float* bond_r0;      /* [n][2]             */
    int64_t n_angles; const int32_t* angle_ijk; const float* angle_k; const float* angle_t0;     /* [n][3]             */
    int64_t n_dih;    const int32_t* dih_ijkl;  const float* dih_k;   const float* dih_n; const float* dih_p;  /* [n][4] */
    int64_t n_pairs;  const int32_t* pair_ij;   const float* pair_a;  const float* pair_b; const float* pair_qq;
    int64_t n_mirror; const int32_t* mirror_dst; const int32_t* mirror_src;
    float scnb, scee;                 /* 1-4 scaling of the reference's HydrogenOptimizer: 1.2, 2.0                  */
    int32_t max_iter;                 /* 10 in the reference                                                         */
    float lr, tol_grad, tol_change;   /* 0.1, 0.1, 0.01 in the reference                                             */
} vb_caph_problem;
int vb_set_caph(vb_handle* h, const vb_caph_problem* problem);          /* host pointers, copied */
/* Refine a packed fragment position buffer in place (device pointer), asynchronous on `stream`. */
int vb_caph_relax(vb_handle* h, float* pos_dev, void* stream);

/* ---- One-shot all-reduce over NVLink peer memory (SURVEY section 8e) ---------------------------------------------
 * One process per GPU.  vb_comm_init allocates this rank's window (2 parities x world slots of max_floats) and returns
 * its 64-byte CUDA IPC handle; the caller exchanges the handles of all ranks (any host transport: torch.distributed,
 * MPI, a file) and passes them, in rank order, to vb_comm_connect.  From then on every evaluation that produces the
 * whole-protein buffer (vb_forward_protein, vb_md_eval, vb_md_run) ends with the all-reduce as ONE more kernel of its
 * CUDA graph: peer stores into every rank's window, a system-scope flag per sender, a fixed-order sum (bit-identical on
 * all ranks).  Option "comm_auto" 0 turns the automatic step off; vb_comm_allreduce runs it on any device buffer.
 * Replaces: the host-side gather of the per-device results (ThreadPoolExecutor + numpy concatenation,
 *           src/Calculators/bonded.py:74-89) ahead of combiner.py:38-39, and the NCCL all-reduce a caller would
 *           otherwise enqueue from the host every step.  Needs peer access between the GPUs (NVLink / NVSwitch). */
int vb_comm_init(vb_handle* h, int rank, int world, int64_t max_floats, void* ipc_handle_out /* 64 bytes */);
int vb_comm_connect(vb_handle* h, const void* all_handles /* world x 64 bytes, rank order */);
int vb_comm_allreduce(vb_handle* h, float* buf_dev, int64_t n, void* stream);

/* Copy the current neighbour list to the host: slots[N*32] (source index or -1), deg[N].
 * Replaces: the edge_index returned by torch_cluster.radius_graph at src/ViSNet/model/utils.py:260-266. */
int vb_get_edges(vb_handle* h, int32_t* slots_host, int32_t* deg_host);

/* Number of kernel launches of one vb_forward(), and whether it replays a captured CUDA graph. */
int vb_launches_per_forward(const vb_handle* h);
/* Tuning knobs: "use_graph" 0/1, "use_pdl" 0/1 (programmatic dependent launch between the stages, default off), "npw" 1/2, "te_fwd" 32/64, "te_bwd" 32/64,
 * "edge_tc" bit0 = forward / bit1 = adjoint edge stage on tensor cores (default 3: both), "tc_rows" 32/64/96/128 fixed edges per tensor-core tile
 * (0 = default: tile length planned so the tiles fill whole waves of CTAs, from an estimate of 17 edges per atom or,
 * after "calibrate" 1, from the edge count of the last evaluation -- synchronises), "timeline" 0/1 in-kernel phase stamps of the tensor-core edge kernels and the SIMT node kernels (vb_debug_read "TL" / "TLN"),
 * "node_tc" 0/1 node stage on tensor cores (default: from 600 atoms), "node_nb" 0/1/2/3/4/8 nodes per CTA of the SIMT node kernels (0 = the
 * fewest that fit one wave), "krot" 0/1 every CTA of the SIMT node kernels walks the K dimension of its weight chunks from a
 * different row (default 1: the CTAs of a wave otherwise ask the same L2 slices for the same rows at the same time),
 * "embed_batch" -1/0..3 batch variants of the embedding kernels, "comm_auto" 0/1.  vb_get_option also answers "edge_overflow" (1 after a step exceeded a trimmed max_edges),
 * "tile_rows" (planned edges per tile), "gxa_parts" (1: every tensor-core node CTA runs all column chunks of its row tile; 3: one
 * chunk per CTA, dE/dxa arrives as three partials), "comm_ready", "comm_timeouts" (all-reduce flag waits that gave up after
 * their 10 s deadline; once nonzero, vb_comm_allreduce and every vb_md_* call but vb_md_setup and vb_md_get_state fail
 * with VB_ERR_STATE), "comm_seq" (all-reduces completed since vb_comm_init: the window parity of the next one is its
 * parity plus one),
 * "caph_ready" and "caph_evals" (energy evaluations of the last hydrogen refinement), "md_frames" (frames the recorder
 * has written) and "md_halt_step" (-1, or the step at which its runaway guard fired); both synchronise. */
int vb_set_option(vb_handle* h, const char* key, int64_t value);
int64_t vb_get_option(const vb_handle* h, const char* key);   /* resolved value (after vb_set_topology) */

/* ---- diagnostics (stage-by-stage parity checks; not part of the hot path) ---- */
int vb_num_stages(const vb_handle* h);
const char* vb_stage_name(const vb_handle* h, int stage);
/* The kernel a stage launches under the current options, as "demangled symbol(...) grid=N" (e.g.
 * "vb::edge_fwd_tc_kernel<64>(...) grid=132"), taken from a dry run of the launch sequence that enqueues nothing. */
const char* vb_stage_kernel(const vb_handle* h, int stage);
/* Run only the first n_stages launches of an evaluation, synchronously (no graph). */
int vb_debug_run(vb_handle* h, const float* pos_dev, int n_stages);
/* Per-launch device time (ms, CUDA events on the launching stream, average of n_iter eager evaluations after
 * one warm-up) for each of the vb_num_stages() launches; used by bench.py for the live roofline numbers. */
int vb_profile_stages(vb_handle* h, const float* pos_dev, int n_iter, float* ms_per_stage_host);
/* Self-test of the wgmma/TMA GEMM pipeline: d[128][128] = a[128][128] * W^T, W given as a tensor-core
 * weight image (ai2bmd_b200.weights.tc_image); repeated `reps` times inside one launch; *ms_out = kernel time. */
int vb_tc_selftest(int device, const float* a_host, const float* img_host, float* d_host, int reps, float* ms_out);
/* The same for a tile capacity of `rows` (32, 64 or 128): only the first `rows` rows of a and d are used; 32 and 64 run the
 * three-stage weight ring of the small-tile edge kernels. */
int vb_tc_selftest_rows(int device, int rows, const float* a_host, const float* img_host, float* d_host, int reps, float* ms_out);
/* Copy an internal buffer to the host.  name: "X","V","F","VN","QKV","V123","VDOT","TU","O" (per layer),
 * "XA","VA","GX","GVEC","GF","GXA","GQKV","GVNMSG","GTU","geom","rbf","eacc","grbf","esrc","edst","rowptr",
 * "eatom","energy","forces","pos" (the packed fragment positions [N*3] the MD placement and hydrogen refinement write),
 * and "RF" (fp64 restraint forces then energy [3*n_protein + 1], while restraints are set).
 * Returns the number of bytes copied (<= cap_bytes) or a negative status. */
int64_t vb_debug_read(vb_handle* h, const char* name, int layer, void* host_dst, int64_t cap_bytes);

#ifdef __cplusplus
}
#endif
#endif /* VISNET_B200_H */
