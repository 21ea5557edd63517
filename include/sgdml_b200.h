/*
 * sgdml_b200 -- C ABI of the H100-native engine for sGDML's two dense hot paths
 * (SURVEY.md section 8).  Plain pointers and sizes only; no torch / C++ types.
 *
 * Conventions
 *  - All arrays are C-order (row-major) float64 / int64, exactly as NumPy hands them over.
 *  - Every data pointer may be a HOST pointer or a DEVICE pointer of the current CUDA
 *    device; the library detects which (cudaPointerGetAttributes) and stages host
 *    buffers through device memory itself (H2D / D2H inside the call).
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls
 *    with host outputs synchronise that stream before returning; calls whose outputs
 *    are device pointers are asynchronous on `stream`.
 *  - Return value: 0 = ok; > 0 = LAPACK-style `info` (leading minor of that order is not
 *    positive definite); < 0 = error (-(cudaError_t) for CUDA errors, <= -1000 for
 *    argument errors).  sgdml_b200_last_error() returns a message for the calling thread.
 *  - Notation: N atoms, D = N(N-1)/2 descriptor size, M training points, S permutations.
 *    Pair order d <-> (a,b), a > b, is np.tril_indices(N,-1) (reference desc.py:109-110).
 *
 * Each entry point cites the reference interface it replaces (paths relative to
 * /root/reference/sgdml/).  The reference is pure Python: there is no FFI to bind to,
 * the seam is its `use_torch` engine objects (train.py:1412-1482, predict.py:358-421);
 * INTEGRATION.md shows the ctypes stubs a maintainer would add there.
 */
#ifndef SGDML_B200_H
#define SGDML_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGDML_B200_ABI_VERSION 1

#define SGDML_B200_OK 0
#define SGDML_B200_ERR_ARG (-1000)
#define SGDML_B200_ERR_UNSUPPORTED (-1001)
#define SGDML_B200_ERR_NO_DEVICE (-1002)

int sgdml_b200_abi_version(void);
/* Frees the persistent device workspaces of the current device (the Cholesky panel workspace, the int8 slice
 * planes): they are kept between calls so that a sigma grid of training runs (cli.py:802-806) pays for them once. */
int sgdml_b200_release_workspaces(void);
const char* sgdml_b200_last_error(void);
/* Number of visible CUDA devices (0 => every compute entry point fails loudly). */
int sgdml_b200_device_count(void);

/* ---------------------------------------------------------------- representation */

/* Desc.perm + tril_perms_lin: utils/desc.py:509-539, train.py:897-904.  Host integer
 * routine, bit-exact.  perms (S,N) int64 -> out (S*D,) int64,
 * out[d*S + p] = d(perms[p][a], perms[p][b]) + p*D for d = d(a,b). */
int sgdml_b200_tril_perms_lin(const int64_t* perms, int64_t n_perms, int64_t n_atoms, int64_t* out);

/* Desc.from_R: utils/desc.py:80-239, 288-365 (no lattice).  R (n_geo, 3N) ->
 * R_desc (n_geo, D), R_d_desc (n_geo, D, 3). */
int sgdml_b200_desc_from_R(const double* R, int64_t n_geo, int64_t n_atoms, double* R_desc,
                           double* R_d_desc, void* stream);

/* Desc.from_R with periodic boundary conditions: utils/desc.py:44-77 (_pbc_diff), 100-108, 200-201.  lattice and
 * lattice_inv are 3 x 3 row-major HOST arrays (lattice vectors as COLUMNS, as task['lattice'] / model['lattice'],
 * train.py:524, 826-827; the inverse as np.linalg.inv gives it, train.py:908-911).  Every pair difference is
 * clamped to the super cell, d -= lattice @ round(lattice_inv @ d), before the distance is taken. */
int sgdml_b200_desc_from_R_pbc(const double* R, int64_t n_geo, int64_t n_atoms, const double* lattice,
                               const double* lattice_inv, double* R_desc, double* R_d_desc, void* stream);

/* Desc.d_desc_dot_vec: utils/desc.py:368-385.  R_d_desc (n_geo, D, 3), vecs (n_geo, 3N)
 * -> out (n_geo, D). */
int sgdml_b200_d_desc_dot_vec(const double* R_d_desc, const double* vecs, int64_t n_geo,
                              int64_t n_atoms, double* out, void* stream);

/* Desc.vec_dot_d_desc: utils/desc.py:388-408.  R_d_desc (n_geo, D, 3), vecs (n_geo, D)
 * -> out (n_geo, 3N). */
int sgdml_b200_vec_dot_d_desc(const double* R_d_desc, const double* vecs, int64_t n_geo,
                              int64_t n_atoms, double* out, void* stream);

/* ---------------------------------------------------------------- predictor (path b) */

typedef struct sgdml_b200_model sgdml_b200_model;

/* GDMLPredict.__init__ / GDMLTorchPredict.__init__: predict.py:249-463,
 * torchtools.py:401-593.  The engine keeps device copies of the (unpermuted) model;
 * permutations are applied to the query inside the kernel, never as an M*S cache
 * (predict.py:426-441 builds that cache on the CPU).
 *   R_desc          (M, D)  -- NOTE: the .npz model stores it transposed (D, M), train.py:807
 *   R_d_desc_alpha  (M, D)
 *   tril_perms_lin  (S*D,)
 *   sig as stored in the model; std, c as GDMLPredict uses them (predict.py:1286-1288). */
int sgdml_b200_model_create(sgdml_b200_model** out, int64_t n_atoms, int64_t n_train,
                            int64_t n_perms, const double* R_desc, const double* R_d_desc_alpha,
                            const int64_t* tril_perms_lin, double sig, double std, double c);
int sgdml_b200_model_destroy(sgdml_b200_model* model);

/* GDMLPredict.predict(R): predict.py:1146-1294 (+ _predict_wkr predict.py:84-245).
 * R (B, 3N) -> E (B,) [may be NULL], F (B, 3N); outputs scaled: F*std, E*std + c. */
int sgdml_b200_predict(sgdml_b200_model* model, const double* R, int64_t n_geo, double* E,
                       double* F, void* stream);

/* Extension (the reference has no such output): sgdml_b200_predict plus the virial W of each geometry, in a cell given
 * per call.  Take the rows r_i of a geometry and a cell L whose lattice vectors are its COLUMNS (model['lattice']), and
 * strain both homogeneously, r_i -> (I + eps) r_i, L -> (I + eps) L.  Then
 *   W = -dE/d(eps) at eps = 0   (symmetric 3 x 3, in the model's energy unit)
 *     = sum_d (dE/dx_d) delta_d delta_d^T / |delta_d|^3,
 * x_d = 1/|delta_d| the descriptor and delta_d = r_a - r_b - L rint(L^-1 (r_a - r_b)) the minimum-image vector of pair d
 * (the rint term is locally constant), with the image the descriptor of the same call picked.  For a free molecule W
 * equals the classical virial sum_i r_i F_i^T; in a periodic cell it does not once pairs wrap.  The stress an ASE
 * calculator reports is -W / V.  Energy-constraint terms (sgdml_b200_model_set_alphas_E) are included.
 *   R (B, 3N) -> E (B,) [may be NULL], F (B, 3N), W (B, 9) row-major; each output host or device as in
 *   sgdml_b200_predict, whose E and F (bit for bit) this call returns for the same cell.
 *   lattice, lattice_inv: 9 HOST doubles each, row-major, lattice vectors as columns (the sgdml_b200_model_set_lattice
 *   convention), used for this call only; both NULL: the model's current cell, which may be none.  A singular or
 *   non-finite cell, one NULL of the two, or device pointers are rejected, and a rejected call changes nothing.
 * Small host batches replay a captured CUDA graph into which the cell is read at run time, so a call with a new cell
 * neither captures again nor synchronises the device. */
int sgdml_b200_predict_virial(sgdml_b200_model* model, const double* R, int64_t n_geo, const double* lattice,
                              const double* lattice_inv, double* E, double* F, double* W, void* stream);

/* Extension: sgdml_b200_predict_virial with one cell per geometry (variable-cell trajectories, NPT replicas).
 *   lattices, lattice_invs: (B, 9) HOST doubles each, row-major per geometry, lattice vectors as columns, as for
 *   sgdml_b200_predict_virial; geometry g is evaluated in cell g.  Device pointers are rejected.  R, E [may be NULL], F
 *   and W: host or device as in sgdml_b200_predict.
 * Every cell is checked (finite, not singular) before any work is queued; a rejected call writes nothing and changes
 * nothing.  With every cell equal to L, E, F and W are bit-identical to sgdml_b200_predict_virial in L.  Small host
 * batches replay a captured CUDA graph that reads the cells from its pinned staging at run time, so new cells neither
 * capture again nor synchronise the device. */
int sgdml_b200_predict_virial_cells(sgdml_b200_model* model, const double* R, int64_t n_geo, const double* lattices,
                                    const double* lattice_invs, double* E, double* F, double* W, void* stream);

/* Extension: directional derivative of the forces, HV = (dF/dR) V = -H V, per geometry.
 * R, V (B, 3N) -> HV (B, 3N); host or device as in sgdml_b200_predict; the model's cell; FP64 always.
 * This is the vector-Jacobian product of F (H is symmetric) that lets autograd differentiate through the forces
 * (sgdml_b200/torchtools.py); it costs about one more prediction.  It runs the four contractions as FP64 GEMMs on query
 * rows stacked with their tangent rows, for every descriptor size and whatever sgdml_b200_model_set_contraction_slices
 * chose.  The first call on a model with D <= 256 keeps transposed copies of its training matrices, which
 * sgdml_b200_model_set_alphas refreshes from then on.
 * Workspace: shared with sgdml_b200_predict_hessian and separate from sgdml_b200_predict's, whose results and captured
 * graphs it does not change.  It grows to the largest request seen and never shrinks, so calls of either entry point at
 * sizes already seen neither allocate nor synchronise the device.  One chunk rule serves both: a stacked row (query or
 * tangent) takes DS + 2 Mpad + DP + 2 doubles, a chunk at most ~2 GB of them and at most 65 536 geometries; a geometry
 * needs (1 + n_dir) S rows, n_dir = 1 here, and sgdml_b200_set_predict_chunk(c), c > 0, caps a chunk at 2 c S rows, that
 * is c geometries.  A rejected call writes nothing. */
int sgdml_b200_predict_hvp(sgdml_b200_model* model, const double* R, const double* V, int64_t n_geo,
                           double* HV, void* stream);

/* Extension: the energy Hessian H = d^2E/dR^2 = -dF/dR of every geometry, in the model's units and cell, FP64 always.
 *   R (B, 3N) -> H (B, 3N, 3N) row-major; host or device as in sgdml_b200_predict.
 * Column i of H[b] equals -sgdml_b200_predict_hvp(R[b], e_i) bit for bit (e_i the i-th unit vector): it is that
 * product's pipeline with n_dir = 3N directions, the S query rows of a geometry built once and shared by its 3N tangent
 * rows J e_i.  H is returned as computed, not symmetrised.  Energy-constrained models (alphas_E) and every descriptor
 * size are covered.  Workspace and chunk rule: those of sgdml_b200_predict_hvp, with n_dir = 3N.  A chunk holds whole
 * geometries when (1 + 3N) S stacked rows fit; otherwise one geometry whose 3N columns run in blocks of consecutive
 * directions.  sgdml_b200_set_predict_chunk(c), c > 0, caps a chunk at 2 c S rows: floor(2 c / (3N + 1)) geometries,
 * or, when that is 0, one geometry in blocks of 2 c - 1 directions (c = 1: one column per block).  A rejected call
 * writes nothing. */
int sgdml_b200_predict_hessian(sgdml_b200_model* model, const double* R, int64_t n_geo, double* H, void* stream);

/* ---------------------------------------------------------------- normal modes (csrc/vib.cu)
 * Extension: the mass-weighted Hessian of n_geo geometries with the rigid modes moved to the top of its spectrum.
 *   H (B, n, n), n = 3 n_atoms, in any consistent units; R (B, n); inv_sqrt_mass (n_atoms,) = m^-1/2 per atom
 *   -> Hp (B, n, n), n_rigid (B,) int64.  DEVICE pointers only; Hp must not alias H.
 * Hm = M^-1/2 (H + H^T) / 2 M^-1/2.  The rigid basis B holds, in mass-weighted coordinates, the 3 translations and,
 * unless periodic != 0, the 3 rotations about the centre of mass, orthonormalised by two Gram-Schmidt passes in the
 * order tx, ty, tz, rx, ry, rz; a vector that keeps less than 1e-6 of its norm is dropped (a linear geometry keeps 2
 * rotations, a single atom none).  n_rigid is the number kept.  Then
 *   Hp = P Hm P + c B B^T,  P = I - B B^T,  c = 2 |Hm|_inf + 1,
 * exactly symmetric.  Every eigenvalue of P Hm P is below c, so the n_rigid largest eigenpairs of Hp are the rigid
 * modes (eigenvalue c) and the others are the vibrations, orthogonal to every rigid mode.  Synchronises the stream. */
int sgdml_b200_vib_project(const double* H, const double* R, const double* inv_sqrt_mass, int64_t n_geo,
                           int64_t n_atoms, int periodic, double* Hp, int64_t* n_rigid, void* stream);

/* Extension: eigenvalues (ascending) and orthonormal eigenvectors of n_geo symmetric n x n matrices, n <= the cap
 * SGDML_B200_SYMEIG_MAX_N (sgdml_b200_symeig_max_n).
 *   A (B, n, n) -> w (B, n), V (B, n, n) row-major with the eigenvectors as columns.  DEVICE pointers only; V must not
 *   alias A, which is read only.
 * Parallel cyclic Jacobi, one CTA per matrix, A in shared memory: sweeps of round-robin rotations until a sweep rotates
 * no pair, where a pair is rotated when |a_pq| > eps |A|_F / n (at most 60 sweeps).  Ties in w keep index order.  No
 * atomics and fixed reduction orders: the same bits on every call.  Stream-ordered, no synchronisation. */
#define SGDML_B200_SYMEIG_MAX_N 160
int sgdml_b200_symeig_batched(const double* A, int64_t n, int64_t n_geo, double* w, double* V, void* stream);
int sgdml_b200_symeig_max_n(void);

/* ---------------------------------------------------------------- molecular dynamics on the device
 * Extension: BAOAB Langevin (velocity Verlet at gamma = 0) trajectories of n_rep replicas of one model, many steps per
 * call.  Positions, velocities and forces stay in device memory between steps and between calls; one step is the
 * integrator kernel followed by sgdml_b200_predict's descriptor and predictor kernels on the device-resident positions,
 * captured once into a CUDA graph and replayed n_steps times on `stream` without host synchronisation
 * (SGDML_B200_GRAPH=0: plain launches, bit-identical).
 * Units: the model's throughout.  Positions in its length unit L, forces and E_pot as sgdml_b200_predict returns them
 * (std and c applied), a time unit T of the caller's choice; inv_mass[a] turns the force on atom a into an acceleration
 * in L / T^2, and kT is in the model's energy unit.
 * One step from (r, v, F(r)), with h = dt / 2, c1 = exp(-gamma dt), s_i the inv_mass of the atom of coordinate i and
 * sigma_i = sqrt((1 - c1^2) kT s_i), all computed once per run on the host in double precision:
 *   B  v = v + h (F s)    A  r = r + h v    O  v = c1 v + sigma xi    A  r = r + h v    F, E_pot at r    B  v = v + h (F s)
 * The B and A updates are rounded exactly as written (no fused multiply-add).  gamma == 0 skips O (no draws).
 * xi: Philox4x32-10 with key (seed mod 2^32, seed >> 32) and counter (j, replica, step mod 2^32, step >> 32) for the
 * coordinates 2j and 2j + 1, step being the handle's step index of the step taken; the output words u0..u3 give
 * U_a = ((u0 2^32 + u1) >> 11 + 0.5) 2^-53, U_b likewise from u2, u3, and xi_2j = sqrt(-2 ln U_a) cos(2 pi U_b),
 * xi_2j+1 = sqrt(-2 ln U_a) sin(2 pi U_b).  A trajectory continued over several runs draws the noise of one long run.
 * E_kin = 1/2 sum_i v_i^2 / s_i per replica, summed in a fixed order (runs are reproducible bit for bit).
 * The model must outlive the handle.  The handle keeps its own predictor workspace: sgdml_b200_predict* calls and MD
 * runs never invalidate each other's buffers or graphs.  The F and E_pot that set_state stored are NOT refreshed when
 * the model changes (set_alphas, set_alphas_E, set_lattice, ...): call sgdml_b200_md_set_state again after such a
 * change.  Later runs do evaluate the changed model.  Batches above the predictor's chunk size (fixed when the handle is
 * created) run their chunks inside each step.  Launches count under family 8 (integrator) and 1 (graph replays).
 * Arrays are host or device pointers as elsewhere in this header; calls with host outputs synchronise `stream`.
 * Argument errors are reported before anything is queued, and a rejected call changes nothing.
 * Handle kinds: the call that makes a handle fixes its kind.  sgdml_b200_md_create, and sgdml_b200_pimd_create with
 * n_beads = 1, make plain handles; sgdml_b200_pimd_create with n_beads > 1 makes ring-polymer handles,
 * sgdml_b200_npt_create NPT handles, sgdml_b200_metad_create metadynamics handles and sgdml_b200_umbrella_create
 * umbrella handles.  An entry point called with a handle of a kind it does not take (no x below) returns an argument
 * error:
 *   entry point                                                              plain  ring  NPT  metadynamics  umbrella
 *   sgdml_b200_md_set_state, _md_get_state, _md_destroy                        x     x     x        x            x
 *   sgdml_b200_md_run, _remd_run, _neb_fire, _dimer_fire, _irc_rk4             x
 *   sgdml_b200_pimd_run, _relax_fire, _relax_lbfgs                             x     x
 *   sgdml_b200_npt_run, _npt_set_cells, _npt_get_cells                                     x
 *   sgdml_b200_metad_run, _metad_get_hills, _metad_set_hills, _metad_get_bias                       x
 *   sgdml_b200_umbrella_run, _umbrella_set_windows, _umbrella_get_bias                                           x */
typedef struct sgdml_b200_md sgdml_b200_md;
/* inv_mass (N,) HOST doubles, each finite and > 0; n_rep >= 1. */
int sgdml_b200_md_create(sgdml_b200_md** out, sgdml_b200_model* model, int64_t n_rep, const double* inv_mass);
int sgdml_b200_md_destroy(sgdml_b200_md* md);
/* R, V (n_rep, 3N); V may be NULL (= 0).  Sets every replica's step index to `step` and evaluates F and E_pot at R.
 * V is the full-step velocity that belongs to R. */
int sgdml_b200_md_set_state(sgdml_b200_md* md, const double* R, const double* V, uint64_t step, void* stream);
/* R, V, F (n_rep, 3N), E_pot (n_rep), step (1,): the state after the last run; any output may be NULL. */
int sgdml_b200_md_get_state(sgdml_b200_md* md, double* R, double* V, double* F, double* E_pot, uint64_t* step,
                            void* stream);
/* n_steps >= 0 steps of size dt (finite, > 0) with friction gamma >= 0 (1 / T) at temperature kT >= 0; kT > 0 with
 * gamma == 0 is rejected.  stride = 0: no frames; otherwise n_steps must be a multiple of stride, and frame k is the
 * state after step (k + 1) stride of this run: R_frames, V_frames (n_frames, n_rep, 3N), E_pot_frames, E_kin_frames
 * (n_frames, n_rep), n_frames = n_steps / stride; each may be NULL.  Needs a state (sgdml_b200_md_set_state). */
int sgdml_b200_md_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, uint64_t seed,
                      int64_t stride, double* R_frames, double* V_frames, double* E_pot_frames,
                      double* E_kin_frames, void* stream);

/* ---------------------------------------------------------------- replica-exchange molecular dynamics on the device
 * Extension: temperature replica exchange (parallel tempering; Sugita & Okamoto, Chem. Phys. Lett. 314, 141 (1999)) of
 * Langevin replicas, with the exchanges inside the step graph (no host round trip per exchange).  The handle (plain:
 * see the handle kinds at sgdml_b200_md_create) holds n_rep = n_ladders n_temps replicas: slot
 * l n_temps + k sits at temperature kT[k] of ladder l for the whole run, and exchanges move configurations between
 * neighbouring slots, never temperatures, so frames and the state are sorted by temperature.  Between exchanges every
 * slot runs sgdml_b200_md_run's BAOAB step with its own sigma_i = sqrt((1 - c1^2) kT[k] s_i); units, streams, the
 * Philox noise, frames (stride as there), E_kin, SGDML_B200_GRAPH=0, the workspace and the step counters are those of
 * sgdml_b200_md_run.  The step graph is the exchange kernel (k_remd_exchange, one CTA per ladder), then k_md_step, then
 * the forces of every replica.
 * Schedule: let c be the handle's step index of the state R holds.  With exchange_every = E >= 1 an exchange is
 * attempted on the state at c when c > run_start (the index when this run began) and c % E == 0; with e = c / E the
 * pairs (k, k + 1) with k % 2 == e % 2 and k + 1 < n_temps are attempted, each independently.  The last state of a run
 * is exchanged before the run returns and the first is not, so a run continued over several calls is one long run.
 * E = 0: no exchanges, every slot runs Langevin at its own temperature.
 * Acceptance: D = (beta_k - beta_k+1) (E_k - E_k+1), rounded as written, beta = 1 / kT computed on the host and E_pot
 * as sgdml_b200_predict returns it (std and c applied; c cancels).  The swap is accepted iff D >= 0 or u < exp(D), with
 * u = ((w0 2^32 + w1) >> 11 + 0.5) 2^-53 from the words w0, w1 of Philox4x32-10 under the run's key with counter
 * (0x80000000 | k, l, c mod 2^32, c >> 32): the high bit keeps this stream apart from the O noise, whose first counter
 * word is a coordinate-pair index below 2^31.
 * Velocities: an accepted swap moves the R, V, F and E_pot rows together and swaps the two walker labels.  The
 * full-step velocity w of a configuration moving from kT_a to kT_b is scaled by lam = sqrt(kT_b / kT_a), computed on
 * the host: the handle holds v = w - h (F s) (before the step's pending half-kick), w = v + h (F s) and
 * v' = lam w - h (F s), rounded as written with the configuration's own F.  Frame c shows the state after its exchange.
 * Walker labels: one int32 per slot follows each configuration; it is the slot the configuration held at
 * sgdml_b200_md_set_state, which resets the labels to the identity (the first replica-exchange call on a handle sets
 * them to the identity too).
 * Arguments: n_temps >= 2 dividing n_rep; kT (n_temps) HOST doubles, each finite and > 0; gamma > 0; exchange_every
 * >= 0; n_steps, dt, seed, stride as sgdml_b200_md_run.  Outputs, each host, device or NULL: R_frames, V_frames
 * (n_frames, n_rep, 3N), E_pot_frames, E_kin_frames (n_frames, n_rep) doubles and walker_frames (n_frames, n_rep)
 * int32 as the frames of sgdml_b200_md_run; walkers_out (n_rep) int32, the labels after the run; n_accepted and
 * n_attempted (n_ladders, n_temps - 1) int64, this run's accepted and attempted swaps of each neighbour pair.  Needs a
 * state.  Launches count under family 8 (exchange, integrator) and 1 (graph replays).  Argument errors are reported
 * before anything is queued, and a rejected call changes nothing. */
int sgdml_b200_remd_run(sgdml_b200_md* md, int64_t n_temps, const double* kT, int64_t n_steps, double dt, double gamma,
                        uint64_t seed, int64_t exchange_every, int64_t stride, double* R_frames, double* V_frames,
                        double* E_pot_frames, double* E_kin_frames, int* walker_frames, int* walkers_out,
                        int64_t* n_accepted, int64_t* n_attempted, void* stream);

/* ---------------------------------------------------------------- constant-pressure molecular dynamics on the device
 * Extension: NPT trajectories of periodic models: BAOAB Langevin replicas (sgdml_b200_md_run's step) with the isotropic
 * stochastic cell rescaling barostat of Bernetti & Bussi (J. Chem. Phys. 153, 114107 (2020)), each replica in a cell of
 * its own that the barostat scales.  Units are the model's: P0 in energy / L^3, beta_T (isothermal compressibility) in
 * L^3 / energy, tau_p in T.  An NPT handle is an sgdml_b200_md handle with one cell per replica:
 * sgdml_b200_md_set_state evaluates F, E_pot and the virial W = -dE/d(strain) of each replica in its own cell;
 * sgdml_b200_md_get_state and sgdml_b200_md_destroy are unchanged.  Which other entry points take an NPT handle: the
 * handle kinds at sgdml_b200_md_create.
 * Barostat state per replica: eps, the log of its volume ratio V / V0 since the cell was set, its base cell L0 with
 * the caller's inverse, and V0 = |det L0| (host).  The replica is evaluated in L = a L0 with inverse L0^-1 / a,
 * a = exp(eps / 3).  One step, with the replica's step index at n and its W of the current state:
 *   pending B and frame as sgdml_b200_md_run;  K = 1/2 sum_i v_i^2 / s_i in E_kin's order;  V = V0 exp(eps);
 *   P_int = (2 K + ((W_0 + W_4) + W_8)) / (3 V);
 *   de = -c_a (P0 - P_int) + sqrt(c_b / V) eta,  c_a = (beta_T / tau_p) dt, c_b = 2 kT (beta_T / tau_p) dt (host);
 *   B, A, O, A as sgdml_b200_md_run;  mu = exp(de / 3),  r = r mu,  v = v / mu,  eps = eps + de;
 *   F, E_pot and W at the new positions in the new cell.
 * Every update is rounded as written.  eta = sqrt(-2 ln U_a) cos(2 pi U_b), U_a, U_b from the words of Philox4x32-10
 * under the run's key with counter (0xFFFFFFFF, replica, n mod 2^32, n >> 32), apart from the O noise and the exchange
 * draws; c_b == 0 draws nothing.  With beta_T = 0 every replica keeps its cell and its trajectory is
 * sgdml_b200_md_run's bit for bit in that cell.  Positions are never wrapped into the cell.  Streams, host/device
 * outputs, SGDML_B200_GRAPH=0, the workspace and the launch families (8 and 1) are those of sgdml_b200_md_run;
 * argument errors are reported before anything is queued, and a rejected call changes nothing. */
/* lattices, lattice_invs: (n_rep, 9) HOST doubles, row-major, lattice vectors as columns (the
 * sgdml_b200_predict_virial_cells convention), each cell finite and not singular; inv_mass and n_rep as
 * sgdml_b200_md_create. */
int sgdml_b200_npt_create(sgdml_b200_md** out, sgdml_b200_model* model, int64_t n_rep, const double* inv_mass,
                          const double* lattices, const double* lattice_invs);
/* Replaces every replica's base cell (eps = 0), checked as at creation, and re-evaluates F, E_pot and W when the
 * handle has a state.  Positions do not move. */
int sgdml_b200_npt_set_cells(sgdml_b200_md* md, const double* lattices, const double* lattice_invs, void* stream);
/* lattices, lattice_invs, W: (n_rep, 9) each, the current cells a L0, their inverses and the virial of the state;
 * any output may be NULL. */
int sgdml_b200_npt_get_cells(sgdml_b200_md* md, double* lattices, double* lattice_invs, double* W, void* stream);
/* n_steps, dt, gamma, kT, seed and stride as sgdml_b200_md_run; P0 finite; beta_T finite and >= 0; tau_p finite and
 * > 0.  Frames: R_frames, V_frames, E_pot_frames, E_kin_frames as sgdml_b200_md_run; cell_frames (n_frames, n_rep, 9)
 * the cells a L0; P_frames (n_frames, n_rep) the instantaneous pressure P_int of the frame's state.  Each may be NULL.
 * Needs a state. */
int sgdml_b200_npt_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, double P0,
                       double beta_T, double tau_p, uint64_t seed, int64_t stride, double* R_frames,
                       double* V_frames, double* E_pot_frames, double* E_kin_frames, double* cell_frames,
                       double* P_frames, void* stream);

/* ---------------------------------------------------------------- metadynamics on the device
 * Extension: well-tempered multiple-walker metadynamics (Raiteri et al., J. Phys. Chem. B 110, 3533 (2006); Barducci,
 * Bussi & Parrinello, PRL 100, 020603 (2008)) on 1 to 4 collective variables (CVs).  A metadynamics handle is an
 * sgdml_b200_md handle of n_rep = n_groups n_walkers replicas, replica g n_walkers + w walker w of group g, each
 * integrated by sgdml_b200_md_run's BAOAB step with the force F = F_model + F_bias.  The walkers of a group deposit
 * Gaussian hills into one store and are biased by its sum V(s) = sum_k h_k exp(-sum_j (s_j - c_kj)^2 / (2 w_kj^2));
 * groups never see each other's hills.  CVs (cv_type[j], atoms cv_atoms[4 j ...]): 0 distance |r_j - r_i| (atoms
 * i, j), 1 angle atan2(|a x b|, a.b) with a = r_i - r_j, b = r_k - r_j, in [0, pi] (atoms i, j, k), 2 dihedral
 * atan2(|b2| b1.(b2 x b3), (b1 x b2).(b2 x b3)), b1 = r_j - r_i, b2 = r_k - r_j, b3 = r_l - r_k, in (-pi, pi]
 * (atoms i, j, k, l), on plain coordinate differences (no minimum image; positions are never wrapped).  A dihedral's
 * hill difference is wrapped into [-pi, pi).  The formulas, their roundings and gradients are in csrc/md.cuh.
 * Deposition: inside a run, walker w deposits on every state c > the run's first with c % pace == 0 a hill centred on
 * its CVs, with the run's widths and height w0 exp(-V(s) / dkT) (w0 with dkT = +INFINITY: plain metadynamics).  Every
 * walker of a group is biased by the same hills, those committed before state c: a hill becomes visible to the
 * evaluation of the next state, never to its own.  sgdml_b200_md_set_state evaluates the model and then the bias
 * without a deposit, so a run continued over several calls is one long run.  sgdml_b200_md_get_state's F and E_pot
 * stay the model's.  Which entry points take a metadynamics handle: the handle kinds at sgdml_b200_md_create.
 * Streams, host/device outputs, SGDML_B200_GRAPH=0 and the workspace are those of sgdml_b200_md_run; argument errors
 * are reported before anything is queued, and a rejected call changes nothing. */
/* n_groups, n_walkers >= 1, n_groups n_walkers <= INT32_MAX; 1 <= n_cv <= 4; cv_type (n_cv) and cv_atoms (n_cv, 4)
 * HOST arrays, the atoms of each CV distinct and in [0, N) (unused entries ignored); inv_mass as sgdml_b200_md_create. */
int sgdml_b200_metad_create(sgdml_b200_md** out, sgdml_b200_model* model, int64_t n_groups, int64_t n_walkers,
                            const double* inv_mass, int64_t n_cv, const int* cv_type, const int64_t* cv_atoms);
/* n_steps, dt, gamma, kT, seed and stride as sgdml_b200_md_run; w0 finite and >= 0 (energy); widths (n_cv) HOST, each
 * finite and > 0 (L or radians); pace >= 1; dkT > 0, finite or +INFINITY (energy).  Frames: R, V, E_pot (the model's),
 * E_kin as sgdml_b200_md_run; cv_frames (n_frames, n_rep, n_cv) and bias_frames (n_frames, n_rep) the CVs and bias
 * energy of the frame's state (before its deposit).  Each may be NULL.  Needs a state.  The hill store grows before
 * anything is queued to hold the run's n_walkers #{c in (start, start + n_steps] : c % pace == 0} new hills per group. */
int sgdml_b200_metad_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, double w0,
                         const double* widths, int64_t pace, double dkT, uint64_t seed, int64_t stride,
                         double* R_frames, double* V_frames, double* E_pot_frames, double* E_kin_frames,
                         double* cv_frames, double* bias_frames, void* stream);
/* n_hills (n_groups) HOST int64: the hills of each group; centers, widths (H, n_cv) and heights (H), H = sum n_hills,
 * group after group in deposition order; each may be NULL. */
int sgdml_b200_metad_get_hills(sgdml_b200_md* md, int64_t* n_hills, double* centers, double* widths, double* heights,
                               void* stream);
/* Replaces every group's hills, laid out as sgdml_b200_metad_get_hills gives them (HOST arrays; every centre and height
 * finite, every width finite and > 0), and re-evaluates the bias of the state when the handle has one. */
int sgdml_b200_metad_set_hills(sgdml_b200_md* md, const int64_t* n_hills, const double* centers, const double* widths,
                               const double* heights, void* stream);
/* cv (n_rep, n_cv), V_bias (n_rep) and F_bias (n_rep, 3N): the CVs, bias energy and bias force of the state; any may be
 * NULL.  Needs a state. */
int sgdml_b200_metad_get_bias(sgdml_b200_md* md, double* cv, double* V_bias, double* F_bias, void* stream);

/* ---------------------------------------------------------------- umbrella sampling on the device
 * Extension: umbrella sampling with Hamiltonian replica exchange between neighbouring windows (REUS; Sugita, Kitao &
 * Okamoto, J. Chem. Phys. 113, 6042 (2000)) on 1 to 4 CVs, and its reweighting by MBAR (Shirts & Chodera, J. Chem.
 * Phys. 129, 124105 (2008)).  An umbrella handle is an sgdml_b200_md handle of n_rep = n_ladders n_windows replicas:
 * slot l n_windows + k sits in window k of ladder l for the whole run, each integrated by sgdml_b200_md_run's BAOAB
 * step at one temperature with F = F_model + F_bias.  The CVs are those of sgdml_b200_metad_create.  Window k restrains
 * CV j harmonically: b_k(s) = sum_j (0.5 kappa_kj e_j) e_j with e_j = s_j - c_kj (a dihedral's e_j wrapped into
 * [-pi, pi)), summed in increasing j from 0.0 and rounded as written (csrc/md.cuh).
 * Exchanges: the schedule, pairing, Philox draw and walker labels of sgdml_b200_remd_run.  With configuration a in slot
 * k and b in slot k + 1, d = -(beta ((b_k(s_b) + b_k+1(s_a)) - (b_k(s_a) + b_k+1(s_b)))), beta = 1 / kT; accepted iff
 * d >= 0 or u < exp(d).  An accepted swap moves R, the model's F and E_pot, the CVs and the labels, re-evaluates the
 * bias of both slots in their new windows, and keeps each configuration's full-step velocity w: the handle holds
 * v = w - h (F s), and stores v' = w - h (F_new s) against the new total force.  The last state of a run is exchanged
 * before the run returns and the first is not.  sgdml_b200_md_set_state evaluates the model and the restraints and
 * resets the labels to the identity; sgdml_b200_md_get_state's F and E_pot stay the model's.  Which entry points take
 * an umbrella handle: the handle kinds at sgdml_b200_md_create.  Streams, host/device outputs, SGDML_B200_GRAPH=0 and
 * the workspace are those of sgdml_b200_md_run; argument errors are reported before anything is queued, and a rejected
 * call changes nothing. */
/* n_ladders, n_windows >= 1, n_ladders n_windows <= INT32_MAX; n_cv, cv_type, cv_atoms as sgdml_b200_metad_create;
 * centers, kappas (n_windows, n_cv) HOST doubles: finite, kappa >= 0 (energy / L^2 or energy / rad^2), a dihedral's
 * centre in (-pi, pi]; inv_mass as sgdml_b200_md_create. */
int sgdml_b200_umbrella_create(sgdml_b200_md** out, sgdml_b200_model* model, int64_t n_ladders, int64_t n_windows,
                               const double* inv_mass, int64_t n_cv, const int* cv_type, const int64_t* cv_atoms,
                               const double* centers, const double* kappas);
/* Replaces every window (checked as at creation) and re-evaluates the restraints of the state when there is one. */
int sgdml_b200_umbrella_set_windows(sgdml_b200_md* md, const double* centers, const double* kappas, void* stream);
/* n_steps, dt, gamma, kT, seed and stride as sgdml_b200_md_run; exchange_every >= 0 (0: no exchanges; > 0 needs
 * kT > 0 and n_windows >= 2).  Outputs, each host, device or NULL: R, V, E_pot (the model's), E_kin frames as
 * sgdml_b200_md_run; cv_frames (n_frames, n_rep, n_cv), bias_frames (n_frames, n_rep) and walker_frames (n_frames,
 * n_rep) int32 of the frame's state after its exchange; walkers_out (n_rep) int32; n_accepted, n_attempted
 * (n_ladders, n_windows - 1) int64, this run's swaps of each neighbour pair.  Needs a state. */
int sgdml_b200_umbrella_run(sgdml_b200_md* md, int64_t n_steps, double dt, double gamma, double kT, uint64_t seed,
                            int64_t exchange_every, int64_t stride, double* R_frames, double* V_frames,
                            double* E_pot_frames, double* E_kin_frames, double* cv_frames, double* bias_frames,
                            int* walker_frames, int* walkers_out, int64_t* n_accepted, int64_t* n_attempted,
                            void* stream);
/* cv (n_rep, n_cv), V_bias (n_rep) and F_bias (n_rep, 3N) of the state under its windows; any may be NULL. */
int sgdml_b200_umbrella_get_bias(sgdml_b200_md* md, double* cv, double* V_bias, double* F_bias, void* stream);
/* MBAR over n_samples >= 1 samples (n_samples, n_cv) of CVs (host or device), pooled window after window with
 * n_per_window (n_windows) HOST int64 >= 0 of them, summing to n_samples; the windows (centers, kappas) and CVs as
 * sgdml_b200_umbrella_create, beta = 1 / kT > 0; every sample finite.  Iterates the self-consistent equations from
 * f = 0 until max_k |df_k| < tol (>= 0) or max_iter (>= 1) iterations, f_0 held at 0 (csrc/md.cuh has the reduction
 * order: the result is the same bits on every call).  Outputs, host or device: f (n_windows) the reduced free energies
 * (f_k = beta F_k), log_w (n_samples) the log unbiased weights, normalised so that sum_n exp(log_w_n) = 1; n_iter (1)
 * int64 the iterations run and resid (1) the last max_k |df_k| (HOST or NULL). */
int sgdml_b200_umbrella_mbar(int64_t n_windows, int64_t n_cv, const int* cv_type, const double* centers,
                             const double* kappas, double beta, int64_t n_samples, const double* samples,
                             const int64_t* n_per_window, double tol, int64_t max_iter, double* f, double* log_w,
                             int64_t* n_iter, double* resid, void* stream);

/* ---------------------------------------------------------------- path-integral molecular dynamics on the device
 * Extension: ring polymers of P beads (1 <= P <= 64), thermostatted mode by mode with PILE-L (Ceriotti, Parrinello,
 * Markland & Manolopoulos, J. Chem. Phys. 133, 124104 (2010)) in the BAOAB order of Liu, Li & Liu (J. Chem. Phys. 145,
 * 024103 (2016)).  A handle from sgdml_b200_pimd_create holds n_poly polymers; replica r = p P + j is bead j of polymer
 * p, and every state array has the layout of sgdml_b200_md_*: (n_poly P, 3N).  sgdml_b200_md_destroy, _set_state and
 * _get_state work on it unchanged (the other entry points that take it: the handle kinds at
 * sgdml_b200_md_create), and a handle from sgdml_b200_md_create runs sgdml_b200_pimd_run as P = 1.  Units, streams,
 * the step graph (one k_pimd_step launch, then the forces of every bead as ordinary replicas, chunk by chunk),
 * SGDML_B200_GRAPH=0, the step counters, the workspace and the launch families are those of sgdml_b200_md_run above.
 * Per run, on the host in double precision: h = dt / 2, kT_P = P kT, omega_P = kT_P / hbar,
 * omega_k = 2 omega_P sin(k pi / P); per mode cos(omega_k h), sin(omega_k h) / omega_k and -omega_k sin(omega_k h)
 * (1, h and 0 for k = 0); frictions gamma_0 = gamma, gamma_k = 2 lambda omega_k (k >= 1); c1_k = exp(-gamma_k dt) and
 * sigma_{k,i} = sqrt((1 - c1_k c1_k) kT_P s_i).  Normal modes through the real orthonormal C (P x P): C_j0 = sqrt(1/P);
 * C_jk = sqrt(2/P) cos(2 pi j k / P) for 1 <= k < P/2; C_jk = sqrt(1/P) (-1)^j for k = P/2;
 * C_jk = sqrt(2/P) sin(2 pi j k / P) for P/2 < k < P.
 * One step, bead by bead and mode by mode:
 *   B  v += h (F s)      q_k = sum_j C_jk x_j, u_k = sum_j C_jk v_j (j in order, no fused multiply-add)
 *   A  (q_k, u_k) = (cos q_k + (sin / omega) u_k, (-omega sin) q_k + cos u_k)
 *   O  u_k = c1_k u_k + sigma_{k,i} xi      A again      x_j = sum_k C_jk q_k, v_j likewise
 *   F, E_pot at the new positions            B  v += h (F s)
 * Every update rounds as written.  xi is sgdml_b200_md_run's Philox normal with replica index p P + k (k the mode), so
 * P = 1 gives sgdml_b200_md_run's trajectory bit for bit.  No mode is thermostatted (no draws) when gamma == 0 and
 * (lambda == 0 or P == 1).  lambda = 1 damps every internal mode critically; lambda = 0.5 with gamma = 0 is
 * thermostatted RPMD; gamma = lambda = 0 is NVE RPMD.
 * Frames (stride as in sgdml_b200_md_run): R_frames, V_frames (n_frames, n_poly P, 3N) and E_pot_frames, E_kin_frames
 * (n_frames, n_poly P) per bead as there; per polymer (n_frames, n_poly), with beads cyclic (x_P = x_0), m_i = 1 / s_i
 * and xbar the centroid:
 *   K_prim = 3N P kT / 2 - (1 / P) sum_j sum_i 1/2 m_i omega_P^2 (x_{j,i} - x_{j+1,i})^2
 *   K_cv   = 3N kT / 2 - (1 / 2P) sum_j (x_j - xbar) . F_j
 * the per-coordinate sums over beads in order, then over coordinates in sgdml_b200_md_run's E_kin order.  Positions
 * are never wrapped into a cell, so both estimators hold for periodic models too. */
/* inv_mass (N,) HOST doubles, each finite and > 0; n_poly >= 1, 1 <= n_beads <= 64, n_poly n_beads <= 2^31 - 1. */
int sgdml_b200_pimd_create(sgdml_b200_md** out, sgdml_b200_model* model, int64_t n_poly, int64_t n_beads,
                           const double* inv_mass);
/* n_steps >= 0 steps of size dt (finite, > 0) at temperature kT >= 0 with hbar > 0 in the model's energy unit times T,
 * centroid friction gamma >= 0 (1 / T) and PILE-L scale lambda >= 0.  P > 1 needs kT > 0; P = 1 follows
 * sgdml_b200_md_run's rules (kT > 0 needs gamma > 0).  Each frame output may be NULL.  Needs a state. */
int sgdml_b200_pimd_run(sgdml_b200_md* md, int64_t n_steps, double dt, double kT, double hbar, double gamma,
                        double lambda, uint64_t seed, int64_t stride, double* R_frames, double* V_frames,
                        double* E_pot_frames, double* E_kin_frames, double* K_prim_frames, double* K_cv_frames,
                        void* stream);

/* ---------------------------------------------------------------- geometry optimisation on the device
 * Extension: relax every replica of an sgdml_b200_md handle to a local minimum of the model's energy with FIRE or
 * L-BFGS, many steps per call and no host round trip per step.  The handle needs a state (sgdml_b200_md_set_state);
 * its inverse masses are not read.  Beads of a ring-polymer handle are relaxed as independent replicas.  One step is
 * the optimiser kernel (k_fire_step or k_lbfgs_step, one CTA per replica) followed by the forces of every replica,
 * chunk by chunk, as in sgdml_b200_md_run: the handle's step graph with the optimiser as its integrator, captured again
 * when the optimiser changes (SGDML_B200_GRAPH=0: plain launches, bit-identical).
 * Convergence (ASE's criterion): max over atoms of Fx^2 + Fy^2 + Fz^2 < fmax^2, tested on the forces at the current
 * positions before every step.  A replica that has converged is frozen: its positions never change again in this
 * call.  fmax = 0 runs max_steps steps.  Replays run in blocks; after each block a kernel counts the unconverged
 * replicas into mapped pinned memory and the call returns once none is left or max_steps steps have run.  The block
 * length changes only the cost, never a result.
 * Every call starts its optimiser afresh (as a new ASE optimiser would).  After it, R holds the final positions with F
 * and E_pot evaluated there, V is zero (a following sgdml_b200_md_run starts at rest), and the step counter is
 * unchanged (the Philox stream is untouched).  The stored F and E_pot are those of the last force evaluation, as for
 * sgdml_b200_md_run: call sgdml_b200_md_set_state again after the model changes.
 * Outputs, each host, device or NULL: n_steps_out (n_rep) int64, the position updates each replica took;
 * converged_out (n_rep) int32, 1 if max_a |F_a| < fmax at the final positions; fmax_out (n_rep) double,
 * max_a |F_a| there.  Calls with host outputs synchronise `stream`; every call waits for its convergence read-backs.
 * Units are the model's: positions in L, forces as sgdml_b200_predict returns them.  The exact update of each
 * optimiser, every sum's order and every rounding are stated in csrc/md.cuh; sums run in a fixed order, so results
 * are reproducible bit for bit.  The optimiser state (for L-BFGS 2 m + 2 vectors of 3N doubles per replica) is made
 * on the handle at the first relaxation, grown when a call asks for more memory, and freed with the handle.  Launches
 * count under family 8 (optimiser, test, count) and 1 (graph replays).  Argument errors are reported before anything
 * is queued, and a rejected call changes nothing. */
/* FIRE (Bitzek et al., PRL 97, 170201 (2006)) in ASE's mass-free form with its constants (Nmin 5, finc 1.1, fdec 0.5,
 * alpha_start 0.1, f_alpha 0.99): max_steps >= 0; fmax >= 0 (force unit); maxstep > 0 (L), the cap on |dr| of a
 * replica's whole step; dt > 0 the initial and dtmax > 0 the largest time step, in sqrt(L^2 / force unit). */
int sgdml_b200_relax_fire(sgdml_b200_md* md, int64_t max_steps, double fmax, double maxstep, double dt, double dtmax,
                          int64_t* n_steps_out, int* converged_out, double* fmax_out, void* stream);
/* L-BFGS (two-loop recursion, Nocedal & Wright Alg. 7.4) without line search: memory m in [1, 32] pairs; h0 > 0
 * (L^2 / energy) the inverse Hessian guess while the history is empty, afterwards s.y / y.y of the newest pair; a pair
 * with s.y <= 0, an energy rise or a non-descent direction clears the history.  maxstep > 0 (L) caps the step of
 * every atom (ASE's rule: the whole step is scaled so that its longest atom step is maxstep). */
int sgdml_b200_relax_lbfgs(sgdml_b200_md* md, int64_t max_steps, double fmax, double maxstep, int memory, double h0,
                           int64_t* n_steps_out, int* converged_out, double* fmax_out, void* stream);
/* ---------------------------------------------------------------- nudged elastic band on the device
 * Extension: minimum-energy paths and saddle points with the nudged elastic band (NEB) and its climbing-image form
 * (CI-NEB), optimised by FIRE on each whole band, many bands and many steps per call.  The handle (plain: see handle
 * kinds at sgdml_b200_md_create) holds n_rep = n_bands n_images replicas: replica b n_images + j is image j of band
 * b.  Images 0 and n_images - 1 are fixed endpoints: they never move, but their forces and energies are evaluated with
 * the rest of the batch every step.  Image differences are plain coordinate differences, with no minimum image, also
 * for periodic models.  Tangents are Henkelman & Jonsson's improved tangent (J. Chem. Phys. 113, 9978 (2000)), the
 * spring force k (|R[i+1] - R[i]| - |R[i] - R[i-1]|) acts along it; with climb != 0 the interior image of highest
 * energy (the lowest index on ties, chosen again at every step) feels the model force with its tangent component
 * reversed and no spring (Henkelman, Uberuaga & Jonsson, J. Chem. Phys. 113, 9901 (2000)).  The interior images of a
 * band are one FIRE vector of (n_images - 2) 3N coordinates, as for ASE's optimisers on an NEB object: the FIRE rules,
 * constants and arguments are sgdml_b200_relax_fire's, maxstep caps |dr| of the whole band, and a band has converged
 * when max over the atoms of all its interior images of |F_neb,a| < fmax; it is frozen from then on.  L-BFGS is not
 * offered: its energy-rise reset has no meaning for NEB forces, which are not a gradient.  The step graph is the NEB
 * force kernel and the band FIRE kernel (k_neb_force, k_neb_fire_step) followed by the forces of every image; the
 * driver, the block read-backs, the final state (R, F, E_pot at the final positions, V zero, step counter unchanged)
 * and the launch families are those of sgdml_b200_relax_* above.  Exact sums and roundings are in csrc/md.cuh.
 * Arguments: n_images >= 3 dividing n_rep; k >= 0 (force unit / L); fmax, maxstep, dt, dtmax as for
 * sgdml_b200_relax_fire.  Outputs, each host, device or NULL, per band (n_rep / n_images): n_steps_out int64,
 * converged_out int32, fmax_out double (max_a |F_neb,a| at the final positions) and climbing_out int32, the index of
 * the band's highest interior image at the final positions.  Argument errors are reported before anything is queued,
 * and a rejected call changes nothing. */
int sgdml_b200_neb_fire(sgdml_b200_md* md, int64_t n_images, int64_t max_steps, double fmax, double k, int climb,
                        double maxstep, double dt, double dtmax, int64_t* n_steps_out, int* converged_out,
                        double* fmax_out, int* climbing_out, void* stream);
/* ---------------------------------------------------------------- dimer saddle search on the device
 * Extension: first-order saddle points next to a minimum, with no final state, by the dimer method (Henkelman &
 * Jonsson, J. Chem. Phys. 111, 7010 (1999)), many dimers and many steps per call.  The handle (plain: see the
 * handle kinds at sgdml_b200_md_create) holds n_rep = 2 n_dimers replicas: replica 2d is the
 * centre R0 of dimer d and replica 2d + 1 its image R0 + separation N, N the dimer's unit mode; both are evaluated
 * every step, the other image is the central difference 2 F0 - F1.  Each step first tests the dimer: it has converged
 * when max_a |F0_a| < fmax and the curvature along N, measured at the current centre, is negative; it is frozen from
 * then on.  Otherwise, when the rotational force exceeds rot_min, it rotates once (a trial image at angle phi_t with
 * cos_trial, sin_trial, then the analytic minimum of the fitted curvature, Heyden, Bell & Keil, J. Chem. Phys. 123,
 * 224101 (2005)), which costs one extra force evaluation; then it translates the centre by one FIRE step (the rules,
 * constants and arguments of sgdml_b200_relax_fire, maxstep capping the centre's whole step) with the force whose
 * component along N is reversed (negative curvature) or alone and reversed (positive curvature).  N is kept orthogonal
 * to rigid translations and, for free molecules, infinitesimal rotations of the centre.  L-BFGS is not offered: the
 * dimer force is no gradient.  Exact sums and roundings are in csrc/md.cuh; the driver, block read-backs, final state
 * (V zero, step counter unchanged) and launch families are those of sgdml_b200_relax_*.
 * Arguments: modes (n_rep / 2, 3N), host or device, the initial modes (any length; projected and normalised at each
 * centre), or NULL to keep the handle's modes from its previous dimer call (an argument error on the first); a mode
 * that is not finite or is (almost) a rigid motion is an argument error.  max_steps bounds the force evaluations of
 * the pairs (a rotating step takes two); separation > 0 (L); cos_trial, sin_trial > 0 with c^2 + s^2 = 1 within 1e-12;
 * rot_min >= 0 (force / L^2, as the curvature); fmax, maxstep, dt, dtmax as for sgdml_b200_relax_fire.  Outputs,
 * each host, device or NULL, per dimer: n_steps_out int64 (translations), converged_out int32, fmax_out double
 * (max_a |F0_a|), curvature_out double (along the final mode at the final centre), n_rot_out int64 (rotations) and
 * modes_out (n_rep / 2, 3N) double.  Argument errors are reported before anything of the handle changes (the modes are
 * checked on scratch), and a rejected call changes nothing. */
int sgdml_b200_dimer_fire(sgdml_b200_md* md, const double* modes, int64_t max_steps, double fmax, double separation,
                          double cos_trial, double sin_trial, double rot_min, double maxstep, double dt, double dtmax,
                          int64_t* n_steps_out, int* converged_out, double* fmax_out, double* curvature_out,
                          int64_t* n_rot_out, double* modes_out, void* stream);
/* ---------------------------------------------------------------- intrinsic reaction coordinate on the device
 * Extension: which two minima a first-order saddle connects, by the intrinsic reaction coordinate (IRC): the
 * steepest-descent path in mass-weighted coordinates x_i = R_i / sqrt(s_i), s the handle's inverse masses, followed
 * downhill from each saddle in both directions along its imaginary mode by classical RK4 (Schmidt, Gordon & Dupuis,
 * JACS 107, 2585 (1985)) of dx/ds = r F / |r F|, r_i = sqrt(s_i), with a fixed step; many saddles and many points per
 * call.  The handle (plain: see the handle kinds at sgdml_b200_md_create) holds n_rep = 2 n_saddles replicas (n_rep
 * even): replica 2k's state is saddle k at the start of the call (as set_state stored it: R, F, E_pot), and replica
 * 2k + 1's is overwritten with it; replica 2k follows +mode (forward), 2k + 1 -mode (backward).  Point 0 of a branch
 * is the saddle, point 1 the saddle plus step along the mass-weighted unit mode, every later point one RK4 step (four
 * force evaluations) from the one before.  A new point whose energy is not below the previous one's is rejected and
 * the branch ends at the previous point (end 2); otherwise it is recorded, and the branch ends there when
 * max_a |F_a| < fmax (end 1, ASE's criterion) or when it holds max_points points (end 3).  An ended branch is frozen
 * for the rest of the call (its forces are still evaluated with the batch).  No rigid-mode projection: the model's
 * energy is invariant under rigid motions.  Exact sums and roundings are in csrc/md.cuh; the driver, block read-backs
 * and launch families are those of sgdml_b200_relax_*.
 * Arguments: modes (n_rep / 2, 3N), host or device, the Cartesian displacement of each saddle's imaginary mode (any
 * length; GDMLVibrations' modes or a dimer's mode); a mode that is not finite or whose mass-weighted norm is 0 is an
 * argument error, checked before anything of the handle changes.  max_points >= 2; step > 0 in the handle's
 * mass-weighted unit (L / sqrt(inverse-mass unit)); fmax >= 0 (force unit; 0: never ends by force).  Outputs, each
 * host, device or NULL: R_path (n_rep, max_points, 3N) and E_path (n_rep, max_points), every entry written, NaN past
 * the branch's n_points; n_points_out (n_rep) int64, the points recorded, the saddle included; end_out (n_rep) int32,
 * 1, 2 or 3 as above; fmax_out (n_rep) double, max_a |F_a| at the branch end.  After the call R, F and E_pot of each
 * replica are its branch end and the forces there, V is zero and the step counter is unchanged.  Argument errors are
 * reported before anything is queued, and a rejected call changes nothing. */
int sgdml_b200_irc_rk4(sgdml_b200_md* md, const double* modes, int64_t max_points, double step, double fmax,
                       double* R_path, double* E_path, int64_t* n_points_out, int* end_out, double* fmax_out,
                       void* stream);
/* Test hook: graph replays between convergence read-backs of sgdml_b200_relax_*, sgdml_b200_neb_fire,
 * sgdml_b200_dimer_fire and sgdml_b200_irc_rk4; 0 = the default (16).  Negative values are rejected. */
int sgdml_b200_set_relax_block(int64_t n_steps);

/* Periodic model (predict.py:332-334: lat_and_inv from model['lattice']): query descriptors of
 * sgdml_b200_predict are built with the minimum-image convention.  Both NULL: back to a free molecule. */
int sgdml_b200_model_set_lattice(sgdml_b200_model* model, const double* lattice, const double* lattice_inv);

/* Energy constraints in the kernel (use_E_cstr models; predict.py:219-229, 443-447, 594-601): alphas_E (M,) or
 * NULL to switch the terms off.  With alphas_E set, every (virtual query row, training point) pair additionally
 * contributes alphas_E[m] * c2 * delta to the descriptor-space force and alphas_E[m] * K_ee to the energy,
 * K_ee = (1 + (n/sig)(1 + n/(3 sig))) exp(-n/sig). */
int sgdml_b200_model_set_alphas_E(sgdml_b200_model* model, const double* alphas_E, void* stream);

/* GDMLPredict.set_R_desc / set_R_d_desc: predict.py:511-549.  Caches the training
 * descriptor Jacobians (M, D, 3) on the device so that set_alphas and the training-point
 * evaluation need no host data. */
int sgdml_b200_model_set_R_d_desc(sgdml_b200_model* model, const double* R_d_desc);

/* GDMLPredict.set_alphas: predict.py:551-601 / torchtools.py:760-875.
 * alphas_F (3NM,) -> R_d_desc_alpha = J_m alpha_m on the device. */
int sgdml_b200_model_set_alphas(sgdml_b200_model* model, const double* alphas_F, void* stream);

/* GDMLPredict.predict() with R=None (training points from the cached descriptors):
 * predict.py:1219-1235; the K.v operator of the iterative solver (iterative.py:183-204)
 * and _recov_int_const (train.py:1136-1147).  Evaluates training points
 * [m_begin, m_end).  scaled != 0: outputs scaled as sgdml_b200_predict; scaled == 0:
 * raw sums (std = 1, c = 0), i.e. F = (K v)[m_begin*3N : m_end*3N] for alphas = v. */
int sgdml_b200_predict_train(sgdml_b200_model* model, int64_t m_begin, int64_t m_end, int scaled,
                             double* E, double* F, void* stream);

/* Extension: sgdml_b200_predict_train plus the virial W (B, 9) of each training point (see sgdml_b200_predict_virial),
 * with the same `scaled` semantics; E and F are bit-identical to sgdml_b200_predict_train.  W comes from the cached
 * training Jacobians (sgdml_b200_model_set_R_d_desc), so it is in the cell those were built in. */
int sgdml_b200_predict_train_virial(sgdml_b200_model* model, int64_t m_begin, int64_t m_end, int scaled,
                                    double* E, double* F, double* W, void* stream);

/* Large-descriptor models (D > 256: the predictor is four GEMMs around two element-wise kernels): run those GEMMs on
 * the int8 tensor cores (wgmma) through `slices` exact int8 slices per operand (2..7; csrc/ozaki.cu) or in FP64 DMMA (0, the
 * default unless SGDML_B200_OZAKI_PREDICT_SLICES is set when the model is created).  Forces against the FP64 oracle,
 * measured on an H100 (N = 24, M = 29; tests/test_ozaki_predict_classes.py): 1.2e-8 / 1.3e-10 / 1.1e-12 / 9.3e-15
 * relative for 4 / 5 / 6 / 7 slices; tests/ozaki_predict_model.py bounds them componentwise.  The iterative solver sets 5 for its K.v products
 * (iterative.py:183-204: tolerance 1e-4).  No effect for D <= 256. */
int sgdml_b200_model_set_contraction_slices(sgdml_b200_model* model, int slices, void* stream);

/* Test hook: at most max_geos queries (or training points) per chunk of sgdml_b200_predict and
 * sgdml_b200_predict_train, for every model, and 2 max_geos S stacked rows per chunk of sgdml_b200_predict_hvp and
 * sgdml_b200_predict_hessian (their one chunk rule, see sgdml_b200_predict_hvp: max_geos geometries for the HVP);
 * 0 = no cap (the default: chunks bounded by workspace size only).  Negative values are rejected.  The cap also bounds
 * the minimum per-batch workspace, which limits how far small batches split the sweep over the training points.
 * Workspaces never shrink: it applies fully to models created after the call.  Tests lower it to cover the
 * multi-chunk, pipelined and tail-chunk paths at small batch sizes. */
int sgdml_b200_set_predict_chunk(int64_t max_geos);

/* Test hook (large-descriptor models): the stages of one chunk of the GEMM-composed predictor, copied out of the
 * production sequence before the next stage overwrites them in place.  Every pointer is a device pointer or NULL (that
 * stage is not copied).  rows = n_geo * n_perms virtual query rows, row b * n_perms + p being query b under
 * permutation p; DS = DP + 4, DP = D rounded up to 8, Mpad = M rounded up to 8 (written back by the call). */
typedef struct sgdml_b200_predict_taps {
  double* Qg;    /* rows x DS: x[pinv_p] - mu, zero beyond D */
  double* qq;    /* rows: |Qg row|^2 */
  double* S1;    /* rows x Mpad: Qg Xc^T as the first GEMM pair left it */
  double* S2;    /* rows x Mpad: Qg JA^T */
  double* C1;    /* rows x Mpad: the Matern factors after the transform (zero for m >= M) */
  double* C2;    /* rows x Mpad */
  double* csum;  /* rows: sum_m C1 */
  double* Erow;  /* rows: the energy terms of each row */
  double* acc;   /* rows x DP: C1 XcT^T + C2 JAT^T, before the combine */
  double* G;     /* rows x DP: csum Qg - acc */
  double* Xc;    /* Mpad x DS: the centred training descriptors */
  double* JA;    /* Mpad x DS: R_d_desc_alpha */
  double* XcT;   /* DP x Mpad */
  double* JAT;   /* DP x Mpad */
  double* mm;    /* Mpad: |Xc row|^2 */
  double* xja;   /* Mpad: Xc row . JA row */
  double* mu;    /* DS: the training mean */
  double* ae;    /* Mpad: alphas_E, or zeros when the model has none */
  int oz_s;      /* written: the slice count the four GEMMs ran with, 0 for FP64 */
  int use_ae;    /* written: 1 when the energy-constraint terms were on */
  int64_t DS, DP, Mpad;  /* written */
} sgdml_b200_predict_taps;
/* R != NULL: n_geo device geometries in the model's cell; R == NULL: the training points m_begin .. m_begin + n_geo - 1,
 * raw or scaled as sgdml_b200_predict_train.  E (may be NULL) and F are device outputs and bit-identical to those of the
 * untapped call.  n_geo must fit one chunk; models with D <= 256 are rejected (they run the fused kernel).  The call
 * synchronises the stream. */
int sgdml_b200_predict_stages(sgdml_b200_model* model, const double* R, int64_t n_geo, int64_t m_begin, int scaled,
                              sgdml_b200_predict_taps* taps, double* E, double* F, void* stream);

/* Shape of a model: n_atoms, n_train, n_perms (any pointer may be NULL). */
int sgdml_b200_model_dims(const sgdml_b200_model* model, int64_t* n_atoms, int64_t* n_train, int64_t* n_perms);

/* Reads back R_d_desc_alpha (M, D) -- the `R_d_desc_alpha` key of the model file
 * (train.py:791, 808). */
int sgdml_b200_model_get_R_d_desc_alpha(sgdml_b200_model* model, double* out);

/* ---------------------------------------------------------------- assembly (path a) */

/* GDMLTrain._assemble_kernel_mat / GDMLTorchAssemble.forward: train.py:1260-1535,
 * train.py:97-232, torchtools.py:110-392 (force-force blocks).
 *   K[i*3N + r, c] = scale * K_ref[i*3N + r, col_idxs[c]],  K is (3NM, n_cols), row
 *   stride ldk (>= n_cols).  col_idxs == NULL: all 3NM columns (n_cols must be 3NM);
 *   otherwise a sorted, duplicate-free int64 list (train.py:1341-1345).
 *   scale = -1 gives the matrix the analytic solver factorises (analytic.py:65). */
int sgdml_b200_assemble(const double* R_desc, const double* R_d_desc, const int64_t* tril_perms_lin,
                        int64_t n_atoms, int64_t n_train, int64_t n_perms, double sig,
                        const int64_t* col_idxs, int64_t n_cols, double scale, double* K,
                        int64_t ldk, void* stream);

/* Row-sharded form of sgdml_b200_assemble (SURVEY.md section 8e "explicit K assembly": blocks are
 * independent, each GPU assembles the block rows of its own training points).  Only the row
 * points [m_begin, m_end) are produced: K is ((m_end - m_begin)*3N, n_cols) and
 *   K[(i - m_begin)*3N + r, c] = scale * K_ref[i*3N + r, col_idxs[c]].
 * This is the loop `for i in range(n_train)` of train.py:193-194 cut into ranges. */
int sgdml_b200_assemble_rows(const double* R_desc, const double* R_d_desc,
                             const int64_t* tril_perms_lin, int64_t n_atoms, int64_t n_train,
                             int64_t n_perms, double sig, const int64_t* col_idxs, int64_t n_cols,
                             double scale, int64_t m_begin, int64_t m_end, double* K, int64_t ldk,
                             void* stream);

/* Energy constraints in the kernel (task['use_E_cstr'], train.py:234-300, 1325-1335): fills the M energy rows and
 * columns and the M x M energy-energy block of the (3NM + M)-square matrix K (DEVICE pointer, row stride ldk >= 3NM + M)
 * whose force-force part sgdml_b200_assemble has written with the same `scale`:
 *   K[3NM + i, blk_j] = K[blk_j, 3NM + i] = scale * K_fe(i, j),   K[3NM + j, 3NM + i] = scale * K_ee(i, j). */
int sgdml_b200_assemble_ecstr(const double* R_desc, const double* R_d_desc, const int64_t* tril_perms_lin,
                              int64_t n_atoms, int64_t n_train, int64_t n_perms, double sig, double scale, double* K,
                              int64_t ldk, void* stream);

/* Row block of the energy-constrained matrix at a column subset (the Nystroem set-up of iterative.py:232-247 with
 * use_E_cstr; train.py:1376-1407): with K_full the (3NM + M)-square matrix of sgdml_b200_assemble(+_ecstr) in the
 * layout [forces (3NM); energies (M)], and col_idxs a sorted, duplicate-free int64 list in [0, 3NM + M),
 *   K[(i - m_begin)*3N + r, c]              = scale * K_full[i*3N + r, col_idxs[c]]   (force rows)
 *   K[(m_end - m_begin)*3N + (i - m_begin), c] = scale * K_full[3NM + i, col_idxs[c]] (energy rows)
 * for i in [m_begin, m_end): (m_end - m_begin)(3N + 1) rows of row stride ldk >= n_cols.  K must be a DEVICE
 * pointer.  The force columns (the prefix of the list) of the force rows are exactly what sgdml_b200_assemble_rows
 * writes; every other entry costs one pass over the (row point, column point) pair.  Padding columns (ldk > n_cols)
 * are neither read nor written.  Same limits as sgdml_b200_assemble_ecstr (N <= 1023, M <= 65535). */
int sgdml_b200_assemble_ecstr_rows(const double* R_desc, const double* R_d_desc, const int64_t* tril_perms_lin,
                                   int64_t n_atoms, int64_t n_train, int64_t n_perms, double sig,
                                   const int64_t* col_idxs, int64_t n_cols, double scale, int64_t m_begin,
                                   int64_t m_end, double* K, int64_t ldk, void* stream);

/* Tuning / test hook: 0 = kernel chosen by molecule size (default), 1 = always the large-molecule
 * kernel (tables in global memory), which molecules above ~50 atoms need; 2 / 4 / 5 = small-molecule kernel with
 * per-permutation phases (k_assemble) / chunks of up to 16 permutations with byte permutation tables and per-kind
 * phases over the kept column atoms (v4: k_assemble_tile on expanded pair tables) / the same on the compressed pair
 * arrays (v5: k_assemble_tile on them), where
 * the shared-memory budget allows it; any other value is rejected; 1000 + r = at most r row
 * points per launch of the small-molecule kernel (default 65535, the grid limit; tests lower it to
 * cover the multi-launch path that row ranges above 65535 training points take). */
int sgdml_b200_set_assemble_variant(int variant);

/* How sgdml_b200_assemble_rows would run a force-force call under the current sgdml_b200_set_assemble_variant hooks,
 * on a device with n_sm SMs: n_atoms atoms, n_perms permutations, n_colpts column points with at most nk kept column
 * atoms each (nk = n_atoms without a column list), n_rowpts row points; square = 1 for the full matrix (no column list,
 * every row point: nk = n_atoms, n_colpts = n_rowpts).  Writes 10 values to out:
 *   {kernel (0 k_assemble, 1 v4 = k_assemble_tile<ExpandedPairs>, 2 v5 = k_assemble_tile<CompressedPairs>,
 *    3 k_assemble_large), TJ, PG, n_chunks (grid.z), grid_x, dynamic shared memory bytes, sym, rows_per_launch, slab (doubles per CTA, large only), dl_in_smem}.
 * Host only: needs no device. */
int sgdml_b200_assemble_plan(int64_t n_atoms, int64_t n_perms, int64_t nk, int64_t n_colpts, int64_t n_rowpts,
                             int square, int n_sm, int64_t* out);

/* ---------------------------------------------------------------- permutation discovery
 * utils/perm.py:53-87 (_bipartite_match_wkr): the pairwise matching of training geometries that perm.find_perms starts
 * from, for all pairs or a list of pairs in one launch.  For the pair (i, j), i < j:
 *   cost = -absv_i absv_j^T;  cost[a][b] += max|cost| where z[a] != z[b]                      (perm.py:70-71, 97-98)
 *   perm = the minimum-cost assignment of rows to columns (shortest augmenting paths, FP64; rows inserted in index
 *          order, ties to the lowest column index), perm[a] = column of row a                 (perm.py:73)
 *   score_before = |adj_i - adj_j|_F,  score = |adj_i[perm][:, perm] - adj_j|_F              (perm.py:75-79)
 *   match_cost = min(score, score_before);  has_perm = score < score_before and not numpy.isclose(score_before, score)
 *                (|a - b| <= 1e-8 + 1e-5 |b|): the pairs whose permutation perm.py:84-85 keeps.
 *   adj   (M, N, N) symmetric pair-distance matrices            absv  (M, N, N) |eigenvectors| of adj, one per column,
 *   z     (N,) atomic numbers                                           columns by descending eigenvalue (perm.py:185-186)
 *   pairs (n_pairs, 2) int64 with 0 <= i < j < M, in any order and with repeats allowed, or NULL = every i < j in
 *         row-major order (n_pairs is then ignored and taken as M(M-1)/2)
 *   match_cost  with a pair list (n_pairs,); for all pairs (M, M) of which entry [i][j], i < j, is written and no other
 *   perms       (n_pairs, N) int32 or NULL;   has_perm (n_pairs,) bytes or NULL: one row per pair, in the list's order
 * adj, absv, match_cost, perms and has_perm may be host or device pointers; z and pairs are read on the host.  2 <= N
 * <= 1023, 1 <= M <= 65535.  Argument errors are reported before the device is touched.  The call returns after the
 * kernel has finished, whatever the pointers.  Results are bit-identical between calls and between the two forms; the
 * kernel ends after a number of steps bounded by the sizes alone for any input, NaN included.
 * Up to 112 atoms the cost matrix of a pair lives in shared memory, above in a per-CTA slab of a persistent global
 * workspace (freed by sgdml_b200_release_workspaces).  Launches count under family 8. */
int sgdml_b200_bipartite_match(const double* adj, const double* absv, const int64_t* z, int64_t n_geo, int64_t n_atoms,
                               const int64_t* pairs, int64_t n_pairs, double* match_cost, int32_t* perms,
                               uint8_t* has_perm, void* stream);
/* How sgdml_b200_bipartite_match runs at n_atoms atoms (host only: needs no device).  Writes 5 values to out:
 *   {cost matrix (0 shared memory, 1 global slab), threads per CTA, dynamic shared memory bytes, slab doubles per CTA,
 *    persistent CTAs per SM}. */
int sgdml_b200_bipartite_match_plan(int64_t n_atoms, int64_t* out);

/* ---------------------------------------------------------------- dense solve (path a) */

/* scipy.linalg.cho_factor (LAPACK dpotrf) as used by analytic.py:94-96 and
 * iterative.py:447-449.  A (n, n) symmetric, row stride lda; only the LOWER triangle
 * (row-major) is read, and on return it holds L (A = L L^T).  Strictly upper entries near
 * the diagonal (inside the diagonal blocks the trailing updates store whole) may be
 * overwritten with intermediate values; nothing reads them.  Padding columns (lda > n) are
 * neither read nor written.  Returns info > 0 if the leading minor of order info is not
 * positive definite (analytic.py:101 catches the resulting LinAlgError). */
int sgdml_b200_potrf(double* A, int64_t n, int64_t lda, void* stream);

/* scipy.linalg.cho_solve (dpotrs), analytic.py:97-99: solves L L^T X = B in place.
 * L from sgdml_b200_potrf; B (n, nrhs) row-major with row stride ldb. */
int sgdml_b200_potrs(const double* L, int64_t n, int64_t lda, double* B, int64_t nrhs,
                     int64_t ldb, void* stream);

/* Analytic.solve core, analytic.py:65-99: given Kneg = -K_ref (n, n) (device or host;
 * overwritten), adds lam to the diagonal, factorises, and returns
 * alphas = -(Kneg + lam I)^-1 y. */
int sgdml_b200_solve_analytic(double* Kneg, int64_t n, int64_t lda, double lam, const double* y,
                              double* alphas, void* stream);

/* ---------------------------------------------------------------- iterative solver blocks (path a)
 * Nystroem preconditioner of solvers/iterative.py:208-351 on X = K_nm (n_rows x m, row stride ldx),
 * the kernel columns at the inducing columns, resident in HBM (all matrix pointers below must be
 * DEVICE pointers; vectors may be host or device). */

/* K_mm = -X[row_idxs, :] (iterative.py:253); out (m x m), row stride ldo. */
int sgdml_b200_gather_rows_neg(const double* X, int64_t ldx, int64_t m, const int64_t* row_idxs,
                               double* out, int64_t ldo, void* stream);
/* A[i][i] += value (the jitter escalation of _cho_factor_stable, iterative.py:414-471). */
int sgdml_b200_add_diag(double* A, int64_t n, int64_t lda, double value, void* stream);
/* X <- X L^-T for lower-triangular L (m x m): scipy.linalg.solve_triangular(L, X.T, lower=True).T, which is
 * iterative.py:278-287 and 337-347 with the upper factor U = L^T of cho_factor.  Only the lower triangle of L
 * is read. */
int sgdml_b200_trsm_right_lt(const double* L, int64_t m, int64_t ldl, double* X, int64_t n_rows,
                             int64_t ldx, void* stream);
/* C = X^T X + lam I, lower triangle (iterative.py:293-295).  Strictly upper entries of C inside the
 * 128 x 128 diagonal tiles may be written too (with the same products); padding columns (ldc > m) are not. */
int sgdml_b200_gram_tn(const double* X, int64_t n_rows, int64_t m, int64_t ldx, double lam, double* C,
                       int64_t ldc, void* stream);
/* Posterior covariance blocks of an analytic-solver model (sgdml_b200/posterior.py, DESIGN.md section 4.1.13).
 * V (DEVICE, (3N + 1) n_query rows of n columns, row stride ldv >= n) holds the solved cross rows C(z, X) L^-T of
 * n_query queries in the row layout of sgdml_b200_assemble_ecstr_rows: the 3N force rows of query q at q 3N + r, then
 * the energy row of q at 3N n_query + q.  prior (n_query, d, d), d = 3N + 1, holds P_q = C(z_q, z_q) in the order
 * [F (3N); E] with the energy row and column standing for -E, as assembled.  Writes, for every query,
 *   out[q][i][j] = scale * sgn(i, j) * (P_q[i][j] - sum_k V[row(q, i)][k] V[row(q, j)][k]),
 * sgn = -1 where exactly one of i, j is the energy component (the blocks are for +E), +1 elsewhere.  Only the lower
 * triangle of P_q is read; each entry i >= j is computed once and stored at [i][j] and [j][i], so out is exactly
 * symmetric.  The sum over k runs in fixed 4096-column slices, each in increasing k, then over the slices in order,
 * without atomics: out[q] is bit-identical whatever n_query and whichever position q has.  prior and out may be host
 * or device pointers.  1 <= n_query <= 65535, 1 <= N <= 1023.  Returns after the kernels have finished. */
int sgdml_b200_posterior_blocks(const double* V, int64_t ldv, int64_t n, int64_t n_query, int64_t n_atoms,
                                const double* prior, double scale, double* out, void* stream);
/* out[r] = |X[r, :]|^2 -- the leverage scores (iterative.py:107-109). */
int sgdml_b200_row_sqnorms(const double* X, int64_t n_rows, int64_t m, int64_t ldx, double* out,
                           void* stream);
/* out = (X (X^T v) - v) / lam -- the preconditioner P v (iterative.py:136-138). */
int sgdml_b200_nystroem_apply(const double* X, int64_t n_rows, int64_t m, int64_t ldx, double lam,
                              const double* v, double* out, void* stream);

/* The two halves of sgdml_b200_nystroem_apply for a ROW-SHARDED factor (SURVEY.md section 8e
 * "Nystroem factor (m,n): shard n"): each GPU holds the rows X_loc of its own training points,
 *   t_loc = X_loc^T v_loc            (project; the caller all-reduces t over the GPUs)
 *   out_loc = (X_loc t - v_loc)/lam  (expand;  the caller all-gathers out)
 * which together are iterative.py:136-138 on the full factor. */
int sgdml_b200_nystroem_project(const double* X, int64_t n_rows, int64_t m, int64_t ldx,
                                const double* v, double* t, void* stream);
int sgdml_b200_nystroem_expand(const double* X, int64_t n_rows, int64_t m, int64_t ldx, double lam,
                               const double* t, const double* v, double* out, void* stream);

/* ---------------------------------------------------------------- device-resident PCG (path a, large systems)
 * scipy.sparse.linalg.cg as driven by Iterative.solve, iterative.py:740-752, on the operators of
 * iterative.py:183-206 (K v = predict_train(alphas = v), here sgdml_b200_model_set_alphas +
 * sgdml_b200_predict_train on `model`, which must have been given its training Jacobians with
 * sgdml_b200_model_set_R_d_desc) and iterative.py:120-142 (P v = (X (X^T v) - v)/lam with the Nystroem
 * factor X = B^T).  Solves (-K + lam I) x = y; the caller takes alphas = -x (iterative.py:803).
 * All CG vectors stay in HBM (`workspace`, DEVICE memory of at least
 * sgdml_b200_pcg_workspace_doubles(n, n_rows_loc, m_ind, check_every) doubles, n = 3N * n_train); the host sees
 * the residual norms of the last iterations every <= check_every iterations through `progress` (non-zero
 * return = stop: the reference's restart / interrupt logic, iterative.py:726-735), nothing else.
 *   y (n), x (n, in: start vector unless x_is_zero, out: solution): host or device.
 *   tol_abs: stop when |r| <= tol_abs (the reference passes tol * |y|, iterative.py:744).
 * Several GPUs (SURVEY.md 8e): this rank evaluates the K.v rows of training points [m_begin, m_end) and holds
 * the rows X_loc ((m_end - m_begin)*3N x m_ind, row stride ldx) of the factor; `exchange` is called, in stream
 * order, with DEVICE buffers inside `workspace`:
 *   op 0: sum `count` doubles at `buf` over the ranks in place   (X^T v, m_ind doubles)
 *   op 1: all-gather: `buf` is the full force vector (count = 3N * n_train), the rows this rank owns are in place
 *   op 2: all-gather of the energy tail (sgdml_b200_pcg_ecstr only): `buf` is the M-entry tail (count = n_train),
 *         entries [m_begin, m_end) are this rank's and in place
 * and must enqueue the collective on `stream` (torch.distributed / NCCL on the Python host).  exchange == NULL:
 * single rank, m_begin = 0, m_end = n_train.  m_ind = 0: no preconditioner (z = r). */
typedef int (*sgdml_b200_exchange_fn)(void* ctx, int op, double* buf, int64_t count);
typedef int (*sgdml_b200_pcg_progress_fn)(void* ctx, int64_t iters_done, const double* resid_hist, int64_t n_new);
int64_t sgdml_b200_pcg_workspace_doubles(int64_t n, int64_t n_rows_loc, int64_t m_ind, int64_t check_every);
int sgdml_b200_pcg(sgdml_b200_model* model, int64_t m_begin, int64_t m_end, const double* X_loc, int64_t m_ind,
                   int64_t ldx, double lam, const double* y, double* x, int x_is_zero, double tol_abs,
                   int64_t max_iters, int64_t check_every, double* workspace, int64_t workspace_doubles,
                   sgdml_b200_exchange_fn exchange, void* exchange_ctx, sgdml_b200_pcg_progress_fn progress,
                   void* progress_ctx, int64_t* iters_out, double* resid_out, void* stream);

/* The same solve with energy constraints in the kernel (use_E_cstr): n = 3N * n_train + n_train, vectors in the
 * layout [forces; energies], K v = [F; -E] of the predictor with alphas_F = v[:3NM], alphas_E = v[3NM:] (raw sums,
 * iterative.py:183-204).  X_loc holds this rank's force rows, then its energy rows: (m_end - m_begin)(3N + 1) rows
 * (sgdml_b200_assemble_ecstr_rows' layout).  Every K.v and P.v ends with op 1 on the force part and op 2 on the
 * energy tail.  `workspace` holds at least sgdml_b200_pcg_ecstr_workspace_doubles(n, n_rows_loc, m_ind,
 * check_every) doubles, n_rows_loc = (m_end - m_begin)(3N + 1): the common layout plus two n_rows_loc-vectors that
 * stage this rank's two segments in X_loc's row order. */
int64_t sgdml_b200_pcg_ecstr_workspace_doubles(int64_t n, int64_t n_rows_loc, int64_t m_ind, int64_t check_every);
int sgdml_b200_pcg_ecstr(sgdml_b200_model* model, int64_t m_begin, int64_t m_end, const double* X_loc, int64_t m_ind,
                         int64_t ldx, double lam, const double* y, double* x, int x_is_zero, double tol_abs,
                         int64_t max_iters, int64_t check_every, double* workspace, int64_t workspace_doubles,
                         sgdml_b200_exchange_fn exchange, void* exchange_ctx, sgdml_b200_pcg_progress_fn progress,
                         void* progress_ctx, int64_t* iters_out, double* resid_out, void* stream);

/* C = alpha * A * B^T + beta * C on the FP64 tensor pipe (the building block of potrf's
 * trailing update; exported for tests and benchmarks).  A (m, k) lda, B (n, k) ldb,
 * C (m, n) ldc, all row-major device or host. */
int sgdml_b200_dgemm_nt(int64_t m, int64_t n, int64_t k, double alpha, const double* A,
                        int64_t lda, const double* B, int64_t ldb, double beta, double* C,
                        int64_t ldc, void* stream);

/* Test hook: the internal GEMM launch exactly as potrf, trsm_right_lt, gram_tn and the large-descriptor predictor issue
 * it, which sgdml_b200_dgemm_nt (mode 0, tri 0, no flag) cannot reach.
 *   mode 0: C = alpha A B^T + beta C (C is not read when beta == 0);  mode 1: C += A B^T, alpha and beta ignored.
 *   tri 1 (needs m == n): only the lower triangle is computed.  The tile kernels write whole 128 x 128 tiles that touch
 *         it, entries above the diagonal inside the diagonal tiles included, and no tile strictly above the diagonal;
 *         the scalar kernel writes no entry with col > row.
 *   abort_flag: NULL, or a device int; when it is non-zero at kernel start the call leaves C unchanged.
 * All pointers must be DEVICE pointers: nothing is staged, and the call returns without synchronising.  The kernel is
 * the one sgdml_b200_set_gemm_variant selects. */
int sgdml_b200_gemm_nt_args(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                            const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int mode, int tri,
                            const int* abort_flag, void* stream);

/* The same product through the int8 tensor
 * cores -- A and B are cut into n_slices signed 7-bit slices per row-scaled entry and every slice pair is
 * multiplied exactly by wgmma s8 (int32 accumulators in registers); C += alpha * A * B^T.
 * n_slices = 7 reproduces the FP64 Cholesky trailing update (analytic.py:94-96) to ~1e-14 relative, 8 would
 * be FP64-equivalent (tools/ozaki_study.py).  n_slices must be 2..7.
 *   k <= 16384: the int32 level sums (at most 64^2 k n_slices) stay exact.  k = 16385 is an argument error.
 *   Each row x of A and of B is x = 2^e sum_p q_p 2^(-7 p), e = frexp(max |x|) + 1, q_p = rint of the remainder scaled
 *         by 2^7, p = 1..n_slices; the pairs with p + q <= n_slices + 1 are summed level by level, smallest level
 *         first, in FP64, and the update is ldexp(alpha * sum, e_A + e_B) (tests/ozaki_model.py states it bit for bit).
 *   Non-finite operands: every entry of C whose row of A or row of B holds a NaN or an infinity becomes NaN.
 *   tri != 0 (needs m == n): the kernel computes 128 x 32 tiles of C and writes every entry of each tile (tm, tn) with
 *         32 tn <= 128 tm + 127, entries above the diagonal included; every other entry of C keeps its bits.
 * All pointers must be device pointers. */
int sgdml_b200_ozaki_gemm_nt(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                             const double* B, int64_t ldb, double* C, int64_t ldc, int n_slices, int tri,
                             void* stream);
/* Test hook: the int8-slice GEMM launched exactly as its callers launch it, which sgdml_b200_ozaki_gemm_nt cannot reach.
 * Each operand is split once (once in all when A == B, m == n and lda == ldb, as potrf's symmetric update does), then
 * one launch: overwrite 0: C += alpha A B^T;  overwrite 1: C = alpha A B^T, the old C is not read (the large-descriptor
 * predictor's first write of S1, S2 and G).  tri and overwrite must be 0 or 1; otherwise the arguments and their
 * rejections are those of sgdml_b200_ozaki_gemm_nt.  Device pointers only; the call synchronises the stream. */
int sgdml_b200_ozaki_gemm_args(int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                               const double* B, int64_t ldb, double* C, int64_t ldc, int n_slices, int tri,
                               int overwrite, void* stream);
/* Bring-up aid for the above: also returns the int8 slice planes ([n_slices][rows padded to 128][k padded to
 * 128]), the row exponents and the raw int32 level sums ([n_slices][m][n]); any output may be NULL. */
int sgdml_b200_ozaki_debug(int64_t m, int64_t n, int64_t k, const double* A, int64_t lda, const double* B,
                           int64_t ldb, double* C, int64_t ldc, int n_slices, int8_t* planes_a, int* exps_a,
                           int8_t* planes_b, int* exps_b, int* levels, void* stream);

/* ---------------------------------------------------------------- launch accounting / profiling
 * Kernel families: 0 predictor main kernel, 1 predictor auxiliary kernels, 2 K assembly,
 * 3 DMMA GEMM (Cholesky trailing update), 4 potf2 diagonal tiles, 5 panel TRSM strips,
 * 6 triangular solves, 7 descriptor kernels, 8 misc (the permutation search's matching kernel among them), 9 the
 * predictor's finishing kernels for
 * descriptors longer than 25,600 entries (N >= 227 atoms; shorter ones finish under family 1).
 * `launches` counts kernel launches per family since the last reset (always on).  With
 * profiling enabled, the library brackets each family's launches with CUDA events on the
 * launching stream and accumulates the device time (this synchronises; benchmarks enable it
 * only for the roofline measurement, never inside a throughput-timed region). */
int sgdml_b200_profile_enable(int on);
int sgdml_b200_profile_reset(void);
int sgdml_b200_profile_get(int family, double* total_ms, int64_t* scopes, int64_t* launches);

/* FP64 tensor-pipe peak of the current device, measured live with a register-resident
 * mma.sync.m8n8k4.f64 loop (TFLOP/s); the roofline denominator for the FP64 kernels. */
int sgdml_b200_fp64_peak_tflops(double* tflops);
/* Same probe held for `seconds` (<= 30); reports the second half: the sustained figure for
 * kernels timed inside a long step (clocks settle under the power cap). */
int sgdml_b200_fp64_peak_tflops_sustained(double seconds, double* tflops);

/* Trailing updates of the Cholesky factorisation: -1 = automatic (default), 0 = FP64 DMMA, 2..7 = that many signed 7-bit
 * slices per operand on the int8 tensor cores (wgmma s8, exact int32 accumulation in registers, summed in FP64;
 * csrc/ozaki.cu).  Automatic = the environment variable SGDML_B200_OZAKI_SLICES if set, otherwise FP64 (on an H100 the
 * FP64 DMMA trailing updates are faster than 7 int8 slices at BASELINE config 2, and exact). */
int sgdml_b200_set_solve_slices(int n_slices);
/* The slice count the next factorisation will use (0 = FP64 DMMA), after resolving the automatic setting. */
int sgdml_b200_get_solve_slices(void);

/* Test / tuning hook: selects the GEMM kernel used by dgemm_nt and potrf's trailing update.
 * 0 = 128x128 DMMA tiles fed by cp.async, 2 = scalar FMA reference kernel, 3 = 128x128 DMMA tiles fed by TMA tensor
 * maps (cp.async.bulk.tensor + mbarrier ring; default).  Any other value is rejected.  Whatever the setting, operands
 * the tiled kernels cannot load (odd k or strides, or not 16-byte aligned) run the scalar kernel, and 3 runs the
 * cp.async tiles when the driver offers no tensor-map encoder. */
int sgdml_b200_set_gemm_variant(int variant);

#ifdef __cplusplus
}
#endif
#endif /* SGDML_B200_H */
