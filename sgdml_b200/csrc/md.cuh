// Molecular dynamics on the device (sgdml_b200_md_*, sgdml_b200_remd_run, sgdml_b200_npt_*, sgdml_b200_metad_*,
// sgdml_b200_umbrella_*, sgdml_b200_pimd_*, sgdml_b200_relax_*, sgdml_b200_neb_fire, sgdml_b200_dimer_fire,
// sgdml_b200_irc_rk4): the contract of the kernels in md.cu -- the BAOAB integrator step, the replica exchange, the NPT
// step, the metadynamics bias, the umbrella restraints and their exchange, the ring-polymer step, their counter-based
// noise, the FIRE and L-BFGS steps, the nudged elastic band, the dimer search and the reaction path -- and of MBAR in
// mbar.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgdml {

// Everything a run changes, read by the step kernel from device memory: a captured step graph bakes in none of it.
// Frame pointers are device pointers or null (that output is not written).
struct MdParams {
  double h;           // dt / 2
  double c1;          // exp(-gamma dt)
  uint32_t key[2];    // Philox key: (seed mod 2^32, seed >> 32)
  int use_O;          // 0: gamma == 0, plain velocity Verlet (no draws)
  int stride;         // 0: no frames
  uint64_t run_start; // the handle's step index when the run began
  double *R_f, *V_f, *Ep_f, *Ek_f;  // frames (n_frames, n_rep, 3N) / (n_frames, n_rep)
  int n_temps;        // rows of the sigma table: replica rep uses row rep % n_temps (1: one temperature)
};

// k_md_step: one step for every replica (grid: one CTA of MD_THREADS per replica).  With the handle's step counter at n:
//   if n != run_start:  v += h (F s)        second half-kick of step n - 1 (F is F(r) of the positions in R)
//                       frame (n - run_start) / stride - 1 when that is whole: R, full-step V, E_pot, E_kin
//   if advance:         B, A, O (noise of step n), A; R and V hold the new positions and half-step velocities,
//                       and the counter becomes n + 1
// advance == 0 only completes the last step of a run.  s: (3N) inverse mass per coordinate; sigma: (n_temps, 3N)
// noise scale per temperature and coordinate, row rep % n_temps for replica rep.
constexpr int MD_THREADS = 128;

// Replica exchange (sgdml_b200_remd_run): a plain MD handle of n_rep = n_ladders n_temps replicas; slot l n_temps + k
// is temperature k of ladder l for the whole run, and exchanges move configurations between slots.
struct RemdParams {
  uint32_t key[2];      // the run's Philox key, as MdParams
  uint64_t run_start;   // as MdParams
  int64_t every;        // E: an exchange on the state at c when E >= 1, c > run_start and c % E == 0 (0: never)
  int n_temps;          // slots per ladder (>= 2)
  int stride;           // as MdParams (0: no walker frames)
  const double* beta;   // (n_temps) 1 / kT_k
  const double* lam_up; // (n_temps - 1) sqrt(kT_k+1 / kT_k): the configuration moving from slot k to k + 1
  const double* lam_dn; // (n_temps - 1) sqrt(kT_k / kT_k+1): the configuration moving from slot k + 1 to k
  int64_t *n_acc, *n_att;  // (n_ladders, n_temps - 1) accepted and attempted swaps of pair (k, k + 1) in this run
  int* W_f;             // walker frames (n_frames, n_rep), or null
};

// k_remd_exchange: one CTA of MD_THREADS per ladder, launched before k_md_step on the same counter c (the state R
// holds).  V holds the velocity before k_md_step's pending half-kick.  On an exchange step, with e = c / E, the pairs
// (k, k + 1) with k % 2 == e % 2 and k + 1 < n_temps are attempted, each independently:
//   D = (beta_k - beta_k+1) (E_k - E_k+1)   (rounded as written)
//   accepted iff D >= 0 or u < exp(D), u = uniform53 of words 0, 1 of Philox4x32-10 under the run's key with counter
//   (0x80000000 | k, l, c mod 2^32, c >> 32)  (the O noise's first counter word is a pair index below 2^31)
// An accepted swap exchanges the R, F and E rows and the walker labels of the two slots, and the velocity of each
// configuration, moving from slot a to slot b with lam = sqrt(kT_b / kT_a), becomes
//   w = v + h (F s)  (k_md_step's rounding),  v' = lam w - h (F s)
// with the configuration's own F.  n_att and n_acc of the pair count the attempt and the acceptance.  On a frame step
// of k_md_step (the same rule) the CTA writes the ladder's walker labels after the swaps into W_f.

// Constant-pressure MD (sgdml_b200_npt_run): an NPT handle (sgdml_b200_npt_create) is an MD handle whose replica rep
// lives in a cell of its own, isotropically scaled by the stochastic cell rescaling barostat (Bernetti & Bussi,
// J. Chem. Phys. 153, 114107 (2020)).  Per replica, in device memory:
struct NptCell {
  double eps;              // log of the volume ratio V / V0 since the cell was set
  double V0;               // |det L0|, computed on the host
  double L0[9], L0inv[9];  // the base cell (lattice vectors as columns, row-major) and the inverse the caller gave
};
// The cell the descriptor kernel reads is the Lattice L = a L0, L^-1 = L0^-1 / a with a = exp(eps / 3) (each entry one
// product or quotient), so it never drifts from its inverse.  W (n_rep, 9) holds the virial of the current state,
// written with F and E by force_eval_run_cells (predict.cuh).
struct NptParams {
  double P0;              // target pressure (energy / L^3)
  double c_a;             // (beta_T / tau_p) dt, on the host
  double c_b;             // 2 kT (beta_T / tau_p) dt, on the host (0: no draws)
  double *cell_f, *P_f;   // frames (n_frames, n_rep, 9) / (n_frames, n_rep), or null
};

// k_npt_step: one CTA of MD_THREADS per replica, k_md_step's counter, run_start and stride rules (MdParams; sigma row
// 0).  With the replica's counter at n:
//   1. if n != run_start:  v += h (F s), as k_md_step; on a frame step R, full-step V, E_pot, E_kin as k_md_step, the
//      cell a L0 (the Lattice's vectors) and P_int of step 2
//   2. K = 1/2 sum_i v_i^2 / s_i in k_md_step's E_kin order (on every step);  V = V0 exp(eps);
//      P_int = (2 K + ((W_0 + W_4) + W_8)) / (3 V), rounded as written
//   3. if advance:  de = -c_a (P0 - P_int) + sqrt(c_b / V) eta, rounded as written (c_b == 0: the first term only,
//      no draw); eta = sqrt(-2 ln U_a) cos(2 pi U_b) from Philox4x32-10 under the run's key with counter
//      (0xFFFFFFFF, rep, n mod 2^32, n >> 32), U_a and U_b as k_md_step's.  That first counter word is above every O
//      pair index (< 2^31) and every exchange word (0x80000000 | k, k <= 2^31 - 3).
//   4. if advance:  B, A, O, A exactly as k_md_step (one copy of the update, its noise), then mu = exp(de / 3),
//      r = r mu, v = v / mu, eps = eps + de, the new Lattice, and the counter becomes n + 1
// The driver then evaluates F, E and W at the new positions in the new cells; the next launch's first action is the
// pending half-kick with those forces.
// Drift: velocities scaled by 1 / mu keep dr dp, and with the instantaneous K in P_int the Ito drift that leaves
// exp(-beta (H + P0 V)) dr dp dV stationary carries no kT / V term (DESIGN.md 4.1.7 has the derivation).

// Multiple-walker metadynamics (sgdml_b200_metad_run): a metadynamics handle (sgdml_b200_metad_create) is an MD handle
// of n_rep = n_groups n_walkers replicas, replica g n_walkers + w walker w of group g, integrated by k_md_step (sigma
// row 0).  The walkers of a group deposit Gaussian hills into one store and are biased by it; groups never see each
// other's hills.  Collective variables (CVs), at most MD_MAX_CV, each of a type and up to 4 distinct atoms i, j, k, l,
// on plain coordinate differences (no minimum image, as NEB: positions are never wrapped).  Every product, sum,
// difference and quotient below is rounded as written (no fused multiply-add); dot(a, b) = (a0 b0 + a1 b1) + a2 b2,
// cross(a, b) = (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0), |a| = sqrt(dot(a, a)), and x / y of a vector by a scalar
// divides each component.
//   CV_DISTANCE  d = r_j - r_i;  s = |d|;  ds/dr_j = d / s, ds/dr_i = -(d / s)  (both 0 when s == 0)
//   CV_ANGLE     a = r_i - r_j, b = r_k - r_j, c = cross(a, b), cn = |c|;  s = atan2(cn, dot(a, b)) in [0, pi];
//                ds/dr_i = cross(a, c) / (dot(a, a) cn), ds/dr_k = cross(c, b) / (dot(b, b) cn),
//                ds/dr_j = -(ds/dr_i + ds/dr_k)  (all 0 when cn == 0: the collinear case)
//   CV_DIHEDRAL  b1 = r_j - r_i, b2 = r_k - r_j, b3 = r_l - r_k, m = cross(b1, b2), n = cross(b2, b3), nb = |b2|;
//                s = atan2(nb dot(b1, n), dot(m, n)) in (-pi, pi] (Blondel & Karplus, J. Comput. Chem. 17, 1132 (1996));
//                gi = -((nb / dot(m, m)) m), gl = (nb / dot(n, n)) n, p = dot(b1, b2) / dot(b2, b2),
//                q = dot(b3, b2) / dot(b2, b2), t = p gi - q gl;  ds/dr_i = gi, ds/dr_l = gl, ds/dr_j = -(gi + t),
//                ds/dr_k = t - gl  (all 0 when dot(m, m) == 0 or dot(n, n) == 0)
// A hill k of the store has a centre c_k, widths w_k (per CV) and a height h_k.  Per hill, j over the CVs in order:
//   e_j = s_j - c_kj, for a dihedral wrapped into [-pi, pi) by one step: e_j >= pi: e_j - 2 pi, e_j < -pi: e_j + 2 pi
//   (pi and 2 pi the doubles nearest them);  u_j = e_j / w_kj;  a = sum_j u_j u_j from 0.0;  x = h_k exp(-0.5 a);
//   V += x;  dV_j -= x (u_j / w_kj)
// V = sum_k h_k exp(-sum_j e_kj^2 / (2 w_kj^2)) and dV_j = dV/ds_j in block_sum's order: thread t adds the terms of
// hills t, t + MD_THREADS, ... from 0.0 in increasing k, then the tree.  The bias force on an atom a touched by a CV is
// Fb_a = sum over the CVs j in order of -(dV_j ds_j/dr_a) from 0.0 (only the CVs that hold a add a term), and the
// force k_md_step reads is F = Fm + Fb_a, rounded once; coordinates no CV touches get F = Fm.
constexpr int MD_MAX_CV = 4;
enum CvType { CV_DISTANCE = 0, CV_ANGLE = 1, CV_DIHEDRAL = 2 };

struct MetadParams {
  int n_cv, n_walkers;
  int type[MD_MAX_CV];
  int atoms[MD_MAX_CV][4];   // unused entries 0
  int64_t pace;              // a deposit on every state c with c % pace == 0
  int64_t cap;               // hill slots per group
  double w0;                 // the initial height
  double dkT;                // the well-tempered Delta kT, > 0 (+inf: plain metadynamics)
  double width[MD_MAX_CV];   // the widths the run deposits
  double *centers, *widths;  // (n_groups, cap, n_cv) the hill store
  double* heights;           // (n_groups, cap)
  const int64_t* count;      // (n_groups) hills committed before the run
  double *cv, *Vb, *Fb;      // the state's CVs (n_rep, n_cv), bias energy (n_rep) and bias force (n_rep, 3N)
  double *cv_f, *bias_f;     // frames (n_frames, n_rep, n_cv) / (n_frames, n_rep), or null
};

// k_metad_bias: one CTA of MD_THREADS per replica, launched after the force evaluation that wrote the model force Fm
// and E of the state R holds, with the replica's counter at c.  It computes s and ds/dR, V and dV over the n_g hills
// of group g committed so far, writes F = Fm + Fb, the state's s, V and Fb, and with deposit == 1 (inside a run, with
// MdParams' run_start and stride):
//   n_g = count[g] + n_walkers ((c - 1) / pace - run_start / pace)  (the deposits of this run before state c; 0 with
//         deposit == 0), so every walker of a group reads the same hills, and a hill deposited on state c becomes
//         visible to the evaluation of state c + 1, never to its own;
//   frame (c - run_start) / stride - 1 when that is whole: s and V of state c (V before its deposit);
//   if c % pace == 0 (and c > run_start, which always holds inside a run): walker w writes slot n_g + w of its group:
//         centre s, widths MetadParams.width, height w0 exp(-V / dkT) (w0 with dkT = +inf).
// The driver commits a run's hills after it: count[g] += n_walkers #{c in (run_start, run_start + n_steps] :
// c % pace == 0}.  The store's address is read from MetadParams, not baked into the step graph.

// Umbrella sampling with Hamiltonian replica exchange (sgdml_b200_umbrella_run; REUS: Sugita, Kitao & Okamoto, JCP 113,
// 6042 (2000)): an umbrella handle (sgdml_b200_umbrella_create) is an MD handle of n_rep = n_ladders n_windows replicas,
// slot l n_windows + k window k of ladder l, integrated by k_md_step (sigma row 0: one temperature).  Its CVs are the
// metadynamics CVs above (types, atoms, formulas, no minimum image).  Window k restrains CV j about the centre c_kj with
// the force constant kappa_kj >= 0; per CV j in increasing order, from b = 0.0, every operation rounded as written:
//   e_j = s_j - c_kj (a dihedral's wrapped into [-pi, pi) by one step, as a hill difference);  u_j = kappa_kj e_j;
//   b = b + (0.5 u_j) e_j;  db/ds_j = u_j
// umbrella_restraint below is the one copy of it: the step graph, the exchange and MBAR all call it.  The bias force
// is the metadynamics one with dV_j = u_j: Fb_a = sum over the CVs j holding atom a of -(u_j ds_j/dr_a) from 0.0, and
// F = Fm + Fb_a rounded once on the touched atoms, F = Fm elsewhere.
struct UmbrellaParams {
  int n_cv, n_windows;
  int type[MD_MAX_CV];
  int atoms[MD_MAX_CV][4];   // unused entries 0
  double beta;               // 1 / kT of the run (read by the exchange only)
  const double* win;         // the window table: centres (n_windows, n_cv), then force constants (n_windows, n_cv)
  double *cv, *Vb, *Fb;      // the state's CVs (n_rep, n_cv), restraint energy (n_rep) and bias force (n_rep, 3N)
  double *cv_f, *bias_f;     // frames (n_frames, n_rep, n_cv) / (n_frames, n_rep), or null
};

#ifdef __CUDACC__
// b of CVs s (n_cv) under one window (centres c, force constants kappa, n_cv each); u (null: not wanted) gets db/ds
__device__ __forceinline__ double umbrella_restraint(int n_cv, const int* type, const double* s, const double* c,
                                                     const double* kappa, double* u) {
  double b = 0.0;
  for (int j = 0; j < n_cv; ++j) {
    double e = __dsub_rn(s[j], c[j]);
    if (type[j] == CV_DIHEDRAL) {
      if (e >= M_PI)
        e = __dsub_rn(e, 2.0 * M_PI);
      else if (e < -M_PI)
        e = __dadd_rn(e, 2.0 * M_PI);
    }
    const double uj = __dmul_rn(kappa[j], e);
    if (u != nullptr) u[j] = uj;
    b = __dadd_rn(b, __dmul_rn(__dmul_rn(0.5, uj), e));
  }
  return b;
}
#endif

// k_umbrella_bias: one CTA of MD_THREADS per replica, launched after the force evaluation that wrote the model force Fm
// and E of the state R holds.  Replica rep under window rep % n_windows: s and ds/dR (cv_eval), b and u, F = Fm + Fb,
// and the state's s, b and Fb.  It writes no frames.
//
// k_umbrella_exchange: one CTA of MD_THREADS per ladder, launched before k_md_step on the same counter c, with
// RemdParams' key, run_start, every, n_temps (= n_windows), stride, n_acc, n_att and W_f.  On an exchange (k_remd_exchange's
// schedule, pairing and Philox draw), with configuration a in slot k and b in slot k + 1 and b_k(s) the restraint of
// window k at the stored CVs s (umbrella_restraint):
//   d = -(beta ((b_k(s_b) + b_k+1(s_a)) - (b_k(s_a) + b_k+1(s_b))))  (rounded as written);  accepted iff d >= 0 or
//   u < exp(d)
// An accepted swap exchanges the R, Fm, E and CV rows and the walker labels of the two slots, recomputes Fb, b and
// F = Fm + Fb of both slots in their new windows (k_umbrella_bias's arithmetic), and each configuration keeps its
// full-step velocity: w = v + h (F_old s), v' = w - h (F_new s) (k_md_step's rounding of the kick).  On a frame step of
// k_md_step (the same rule; also with every == 0) it then writes the ladder's walker labels, CVs and b into W_f, cv_f,
// bias_f; k_md_step writes R, V, E_pot and E_kin of the same state.
//
// MBAR (sgdml_b200_umbrella_mbar; Shirts & Chodera, JCP 129, 124105 (2008), eq. 11), in mbar.cu.  K windows, samples
// s_n (n, n_cv) pooled with N_k of them from window k, u_kn = beta b_k(s_n) by umbrella_restraint (never stored).  From
// f = 0, each iteration:
//   L_n = m_n + log(sum_k exp(a_kn - m_n)), a_kn = (ln N_k + f_k) - u_kn, m_n = max_k a_kn, the sum in increasing k
//         from 0.0 (one thread per sample; ln N_k = -inf for an empty window)
//   f_k' = -logsumexp_n(-u_kn - L_n): thread t of CTA c folds its samples n = c MBAR_CHUNK + t, ... + MBAR_THREADS,
//         ... in increasing n into a running (max, sum) pair, then block_tree's fixed tree over the CTA merges the
//         pairs; one CTA per window then folds the per-CTA pairs, thread t those of CTA t, t + MBAR_THREADS, ... in
//         increasing c, and the same tree merges them (no atomics: the same bits on every call)
//   f' = f' - f'_0;  resid = max_k |f'_k - f_k|;  stop when resid < tol or after max_iter iterations
// The pair fold: (m, S) + x = x > m ? (x, S exp(m - x) + 1) : (m, S + exp(x - m)); a merge (m, S) + (m2, S2) with
// S2 > 0 is (m2, S exp(m - m2) + S2) when m2 > m, else (m, S + S2 exp(m2 - m)), and an empty pair (S = 0) adds nothing;
// logsumexp = m + log(S).  Every operation rounds as written.  After the last iteration L_n is evaluated once more with the final f, and log w_n = f_u - L_n with
// f_u = -logsumexp_n(-L_n) (the unbiased state), so that sum_n w_n = 1.
constexpr int MBAR_THREADS = 256;
constexpr int MBAR_CHUNK = 16 * MBAR_THREADS;  // samples per CTA of the f reduction

// The checks of a window table, shared by sgdml_b200_umbrella_create, _set_windows and _mbar: centers and kappas
// (n_windows, n_cv) HOST arrays, finite, kappa >= 0, a dihedral's centre in (-pi, pi].  Returns 0 or an argument error.
int umbrella_windows_check(int64_t n_windows, int n_cv, const int* type, const double* centers, const double* kappas);

// Path-integral MD (sgdml_b200_pimd_run): replica p P + j is bead j of ring polymer p.
constexpr int PIMD_MAX_BEADS = 64;  // C (P x P) sits in shared memory: 32 KB at the cap
constexpr int PIMD_TILE = 512;      // (bead, coordinate) elements of one tile: 4 per thread

struct PimdParams {
  double h;           // dt / 2
  uint32_t key[2];    // Philox key: (seed mod 2^32, seed >> 32)
  int use_O;          // 0: no mode is thermostatted (no draws)
  int stride;         // 0: no frames
  uint64_t run_start; // the handle's step index when the run began
  double kprim0;      // 3N P kT / 2
  double kspring;     // omega_P^2 / (2 P)
  double kcv0;        // 3N kT / 2
  double kvir;        // 1 / (2 P)
  double *R_f, *V_f, *Ep_f, *Ek_f;  // frames (n_frames, n_poly P, 3N) / (n_frames, n_poly P)
  double *Kp_f, *Kcv_f;             // frames (n_frames, n_poly)
};

// k_pimd_step: one PILE-L step for every ring polymer (grid: one CTA of MD_THREADS per polymer), the counterpart of
// k_md_step: the pending second half-kick and the frame (per bead R, full-step V, E_pot, E_kin; per polymer
// K_prim, K_cv), then, if advance, B, the transform to normal modes, A, O, A, the transform back.  tab: C (nb x nb,
// C[j nb + k]) followed by the mode tables cos(w_k h), sin(w_k h) / w_k, -w_k sin(w_k h), c1_k (nb each);
// sigma (nb, 3N) per mode and coordinate; s (3N) inverse masses.

// Geometry optimisation (sgdml_b200_relax_fire, sgdml_b200_relax_lbfgs): one CTA of MD_THREADS per replica.
//
// Sums.  Every dot product x.y and squared norm of a replica is block_sum's: thread t adds the products x_i y_i of its
// coordinates i = t, t + MD_THREADS, ... in increasing i, starting from 0.0 (each product and each addition rounded),
// then a tree over the MD_THREADS partials adds red[t] + red[t + w] for w = MD_THREADS / 2, ..., 1.  Per-atom maxima
// (|F_a|^2 for convergence, |d_a|^2 for the L-BFGS step cap) take |x_a|^2 = (x_a0 x_a0 + x_a1 x_a1) + x_a2 x_a2,
// rounded as written, and a NaN anywhere makes the maximum NaN.  Every update rounds as written: no fused
// multiply-add, so tests/relax_oracle.py, fed the same forces, reproduces the kernels bit for bit.
//
// Convergence: max_a |F_a|^2 < fmax2 at the current positions (ASE's criterion).  Each step kernel tests first; a replica
// that passes is frozen (its state and positions never change again in this call).  fmax2 = 0 never passes.
constexpr int LBFGS_MAX_MEMORY = 32;

// Per replica, zeroed at the start of every call: n_steps == 0 is the first step of the call.
struct RelaxState {
  double dt, alpha;     // FIRE: time step and mixing (set on the first step)
  double gamma;         // L-BFGS: s.y / y.y of the newest pair
  double E_prev;        // L-BFGS: the energy at r_prev
  double fmax2;         // max_a |F_a|^2 at the last test
  int64_t n_steps;      // position updates taken in this call
  int n_pos;            // FIRE: steps with F.v > 0 since the last reset
  int n_hist, head;     // L-BFGS: pairs in the ring and the slot of the newest
  int conv;             // 1: converged and frozen
};

// Everything a call changes, read from device memory: the captured step graph bakes in none of it.
struct RelaxParams {
  double fmax2;         // fmax^2 (0: run every step)
  double maxstep;       // FIRE: |dr| of the whole replica; L-BFGS: |d_a| of every atom
  double dt0, dtmax;    // FIRE
  double h0;            // L-BFGS: initial inverse Hessian when the history is empty
  int memory;           // L-BFGS: m, 1 <= m <= LBFGS_MAX_MEMORY
  int m_cap;            // L-BFGS: slots per replica in S, Y, rho (>= memory)
  double *S, *Y;        // L-BFGS: (n_rep, m_cap, 3N) ring of s and y
  double* rho;          // L-BFGS: (n_rep, m_cap) 1 / s.y
  double *r_prev, *g_prev;  // L-BFGS: (n_rep, 3N) positions and -F of the previous step
};

// k_fire_step: FIRE (Bitzek et al., PRL 97, 170201 (2006); ASE's mass-free form, Nmin 5, finc 1.1, fdec 0.5, alpha_start 0.1,
// f_alpha 0.99) with velocities V (n_rep, 3N).  After the test, on every step but the first:
//   P = F.v;  P > 0:  vv = v.v, ff = F.F, c = alpha (sqrt(vv) / sqrt(ff)), v = (1 - alpha) v + c F,
//                     if n_pos > 5: dt = min(dt 1.1, dtmax), alpha = alpha 0.99;  n_pos += 1
//             else:   v = 0, alpha = 0.1, dt = dt 0.5, n_pos = 0
// then on every step (the first starts from dt = dt0, alpha = 0.1, n_pos = 0 and the V the driver zeroed):
//   v = v + dt F,  dr = dt v,  |dr| = sqrt(dr.dr),  if |dr| > maxstep: dr = (maxstep dr) / |dr|,  r = r + dr.
//
// k_lbfgs_step: L-BFGS (Nocedal & Wright, Alg. 7.4) with g = -F, direction scratch D (n_rep, 3N).  On every step but the first:
//   s = r - r_prev, y = g - g_prev into the slot after the newest;  sy = s.y, yy = y.y;
//   sy > 0: push (rho = 1 / sy, gamma = sy / yy), the ring holding the newest min(n + 1, m);  else clear the history;
//   E > E_prev: clear the history.
// Then q = g; for pairs newest to oldest: a_k = rho_k (s_k.q), q = q - a_k y_k;  z = gamma q (h0 q with no history);
// for pairs oldest to newest: b = rho_k (y_k.z), z = z + s_k (a_k - b);  d = -z.  If d.g >= 0 (or NaN): clear the
// history and d = h0 F.  Cap: L = sqrt(max_a |d_a|^2), if L > maxstep: d = d (maxstep / L).  r_prev = r, g_prev = g,
// E_prev = E, r = r + d.
//
// advance == 0 runs only the test (it sets conv and fmax2 for every replica).
//
// k_relax_count writes the number of replicas not yet converged into *n_active (host-mapped pinned memory);
// k_relax_report writes n_steps (int64), conv (int32) and sqrt(fmax2) per replica into device arrays, each may be null.
// Both run over the driver's units of convergence: one replica for relaxation, one band for NEB (below).

// Nudged elastic band (sgdml_b200_neb_fire).  The handle's n_rep = n_bands P replicas hold n_bands bands of P >= 3
// images; replica b P + j is image j of band b.  Images 0 and P - 1 are fixed endpoints: they never move, but their
// forces and energies are evaluated every step with the rest of the batch, and their energies enter the tangents of
// their neighbours.  Image differences are plain coordinate differences, with no minimum image, also for periodic
// models.
//
// k_neb_force: one CTA of MD_THREADS per interior image (grid n_bands (P - 2)).  With E the model energy and F = -dE/dR
// of the image i and its neighbours, t+ = R[i+1] - R[i] and t- = R[i] - R[i-1] (each difference rounded), the tangent
// of Henkelman & Jonsson, J. Chem. Phys. 113, 9978 (2000), eqs. 8-11:
//   E[i+1] > E[i] > E[i-1]:  tau = t+;   E[i+1] < E[i] < E[i-1]:  tau = t-;
//   otherwise, dmax / dmin the larger / smaller of |E[i+1] - E[i]|, |E[i-1] - E[i]|:
//     E[i+1] > E[i-1]:  tau = t+ dmax + t- dmin;   else:  tau = t+ dmin + t- dmax
// nt = sqrt(tau.tau), np = sqrt(t+.t+), nm = sqrt(t-.t-), th = tau / nt (th = 0 when nt == 0: coincident images give
// no NaN), fd = F.th, all per image with block_sum's order.  Then
//   ordinary image:  F_neb = (F - fd th) + (k (np - nm)) th                  (eq. 12)
//   climbing image:  F_neb = F - (2 fd) th                                   (Henkelman, Uberuaga & Jonsson, JCP 113, 9901)
// The climbing image is the interior image of highest E, the lowest index on ties, chosen again at every evaluation,
// and climbs only when climb is set.  The CTA of image 1 writes that index per band to climb_idx.
//
// k_neb_fire_step: one CTA per band.  k_fire_step's test and update (fire_update in md.cu, one copy of the FIRE
// arithmetic) on the band's interior images as one vector of (P - 2) 3N coordinates, with F_neb for F: F.v, v.v, F.F,
// |dr| and the convergence test max_a |F_neb,a|^2 < fmax2 run over every atom of every interior image, and one
// RelaxState per band.  FIRE only: L-BFGS's energy-rise reset has no meaning for NEB forces, which are no gradient.
struct NebParams {
  double fmax2, maxstep, dt0, dtmax;  // the band FIRE, as in RelaxParams
  double k;                           // spring constant (force unit / L)
  int climb;                          // 1: the highest interior image climbs
  int P;                              // images per band (>= 3)
};

// Dimer saddle search (sgdml_b200_dimer_fire; Henkelman & Jonsson, J. Chem. Phys. 111, 7010 (1999)).  The handle's
// n_rep = 2 n_dimers replicas: replica 2d is the centre R0 of dimer d, replica 2d + 1 its image R1 = R0 + D N, with N
// the dimer's unit mode (n_dimers, 3N) and D the separation.  Every force evaluation covers both (F0, F1); the image 2
// is the central difference F2 = 2 F0 - F1, never evaluated.  Per dimer, with block_sum's order for every sum below
// (over the dimer's 3N coordinates, thread t adding its coordinates i = t, t + MD_THREADS, ... from 0.0, then the tree)
// and every operation rounded as written (no fused multiply-add):
//   C    = (sum_i (F0_i - F1_i) N_i) / D                        the curvature along N
//   G_i  = (F1_i - F0_i) / D;  g = sum_i G_i N_i;  P_i = G_i - g N_i;  f = sqrt(sum_i P_i P_i)   the rotational force
//
// k_dimer_step: one CTA of MD_THREADS per dimer, the dimer's RelaxState and DimerState.  Each launch:
//   1. Test (as k_fire_step: first, a converged dimer frozen for the rest of the call).  In phase EVAL_N, C_N = C of
//      the current forces.  fmax2 = atom_max2(F0);  conv = fmax2 < fmax2_thr and C_N < 0.  advance == 0 stops here.
//   2. EVAL_N (F1 belongs to R0 + D N).  If f < rot_min or f == 0: translate (4) with C_use = C_N.  Otherwise
//      T_i = P_i / f, C0 = C_N, b1 = -f, the image R1_i = R0_i + D Nt_i with Nt_i = c_t N_i + s_t T_i, phase TRIAL;
//      nothing else moves.
//   3. TRIAL (F1 belongs to R0 + D Nt; F0 unchanged): the curvature fit C(phi) = a0 / 2 + a1 cos 2phi + b1 sin 2phi in
//      the plane (N, T) (Heyden, Bell & Keil, JCP 123, 224101 (2005); Kastner & Sherwood, JCP 128, 014106 (2008)):
//        Ct = (sum_i (F0_i - F1_i) Nt_i) / D;  a1 = ((C0 - Ct) + b1 s2_t) / omc2_t;  r = sqrt(a1 a1 + b1 b1);
//        c2 = (-a1) / r;  s2 = (-b1) / r;
//        c2 >= 0:  c = sqrt((1 + c2) / 2), s = s2 / (2 c);   else:  s = sqrt((1 - c2) / 2), c = s2 / (2 s);
//        N_i = c N_i + s T_i, then the rigid projection and normalisation (5);  C_use = (C0 - a1) - r;  n_rot += 1
//   4. Translate:  p = sum_i F0_i N_i;  C_use < 0:  Fd_i = F0_i - (2 p) N_i;  else  Fd_i = -(p N_i);  then
//      fire_update (k_fire_step's FIRE, its constants and whole-vector maxstep cap) on R0 and the centre's V row with
//      Fd (which it keeps in the handle's Fn, row 2d), which counts the step in n_steps;  R1_i = R0_i + D N_i;  phase
//      EVAL_N.
// c_t = cos phi_t, s_t = sin phi_t, s2_t = 2 s_t c_t and omc2_t = 2 s_t s_t (1 - cos 2phi_t) are computed once on the
// host, so the kernels and tests/dimer_oracle.py use the same doubles.
//
// 5. Rigid projection of a mode N at centre R0 (n atoms), then N = N / sqrt(sum_i N_i N_i).  "Component sums" are
// block_sums over the 3N coordinates of the vector holding x_i at the coordinates i = 3a + c of component c and 0.0
// elsewhere; "atom sums" hold the atom's term at coordinate 3a and 0.0 at 3a + 1, 3a + 2 (a multi-value reduction with
// block_sum's tree for each value gives the same bits).
//   translations:  m_c = (component sum of N) / n,  N_i = N_i - m_c(i)
//   rotations (free molecules only; periodic models remove the translations only):
//     rb_c = (component sum of R0) / n;  x_a = R0_a - rb;  L = atom sums of cross(x_a, N_a);
//     I_00 = atom sum of (x1 x1 + x2 x2), I_11 of (x0 x0 + x2 x2), I_22 of (x0 x0 + x1 x1), I_01 = -(atom sum of
//     x0 x1), I_02 = -(x0 x2), I_12 = -(x1 x2);  cofactors A00 = I11 I22 - I12 I12, A01 = I02 I12 - I01 I22,
//     A02 = I01 I12 - I11 I02, A11 = I00 I22 - I02 I02, A12 = I01 I02 - I00 I12, A22 = I00 I11 - I01 I01;
//     det = (I00 A00 + I01 A01) + I02 A02;  t = ((I00 + I11) + I22) / 3;  if det > 1e-10 ((t t) t):
//     w_0 = ((A00 L0 + A01 L1) + A02 L2) / det, w_1 = ((A01 L0 + A11 L1) + A12 L2) / det,
//     w_2 = ((A02 L0 + A12 L1) + A22 L2) / det, and N_a = N_a - cross(w, x_a); otherwise (a linear or one-atom
//     geometry) no rotational part.
//   cross(a, b) = (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0), as the metadynamics CVs.
//
// k_dimer_init: one CTA of MD_THREADS per dimer, before the force evaluation of a call: the projection (5) of the
// source mode at the dimer's centre into a scratch mode, the image R0 + D N into a scratch image, and bad[d] = 1 when
// the source's N.N (before the projection) is not finite or the projected N.N is not above 1e-12 of it (a mode that is
// (almost) a rigid motion).  The driver commits the scratch rows only when no dimer is bad.
enum DimerPhase { DIMER_EVAL_N = 0, DIMER_TRIAL = 1 };

struct DimerState {  // per dimer, zeroed at the start of every call (phase EVAL_N)
  int phase;
  int64_t n_rot;     // rotations in this call
  double C_N;        // the curvature last measured along N at the current centre
  double C0, b1;     // TRIAL: C_N and -f of the rotation being fitted
};

struct DimerParams {
  double D;                    // separation (L)
  double c_t, s_t, s2_t, omc2_t;  // the trial rotation
  double rot_min;              // below this |rotational force| (force / L^2) the dimer translates without rotating
  double fmax2, maxstep, dt0, dtmax;  // the centre's FIRE, as in RelaxParams
  int periodic;                // 1: remove the translations only
};

// Intrinsic reaction coordinate (sgdml_b200_irc_rk4): the steepest-descent path from a first-order saddle in
// mass-weighted coordinates x_i = R_i / r_i, r_i = sqrt(s_i) with s the handle's inverse masses (the path's geometry
// depends on mass ratios only, so no other mass unit enters), followed downhill in both directions along the saddle's
// imaginary mode by classical RK4 on dx/ds = d(F(x)) (Schmidt, Gordon & Dupuis, JACS 107, 2585 (1985)).  The handle's
// n_rep = 2 n_pairs replicas: pair k is replicas 2k (forward, sigma = +1) and 2k + 1 (backward, sigma = -1), one branch
// each.  No rigid-mode projection: sGDML energies are exactly invariant under rotations and translations, so the
// mass-weighted gradient has no rigid part beyond rounding.  Every sum is block_sum's over the branch's 3N coordinates
// and every operation rounds as written (no fused multiply-add):
//   r_i = sqrt(s_i);  g_i = r_i F_i;  q = sum_i g_i g_i;  d_i = g_i / sqrt(q)  (d = 0 when q == 0: no division)
//
// k_irc_init: one CTA of MD_THREADS per pair, launched twice before the force evaluation of a call.
//   check (commit == 0): the caller's mode m (n_pairs, 3N), a Cartesian displacement, in the scratch rows V:
//     v_i = m_i / r_i;  q = sum_i v_i v_i;  v_i = v_i / sqrt(q);  bad[k] = !(q finite and q > 0)
//     Nothing of the handle changes; the driver reads every verdict back and commits only when no mode is bad.
//   commit (commit == 1), with R0, F0, E0 replica 2k's state (the saddle, as set_state stored it), for both branches b:
//     Rn_b = R0, Fn_b = F0 (point 0: the saddle);  R_b,i = R0_i + r_i ((sigma h) v_i)  (point 1);
//     IrcState {phase IRC_POINT, n_points 1, E_n E0};  path row 0 = (R0, E0), every other path entry NaN.
//   The driver then evaluates F and E of every replica (point 1).
//
// k_irc_step: one CTA of MD_THREADS per branch, its RelaxState z and IrcState y; R, F, E are the replica's state and
// F, E always belong to the positions in R.  Each launch, for a branch that has not ended (an ended one is frozen):
//   1. IRC_POINT (R is a new point n + 1):  if !(E < E_n) (a rise, or NaN): R, F, E = Rn, Fn, E_n (point n again),
//      fmax2 = atom_max2(Fn), end = 2.  Otherwise the point is recorded: Rn = R, Fn = F, path row n_points = (R, E),
//      n_points += 1, E_n = E, fmax2 = atom_max2(F), and end = 1 if fmax2 < fmax2_thr (ASE's criterion, as relax),
//      else 3 if n_points == max_points.  phase = IRC_K1.  z.n_steps = n_points and z.conv = end (k_relax_count and
//      k_relax_report read them).  advance == 0 stops here, and an ended branch stops here.
//   2. Stages (advance == 1 only), d the direction of the current F, K the branch's running sum (3N):
//      IRC_K1:  K_i = d_i;            R_i = Rn_i + r_i (hh d_i);    phase IRC_K2
//      IRC_K2:  K_i = K_i + 2 d_i;    R_i = Rn_i + r_i (hh d_i);    phase IRC_K3
//      IRC_K3:  K_i = K_i + 2 d_i;    R_i = Rn_i + r_i (h d_i);     phase IRC_K4
//      IRC_K4:  K_i = K_i + d_i;      R_i = Rn_i + r_i (h6 K_i);    phase IRC_POINT
//      so that R_n+1 = R_n + (h / 6) r (((k1 + 2 k2) + 2 k3) + k4), summed in that order.
// hh = h / 2 and h6 = h / 6 are computed once on the host, so the kernels and tests/irc_oracle.py use the same doubles.
// One point costs four force evaluations (one step-graph replay each); point 1 costs the one after the commit.
enum IrcPhase { IRC_POINT = 0, IRC_K1 = 1, IRC_K2 = 2, IRC_K3 = 3, IRC_K4 = 4 };

struct IrcState {    // per branch, written by k_irc_init's commit at the start of every call
  int phase;
  int end;           // 0: running;  1: max_a |F_a| < fmax;  2: energy rise;  3: max_points points
  int64_t n_points;  // points recorded, the saddle included
  double E_n;        // the energy of the newest point
};

struct IrcParams {
  double h, hh, h6;            // the step (mass-weighted unit), h / 2, h / 6
  double fmax2;                // fmax^2 (0: never ends by force)
  int64_t max_points;          // >= 2
  double *R_path, *E_path;     // (n_rep, max_points, 3N) / (n_rep, max_points), device pointers or null
};

}  // namespace sgdml
