// Molecular dynamics on the device (sgdml_b200_md_*, sgdml_b200_pimd_*): the BAOAB integrator step, its ring-polymer
// form, and their counter-based noise.
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
};

// One step for every replica (grid: one CTA of MD_THREADS per replica).  With the handle's step counter at n:
//   if n != run_start:  v += h (F s)        second half-kick of step n - 1 (F is F(r) of the positions in R)
//                       frame (n - run_start) / stride - 1 when that is whole: R, full-step V, E_pot, E_kin
//   if advance:         B, A, O (noise of step n), A; R and V hold the new positions and half-step velocities,
//                       and the counter becomes n + 1
// advance == 0 only completes the last step of a run.  s, sigma: (3N) inverse mass and noise scale per coordinate.
constexpr int MD_THREADS = 128;
int launch_md_step(const MdParams* P, const double* s, const double* sigma, double* R, double* V, const double* F,
                   const double* E, uint64_t* step, int64_t n_rep, int dimi, int advance, cudaStream_t st);

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

// One PILE-L step for every ring polymer (grid: one CTA of MD_THREADS per polymer), the counterpart of
// launch_md_step: the pending second half-kick and the frame (per bead R, full-step V, E_pot, E_kin; per polymer
// K_prim, K_cv), then, if advance, B, the transform to normal modes, A, O, A, the transform back.  tab: C (nb x nb,
// C[j nb + k]) followed by the mode tables cos(w_k h), sin(w_k h) / w_k, -w_k sin(w_k h), c1_k (nb each);
// sigma (nb, 3N) per mode and coordinate; s (3N) inverse masses.
int launch_pimd_step(const PimdParams* P, const double* tab, const double* s, const double* sigma, double* R, double* V,
                     const double* F, const double* E, uint64_t* step, int64_t n_poly, int dimi, int nb, int advance,
                     cudaStream_t st);

}  // namespace sgdml
