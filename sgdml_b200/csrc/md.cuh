// Molecular dynamics on the device (sgdml_b200_md_*): the BAOAB integrator step and its counter-based noise.
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

}  // namespace sgdml
