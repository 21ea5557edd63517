// What the device dynamics driver (csrc/md.cu) needs from the predictor: force evaluation of device-resident
// geometries through a workspace of its own, and the CUDA-graph capture both of them use.  The layout of
// sgdml_b200_model stays private to predict.cu.
#pragma once
#include "common.cuh"
#include "desc.cuh"

namespace sgdml {

// SGDML_B200_GRAPH=0 switches every CUDA-graph replay off: predict's small host-buffer batches and the dynamics step
// graph then run the same launches one by one
bool g_graph_enabled();

// Captures the work enqueue() queues on gs (not the legacy stream) into *exec; *n_kernels: the kernel launches counted
// while it was queued, which a replay of the graph counts again
template <class Enqueue>
int capture_graph(cudaStream_t gs, Enqueue&& enqueue, cudaGraphExec_t* exec, int* n_kernels) {
  auto launches = [] {
    int64_t n = 0;
    for (int k = 0; k < KID_COUNT; ++k) {
      int64_t ln = 0;
      sgdml_b200_profile_get(k, nullptr, nullptr, &ln);
      n += ln;
    }
    return n;
  };
  const int64_t before = launches();
  cudaGraph_t graph = nullptr;
  SG_CUDA(cudaStreamBeginCapture(gs, cudaStreamCaptureModeThreadLocal));
  const int rc = enqueue();
  cudaError_t e = cudaStreamEndCapture(gs, &graph);
  if (rc != 0) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  SG_CUDA(e);
  e = cudaGraphInstantiate(exec, graph, 0);
  cudaGraphDestroy(graph);
  SG_CUDA(e);
  *n_kernels = (int)(launches() - before);
  return 0;
}

// F(R) and E(R) of n_geo device-resident geometries in the model's cell, exactly as sgdml_b200_predict evaluates
// device-resident geometries, through a predictor workspace of the evaluator's own: predict calls never touch it, and
// it never touches theirs.
struct ForceEval;
int force_eval_create(sgdml_b200_model* m, int64_t n_geo, ForceEval** out);
// the caller has synchronised
void force_eval_destroy(ForceEval* fe);
// Sizes the workspace for the model's current settings (contraction slices, chunk size); call it before
// force_eval_run whenever the model may have changed.
int force_eval_prepare(ForceEval* fe);
// true when a graph that captured force_eval_run at the last force_eval_mark no longer matches: the workspace has been
// reallocated since, or the model's generation (use_ae, contraction slices) or cell has changed
bool force_eval_stale(const ForceEval* fe);
void force_eval_mark(ForceEval* fe);
// true when the model has a periodic cell
bool force_eval_periodic(const ForceEval* fe);
// R (n_geo, 3N) -> F (n_geo, 3N), E (n_geo), all device arrays; chunk by chunk when n_geo exceeds the predictor's chunk
int force_eval_run(ForceEval* fe, const double* R, double* F, double* E, cudaStream_t s);
// As force_eval_run, with geometry g in its own cell cells[g] (n_geo cells in DEVICE memory), also writing the virial
// W (n_geo, 9): bit for bit what sgdml_b200_predict_virial_cells returns for device-resident R in the same cells
int force_eval_run_cells(ForceEval* fe, const double* R, const Lattice* cells, double* F, double* E, double* W,
                         cudaStream_t s);

// The rule for a caller's periodic cell (sgdml_b200_predict_virial*): every entry of the cell and of its inverse finite,
// and the cell not singular.  0, or an argument error with the last-error message set.
int check_cell(const Lattice& l);

}  // namespace sgdml
