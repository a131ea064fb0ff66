// env_types.h — plain C++ views / job descriptors of the block-envelope solvers (no CUDA), shared by the device kernels
// (envelope.cuh, factor_la.cuh, nd_kernels.cuh), the host plan (nd_plan.h) and the CPU checks under tests/emu/.
#pragma once
#include <stdint.h>

namespace lvba {

struct EnvView {
  int n;                       // block rows
  const int* first;            // [n]
  const long long* row_start;  // [n+1] in blocks
  const int* last;             // [n]   last[k] = max row i with first[i] <= k
  long long nblocks;
};

// One factorisation instance.  The twisted solve (runtime.cuh) runs two at once (gridDim.x = 2): the top half of
// the pose system in natural order and the bottom half in REVERSED order, each on its own SM; both stop at the
// separator (n_stop < n) and dump their Schur-updated trailing window + forward-substituted rhs.  The substructured
// solve (nd_solver.cuh) runs one per chunk interior / per separator.
struct FactorJob {
  EnvView e;
  double* L;       // in: matrix (H + damping) in envelope layout; out: L_ik below the pivots
  double* dinv;    // out: D_k^-1 of every pivot block (36 doubles, full symmetric)
  double* z;       // in: rhs ; out: forward-substituted rhs of the pivots
  int n_stop;      // number of pivots to eliminate (== e.n for a complete factorisation)
  double* wdump;   // [bs*bs*36] trailing window at n_stop, block (i,j) at ((i-n_stop)*bs + (j-n_stop))*36, bs = e.n - n_stop
  double* zdump;   // [bs*6]
  int* status;     // set to 1 when a pivot block is singular / non-finite
  // Optional progress counter for a consumer that runs BESIDE this factorisation (the spike kernel, nd_kernels.cuh): the number of
  // leading columns of L that are final in global memory, published with release semantics every few pivots (values below n_stop) and once more — as
  // the very last global write of the CTA — with the value n_stop.  nullptr: nothing is published.
  int* progress = nullptr;
};
// Jobs live in device memory (one per CTA): two for the twisted solve, one per window for the batched window BA.

struct BacksolveJob {
  EnvView e;
  const double* L;
  double* x;        // in: D^-1 z for the pivots (rows < n_given) and the FINAL solution for rows >= n_given ; out: solution
  int n_given;      // rows >= n_given are given (separator of the twisted solve); == e.n for a plain solve
};

}  // namespace lvba
