// visual_pcg_emu.cpp — TEST INFRASTRUCTURE: the passes of ITERATIVE_SCHUR (global-lvba_b200/csrc/visual_pcg.h) run through the
// host policy, so that tests/test_visual_pcg_emu.py can compare the envelope product with a dense product and the whole
// conjugate-gradients solve with tests/visual_pcg_oracle.py without a GPU.  Never part of the product.
#include <vector>

#include "../../global-lvba_b200/csrc/visual_pcg.h"
#include "host_exec.h"

using namespace lvba;

namespace {
struct Work {
  HostExec::Buf<double> vec, minv, part, sd;
  HostExec::Buf<int> si;
  vpcg::Bufs bufs(int64_t n) {
    const int64_t n6 = 6 * n;
    vec.alloc((size_t)(4 * n6)); minv.alloc((size_t)(6 * n6)); part.alloc((size_t)vpcg::chunks(n6) + 1);
    sd.alloc(vpcg::kNDouble); si.alloc(vpcg::kNInt);
    double* v = vec.p;
    return vpcg::Bufs{v, v + n6, v + 2 * n6, v + 3 * n6, minv.p, vpcg::Ctl{si.p, sd.p, part.p}};
  }
};
}  // namespace

// y = (S + diag(dadd)) x by ProdF; the envelope: first, last [n], row_start [n + 1]
extern "C" void emu_pcg_product(int n, const int* first, const int* last, const long long* row_start, const double* S, const double* dadd,
                                const double* x, double* y) {
  HostExec ex;
  Work w;
  const vpcg::Bufs B = w.bufs(n);
  B.c.si[vpcg::kDone] = 0;
  const EnvView e{n, first, row_start, last, row_start[n]};
  ex.for_each(n, vpcg::ProdF{B.c, e, S, dadd, x, y});
}

// the whole solve of (S + diag(dadd)) x = b; out: x [6n], info[0] iterations, info[1] termination
extern "C" void emu_pcg_solve(int n, const int* first, const int* last, const long long* row_start, const double* S, const double* dadd,
                              const double* b, double eta, int min_iter, int max_iter, double* x, int* info) {
  HostExec ex;
  Work w;
  const vpcg::Bufs B = w.bufs(n);
  const EnvView e{n, first, row_start, last, row_start[n]};
  auto prod = [&](const double* in, double* out) { return ex.for_each(n, vpcg::ProdF{B.c, e, S, dadd, in, out}); };
  int si[vpcg::kNInt];
  int64_t d2h = 0;
  vpcg::solve(ex, e, S, dadd, b, x, B, vpcg::Params{eta, min_iter, max_iter}, prod, si, &d2h);
  info[0] = si[vpcg::kIter];
  info[1] = si[vpcg::kTerm];
}
