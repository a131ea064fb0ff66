// vec3.h — 3-vector helpers compiled for the device and, for the CPU tests of tests/emu/, for the host.
#pragma once

#if defined(__CUDACC__)
#define LVBA_HD __host__ __device__ __forceinline__
#else
#define LVBA_HD inline
#endif
// #pragma unroll for the device pass only (host compilers warn about it)
#if defined(__CUDA_ARCH__)
#define LVBA_UNROLL _Pragma("unroll")
#else
#define LVBA_UNROLL
#endif

namespace lvba {

LVBA_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
LVBA_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
// hat(v): reference include/BALM/tools.hpp:105-112
LVBA_HD void hat3(const double* v, double* H) {
  H[0] = 0.0;   H[1] = -v[2]; H[2] = v[1];
  H[3] = v[2];  H[4] = 0.0;   H[5] = -v[0];
  H[6] = -v[1]; H[7] = v[0];  H[8] = 0.0;
}

}  // namespace lvba
