// exec.cuh — the CUDA execution policy of the item passes (voxel_pipeline.h, lidar_tiles.h and the other *_pipeline.h):
// one grid-stride kernel per pass, cub for the stable radix sorts / scans / min-max.  The CPU tests run the same passes
// through the host policy of tests/emu/host_exec.h.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include "runtime.cuh"

namespace lvba {

// Each pass is a functor over an index range.  Grid: enough 256-thread CTAs to cover n, capped at 16 per SM on the
// 132 SMs of an H100 SXM (grid-stride beyond that); the point passes are HBM streams, the segment / node passes are
// latency-bound gathers that want many warps in flight.
template <class F>
__global__ void __launch_bounds__(256) vox_for_each_kernel(int64_t n, F f) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) f(i);
}

struct CudaExec {
  template <class T>
  using Buf = DevBuf<T>;
  cudaStream_t stream = nullptr;
  int64_t launches = 0;            // launches of this library's own kernels (cub's are library calls, not counted)
  DevBuf<uint8_t> temp;
  DevBuf<int32_t> red;

  template <class F>
  int for_each(int64_t n, const F& f) {
    if (n <= 0) return LVBA_OK;
    const int64_t want = (n + 255) / 256;
    const int grid = (int)std::min<int64_t>(want, kNumSMs * 16);
    vox_for_each_kernel<F><<<grid, 256, 0, stream>>>(n, f);
    LVBA_CUDA(cudaGetLastError());
    ++launches;
    return LVBA_OK;
  }
  template <class T>
  int fill_zero(T* p, size_t n) {
    if (n) LVBA_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), stream));
    return LVBA_OK;
  }
  template <class T>
  int put(T* dev, const T* host, size_t n) {       // host -> device; the host range must stay alive until the next sync()
    if (n) LVBA_CUDA(cudaMemcpyAsync(dev, host, n * sizeof(T), cudaMemcpyHostToDevice, stream));
    return LVBA_OK;
  }
  template <class T>
  int fetch(T* host, const T* dev, size_t n) {
    if (n) LVBA_CUDA(cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, stream));
    LVBA_CUDA(cudaStreamSynchronize(stream));
    return LVBA_OK;
  }
  int reserve_temp(size_t bytes) {
    if (bytes == 0) bytes = 1;                       // cub reads a null temp pointer as a size query
    if (bytes > temp.n) LVBA_TRY(temp.alloc(bytes));
    return LVBA_OK;
  }
  int min_max(const int32_t* p, int64_t n, int32_t* mn, int32_t* mx) {
    if (red.n < 2) LVBA_TRY(red.alloc(2));
    size_t b0 = 0, b1 = 0;
    LVBA_CUDA(cub::DeviceReduce::Min(nullptr, b0, p, red.p, n, stream));
    LVBA_CUDA(cub::DeviceReduce::Max(nullptr, b1, p, red.p + 1, n, stream));
    LVBA_TRY(reserve_temp(std::max(b0, b1)));
    size_t tb = temp.n;
    LVBA_CUDA(cub::DeviceReduce::Min(temp.p, tb, p, red.p, n, stream));
    tb = temp.n;
    LVBA_CUDA(cub::DeviceReduce::Max(temp.p, tb, p, red.p + 1, n, stream));
    int32_t h[2];
    LVBA_TRY(fetch(h, red.p, 2));
    *mn = h[0]; *mx = h[1];
    return LVBA_OK;
  }
  // stable LSD radix sort on key bits [0, end_bit)
  int sort_pairs(const uint64_t* kin, uint64_t* kout, const uint32_t* vin, uint32_t* vout, int64_t n, int end_bit) {
    if (n <= 0) return LVBA_OK;
    size_t bytes = 0;
    LVBA_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin, kout, vin, vout, n, 0, end_bit, stream));
    LVBA_TRY(reserve_temp(bytes));
    bytes = temp.n;
    LVBA_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, bytes, kin, kout, vin, vout, n, 0, end_bit, stream));
    return LVBA_OK;
  }
  template <class T>
  int exclusive_scan(const T* in, T* out, int64_t n) {
    if (n <= 0) return LVBA_OK;
    size_t bytes = 0;
    LVBA_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, stream));
    LVBA_TRY(reserve_temp(bytes));
    bytes = temp.n;
    LVBA_CUDA(cub::DeviceScan::ExclusiveSum(temp.p, bytes, in, out, n, stream));
    return LVBA_OK;
  }
  int sync() {
    LVBA_CUDA(cudaStreamSynchronize(stream));
    return LVBA_OK;
  }
};

}  // namespace lvba
