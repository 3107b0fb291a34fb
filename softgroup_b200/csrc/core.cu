// core.cu -- error reporting, device probe, per-device launch state, device-wide exclusive scan.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace sgb {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static Device g_devices[kMaxDevices];
static DeviceOnce g_devices_once;

int current_device(Device **out) {
  int dev;
  SGB_CUDA_CHECK(cudaGetDevice(&dev));
  SGB_REQUIRE(dev >= 0 && dev < kMaxDevices, SGB_ERR_RANGE, "device ordinal beyond 15");
  Device &d = g_devices[dev];
  int rc = once_per_device(g_devices_once, dev, [&] {
    d.ordinal = dev;
    SGB_CUDA_CHECK(cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev));
    SGB_CUDA_CHECK(cudaMalloc(&d.oflow, 4));
    SGB_CUDA_CHECK(cudaMemset(d.oflow, 0, 4));
    // the zero must land before any stream's kernel can raise the flag: the scan streams do not wait for the default one
    SGB_CUDA_CHECK(cudaStreamSynchronize(0));
    return SGB_OK;
  });
  if (rc) return rc;
  *out = &d;
  return SGB_OK;
}

constexpr int kScanThreads = 512;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

size_t scan_temp_elems(size_t n) {
  size_t tot = 0;
  while (n > 1) {
    size_t nb = (n + kScanTile - 1) / kScanTile;
    tot += align_up(nb * 8, 256) / 8;
    n = nb;
    if (nb == 1) break;
  }
  return tot + 64;
}

template <typename T>
__global__ void __launch_bounds__(kScanThreads) scan_tile_kernel(const T *__restrict__ in, T *__restrict__ out,
                                                                 size_t n, T *__restrict__ block_sums,
                                                                 T *__restrict__ total) {
  __shared__ T warp_tot[kScanThreads / 32];
  size_t base = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanItems;
  T v[kScanItems];
  T sum = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; k++) {
    v[k] = (base + k < n) ? in[base + k] : (T)0;
    sum += v[k];
  }
  // inclusive scan of per-thread sums across the block
  T inc = sum;
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    T t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  if (w == 0) {
    T t = (lane < kScanThreads / 32) ? warp_tot[lane] : (T)0;
    T ti = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      T u = __shfl_up_sync(0xffffffffu, ti, o);
      if (lane >= o) ti += u;
    }
    if (lane < kScanThreads / 32) warp_tot[lane] = ti - t;  // exclusive warp offsets
    if (lane == kScanThreads / 32 - 1) {
      if (block_sums) block_sums[blockIdx.x] = ti;
      if (total && gridDim.x == 1) *total = ti;
    }
  }
  __syncthreads();
  T run = warp_tot[w] + inc - sum;
#pragma unroll
  for (int k = 0; k < kScanItems; k++) {
    if (base + k < n) out[base + k] = run;
    run += v[k];
  }
}

template <typename T>
__global__ void scan_add_kernel(T *__restrict__ out, size_t n, const T *__restrict__ block_offsets) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] += block_offsets[i / kScanTile];
}

template <typename T>
static int exclusive_scan_impl(const T *in, T *out, size_t n, T *total, T *temp, cudaStream_t st) {
  if (n == 0) {
    if (total) SGB_CUDA_CHECK(cudaMemsetAsync(total, 0, sizeof(T), st));
    return SGB_OK;
  }
  size_t nb = (n + kScanTile - 1) / kScanTile;
  if (nb == 1) {
    scan_tile_kernel<T><<<1, kScanThreads, 0, st>>>(in, out, n, nullptr, total);
    SGB_LAUNCH_CHECK();
    return SGB_OK;
  }
  T *sums = temp;
  T *next_temp = temp + align_up(nb * 8, 256) / 8;
  scan_tile_kernel<T><<<(unsigned)nb, kScanThreads, 0, st>>>(in, out, n, sums, nullptr);
  SGB_LAUNCH_CHECK();
  int rc = exclusive_scan_impl<T>(sums, sums, nb, total, next_temp, st);
  if (rc) return rc;
  scan_add_kernel<T><<<div_up((long long)n, 256), 256, 0, st>>>(out, n, sums);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int exclusive_scan_i32(const int32_t *in, int32_t *out, size_t n, int32_t *total, int32_t *temp, cudaStream_t st) {
  return exclusive_scan_impl<int32_t>(in, out, n, total, temp, st);
}
int exclusive_scan_i64(const long long *in, long long *out, size_t n, long long *total, long long *temp,
                       cudaStream_t st) {
  return exclusive_scan_impl<long long>(in, out, n, total, temp, st);
}

}  // namespace sgb

extern "C" {

const char *sgb_last_error(void) { return sgb::g_err; }

int sgb_abi_version(void) { return 1; }

long long sgb_launch_count(void) { return sgb::g_launches.load(); }

int sgb_device_available(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n > 0 ? 1 : 0;
}

}
