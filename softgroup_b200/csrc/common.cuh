// common.cuh -- shared device/host helpers for libsgb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <mutex>

#include "../../include/sgb200.h"

namespace sgb {

void set_error(const char *fmt, ...);
void count_launch();  // bumps the process-wide kernel-launch counter (sgb_launch_count)

#define SGB_CUDA_CHECK(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      sgb::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return SGB_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define SGB_LAUNCH_CHECK()               \
  do {                                   \
    sgb::count_launch();                 \
    SGB_CUDA_CHECK(cudaGetLastError()); \
  } while (0)

#define SGB_REQUIRE(cond, code, msg)                                 \
  do {                                                               \
    if (!(cond)) {                                                   \
      sgb::set_error("%s:%d %s (%s)", __FILE__, __LINE__, msg, #cond); \
      return (code);                                                 \
    }                                                                \
  } while (0)

// Per-device launch state, built on a device's first use, once, thread-safely. Grids that cover the machine are sized
// from `sms`.
constexpr int kMaxDevices = 16;

struct Device {
  int ordinal;
  int sms;     // multiprocessors
  int *oflow;  // flag raised by the packing code when a value leaves the fp16 range (sgb_spconv_overflow)
};

// The current device's record (errors through set_error). SGB_CURRENT_DEVICE(d) declares `Device *d` or returns the error.
int current_device(Device **d);
#define SGB_CURRENT_DEVICE(d) \
  sgb::Device *d;             \
  if (const int _rc = sgb::current_device(&d)) return _rc

// One-time set-up of a module, per device: init() runs until it first returns SGB_OK, then never again. A failed
// init has reported its error on the calling thread, and the next call tries again.
struct DeviceOnce { std::atomic<bool> done[kMaxDevices] = {}; std::mutex m; };

template <typename F>
int once_per_device(DeviceOnce &once, int dev, F &&init) {
  if (once.done[dev].load(std::memory_order_acquire)) return SGB_OK;
  std::lock_guard<std::mutex> lock(once.m);
  if (once.done[dev].load(std::memory_order_relaxed)) return SGB_OK;
  const int rc = init();
  if (rc == SGB_OK) once.done[dev].store(true, std::memory_order_release);
  return rc;
}

static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Bump allocator over the caller-provided workspace.
struct Arena {
  char *base;
  size_t size, off;
  Arena(void *p, size_t n) : base((char *)p), size(n), off(0) {}
  template <typename T>
  T *take(size_t count) {
    size_t bytes = align_up(count * sizeof(T));
    if (off + bytes > size) return nullptr;
    T *r = (T *)(base + off);
    off += bytes;
    return r;
  }
};

static inline size_t pow2_at_least(size_t x) {
  size_t c = 1;
  while (c < x) c <<= 1;
  return c;
}

// ---------------------------------------------------------------------------------------------
// 64-bit key hash table (open addressing, linear probing). EMPTY = all ones.
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

__device__ __forceinline__ uint32_t hash64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (uint32_t)k;
}

// Insert-or-find; returns the slot. cap_mask = capacity-1 (capacity is a power of two >= 2*#keys). key must not be
// kEmptyKey: that key "finds" the first empty slot without claiming it.
__device__ __forceinline__ uint32_t hash_insert(unsigned long long *keys, uint32_t cap_mask, unsigned long long key) {
  uint32_t s = hash64(key) & cap_mask;
  while (true) {
    unsigned long long cur = keys[s];
    if (cur == key) return s;
    if (cur == kEmptyKey) {
      unsigned long long old = atomicCAS(&keys[s], kEmptyKey, key);
      if (old == kEmptyKey || old == key) return s;
    }
    s = (s + 1) & cap_mask;
  }
}

// Find; returns slot or 0xFFFFFFFF.
__device__ __forceinline__ uint32_t hash_find(const unsigned long long *__restrict__ keys, uint32_t cap_mask,
                                              unsigned long long key) {
  uint32_t s = hash64(key) & cap_mask;
  while (true) {
    unsigned long long cur = __ldg(&keys[s]);
    if (cur == key) return s;
    if (cur == kEmptyKey) return 0xFFFFFFFFu;
    s = (s + 1) & cap_mask;
  }
}

// ---------------------------------------------------------------------------------------------
// Device-wide exclusive scan (int32 / int64), multi-level. out may alias in.
// total (device scalar, may be null) receives the grand total.
// temp must hold scan_temp_elems(n) elements of T.
// ---------------------------------------------------------------------------------------------
size_t scan_temp_elems(size_t n);
int exclusive_scan_i32(const int32_t *in, int32_t *out, size_t n, int32_t *total, int32_t *temp, cudaStream_t st);
int exclusive_scan_i64(const long long *in, long long *out, size_t n, long long *total, long long *temp,
                       cudaStream_t st);

// warp helpers
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace sgb
