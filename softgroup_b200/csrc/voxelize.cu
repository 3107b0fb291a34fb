// voxelize.cu -- point->voxel hashing (voxelize_idx) and voxel feature pooling (voxelize_fp/bp).
//
// Replaces softgroup/ops/src/voxelize/voxelize.cpp:11-165 (single-thread CPU dense_hash_map) and
// voxelize.cu:9-62 of the reference. Semantics kept bit-exact:
//   voxel id = rank of the voxel's FIRST point in point order; rows = ascending point indices.
// GPU algorithm: 64-bit packed keys -> open-addressing hash (atomicCAS) -> atomicMin first point per
// slot -> flags/scan over points (rank of first occurrences) -> map fill + per-row ordering.
#include <algorithm>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace sgb {

// key: [batch:16][x+32768:16][y+32768:16][z+32768:16]
__device__ __forceinline__ bool pack_key(const long long *c, int ncol, unsigned long long &key) {
  long long b = 0, x, y, z;
  if (ncol == 4) { b = c[0]; x = c[1]; y = c[2]; z = c[3]; }
  else { x = c[0]; y = c[1]; z = c[2]; }
  // the reference narrows coordinates to int32 (datatype.h:11); identical for in-range values
  bool ok = (b >= 0 && b < 65536) && (x >= -32768 && x < 32768) && (y >= -32768 && y < 32768) &&
            (z >= -32768 && z < 32768);
  key = ((unsigned long long)(b & 0xFFFF) << 48) | ((unsigned long long)((x + 32768) & 0xFFFF) << 32) |
        ((unsigned long long)((y + 32768) & 0xFFFF) << 16) | (unsigned long long)((z + 32768) & 0xFFFF);
  return ok;
}

// The point (65535, 32767, 32767, 32767) packs to kEmptyKey, which the table cannot hold: its points skip the table
// and share the reserved slot `cap` of the per-slot arrays.
struct VoxWs {
  unsigned long long *keys;  // [cap]
  int32_t *first;            // [cap + 1] min point index of the slot
  int32_t *last;             // [cap + 1] max point index
  int32_t *cnt;              // [cap + 1]
  int32_t *vid;              // [cap + 1] voxel id of slot
  int32_t *slot_of;          // [N] slot of the point, -1 for a point outside the key range
  int32_t *rank;             // [N] flags -> exclusive scan
  int32_t *fill;             // [N] (>= M) per-voxel fill cursor
  int32_t *scalars;          // [8]: 0 = M, 1 = maxActive, 2 = range error flag
  int32_t *scan_tmp;
  uint32_t cap;
};

static size_t vox_cap(int N) { return pow2_at_least((size_t)std::max(N, 1) * 2); }

static bool vox_carve(void *ws, size_t bytes, int N, VoxWs &w) {
  Arena a(ws, bytes);
  w.cap = (uint32_t)vox_cap(N);
  w.scalars = a.take<int32_t>(64);
  w.keys = a.take<unsigned long long>(w.cap);
  w.first = a.take<int32_t>((size_t)w.cap + 1);
  w.last = a.take<int32_t>((size_t)w.cap + 1);
  w.cnt = a.take<int32_t>((size_t)w.cap + 1);
  w.vid = a.take<int32_t>((size_t)w.cap + 1);
  w.slot_of = a.take<int32_t>((size_t)N + 1);
  w.rank = a.take<int32_t>((size_t)N + 1);
  w.fill = a.take<int32_t>((size_t)N + 1);
  w.scan_tmp = a.take<int32_t>(scan_temp_elems((size_t)N + 1));
  return w.scan_tmp != nullptr;
}

__global__ void vox_insert_kernel(const long long *__restrict__ coords, int N, int ncol, VoxWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  unsigned long long key;
  if (!pack_key(coords + (size_t)i * ncol, ncol, key)) { w.scalars[2] = 1; w.slot_of[i] = -1; return; }
  uint32_t s = (key == kEmptyKey) ? w.cap : hash_insert(w.keys, w.cap - 1, key);
  w.slot_of[i] = (int32_t)s;
  atomicMin(&w.first[s], i);
  atomicMax(&w.last[s], i);
  atomicAdd(&w.cnt[s], 1);
}

__global__ void vox_flag_kernel(int N, VoxWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int s = w.slot_of[i];
  w.rank[i] = (s >= 0 && w.first[s] == i) ? 1 : 0;
}

// after the scan: rank[i] = voxel id for first-occurrence points
__global__ void vox_assign_kernel(int N, int mode, VoxWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int s = w.slot_of[i];
  if (s >= 0 && w.first[s] == i) {
    w.vid[s] = w.rank[i];
    int c = (mode == 3 || mode == 4) ? w.cnt[s] : 1;
    // filtered atomic: only rows that beat the (possibly stale) running maximum touch the counter
    if (c > *(volatile int32_t *)&w.scalars[1]) atomicMax(&w.scalars[1], c);
  }
}

__global__ void vox_inputmap_kernel(int N, int32_t *__restrict__ input_map, VoxWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int s = w.slot_of[i];
  input_map[i] = (s >= 0) ? w.vid[s] : -1;
}

__global__ void vox_fill_kernel(const long long *__restrict__ coords, int N, int ncol, int mode, int W,
                                long long *__restrict__ out_coords, int32_t *__restrict__ out_map, VoxWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int s = w.slot_of[i];
  int v = w.vid[s];
  bool is_first = (w.first[s] == i);
  if (mode == 3 || mode == 4) {
    int pos = atomicAdd(&w.fill[v], 1);
    out_map[(size_t)v * W + 1 + pos] = i;
    if (is_first) out_map[(size_t)v * W] = w.cnt[s];
  } else if (is_first) {
    out_map[(size_t)v * W] = 1;
    out_map[(size_t)v * W + 1] = (mode == 2) ? w.last[s] : i;  // mode 1 -> front(), mode 2 -> back() (voxelize.cpp:139-149)
  }
  if (is_first) {
    // voxelize_outputmap (voxelize.cpp:41-57) copies the coords of rule[1], i.e. of the first listed point
    int src = (mode == 2) ? w.last[s] : i;
    for (int j = 0; j < ncol; j++) out_coords[(size_t)v * ncol + j] = coords[(size_t)src * ncol + j];
  }
}

// Order each row ascending. Rows are tiny (mean ~1.2 points/voxel at 2 cm): insertion sort per thread;
// rows longer than 24 entries (cluster re-voxelisation) are rank-sorted by the whole warp.
__global__ void vox_sort_rows_kernel(int M, int W, int32_t *__restrict__ out_map) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  int row0 = warp * 32;
  if (row0 >= M) return;
  int row = row0 + lane;
  int c = (row < M) ? out_map[(size_t)row * W] : 0;
  bool long_row = c > 24;
  if (!long_row && c > 1) {
    int32_t *r = out_map + (size_t)row * W + 1;
    for (int a = 1; a < c; a++) {
      int x = r[a];
      int b = a - 1;
      while (b >= 0 && r[b] > x) { r[b + 1] = r[b]; b--; }
      r[b + 1] = x;
    }
  }
  __syncwarp();
  unsigned long_mask = __ballot_sync(0xffffffffu, long_row);
  while (long_mask) {
    int l = __ffs(long_mask) - 1;
    long_mask &= long_mask - 1;
    int cc = __shfl_sync(0xffffffffu, c, l);
    int32_t *r = out_map + (size_t)(row0 + l) * W + 1;
    int nchunk = (cc + 31) >> 5;
    if (nchunk <= 32) {
      // rank(e) = #entries smaller than e (entries are distinct point indices); compute all ranks, then permute
      int vals[32], ranks[32];
      for (int ch = 0; ch < nchunk; ch++) {
        int e = ch * 32 + lane;
        int x = (e < cc) ? r[e] : 0x7fffffff;
        int rank = 0;
        for (int k = 0; k < cc; k++) rank += (r[k] < x);
        vals[ch] = x;
        ranks[ch] = rank;
      }
      __syncwarp();
      for (int ch = 0; ch < nchunk; ch++)
        if (ch * 32 + lane < cc) r[ranks[ch]] = vals[ch];
    } else if (lane == 0) {
      // > 1024 points in one voxel: single-lane shell sort (never seen on the reference configs)
      for (int gap = cc / 2; gap > 0; gap /= 2)
        for (int a = gap; a < cc; a++) {
          int x = r[a];
          int b = a;
          while (b >= gap && r[b - gap] > x) { r[b] = r[b - gap]; b -= gap; }
          r[b] = x;
        }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// voxelize_fp / bp
// ---------------------------------------------------------------------------------------------
// One thread per (row, channel) keeps the reference's sequential order ((0 + m*x0) + m*x1) + ...
// (voxelize.cu:13-24: the atomicAdd of one (row,plane) is issued by a single thread, in list order).
__global__ void voxelize_fp_kernel(const float *__restrict__ feats, float *__restrict__ out,
                                   const int32_t *__restrict__ rules, int M, int W, int C, int average) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)M * C) return;
  int row = (int)(t / C), c = (int)(t % C);
  const int32_t *r = rules + (size_t)row * W;
  int n = r[0];
  float m = (average && n > 0) ? __fdiv_rn(1.0f, (float)n) : 1.0f;
  float acc = 0.f;
  for (int i = 1; i <= n; i++) acc = __fadd_rn(acc, __fmul_rn(m, __ldg(&feats[(size_t)r[i] * C + c])));
  out[(size_t)row * C + c] = acc;
}

__global__ void voxelize_bp_kernel(const float *__restrict__ d_out, float *__restrict__ d_feats,
                                   const int32_t *__restrict__ rules, int M, int W, int C, int average) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)M * C) return;
  int row = (int)(t / C), c = (int)(t % C);
  const int32_t *r = rules + (size_t)row * W;
  int n = r[0];
  float m = (average && n > 0) ? __fdiv_rn(1.0f, (float)n) : 1.0f;
  float g = __fmul_rn(m, d_out[(size_t)row * C + c]);
  // every point belongs to exactly one voxel row -> no write conflicts; += keeps the reference's accumulate
  for (int i = 1; i <= n; i++) d_feats[(size_t)r[i] * C + c] += g;
}

__global__ void bn_relu_kernel(const float *__restrict__ x, int xs, const float *__restrict__ scale,
                               const float *__restrict__ shift, int relu, float *__restrict__ y, int ys, int M, int C) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)M * C) return;
  int row = (int)(t / C), c = (int)(t % C);
  float v = fmaf(x[(size_t)row * xs + c], scale[c], shift[c]);
  if (relu) v = fmaxf(v, 0.f);
  y[(size_t)row * ys + c] = v;
}

__global__ void gather_rows_kernel(const float *__restrict__ in, const int32_t *__restrict__ index,
                                   float *__restrict__ out, int N, int C4) {
  // one thread per float4 of the output
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * C4) return;
  int row = (int)(t / C4), q = (int)(t % C4);
  int src = __ldg(&index[row]);
  reinterpret_cast<float4 *>(out)[(size_t)row * C4 + q] = __ldg(&reinterpret_cast<const float4 *>(in)[(size_t)src * C4 + q]);
}
__global__ void gather_rows_scalar_kernel(const float *__restrict__ in, const int32_t *__restrict__ index,
                                          float *__restrict__ out, int N, int C) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * C) return;
  int row = (int)(t / C), c = (int)(t % C);
  out[(size_t)row * C + c] = __ldg(&in[(size_t)__ldg(&index[row]) * C + c]);
}

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_voxelize_idx_workspace_bytes(int N) {
  if (N < 0) N = 0;
  size_t cap = vox_cap(N);
  size_t b = 0;
  b += align_up(64 * 4);
  b += align_up(cap * 8);
  b += 4 * align_up((cap + 1) * 4);
  b += 3 * align_up(((size_t)N + 1) * 4);
  b += align_up(scan_temp_elems((size_t)N + 1) * 4);
  return b + 1024;
}

int sgb_voxelize_idx_count(const int64_t *d_coords, int N, int ncol, int mode, int32_t *d_input_map, void *d_ws,
                           size_t ws_bytes, int *h_M, int *h_maxActive, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(N >= 0 && (ncol == 3 || ncol == 4) && mode >= 0 && mode <= 4, SGB_ERR_ARG, "voxelize_idx arguments");
  SGB_REQUIRE(h_M && h_maxActive, SGB_ERR_ARG, "null output");
  if (N == 0) { *h_M = 0; *h_maxActive = 1; return SGB_OK; }
  SGB_REQUIRE(d_coords && d_input_map && d_ws, SGB_ERR_ARG, "null pointer");
  VoxWs w;
  SGB_REQUIRE(vox_carve(d_ws, ws_bytes, N, w), SGB_ERR_WORKSPACE, "voxelize_idx workspace too small");
  SGB_CUDA_CHECK(cudaMemsetAsync(w.keys, 0xFF, (size_t)w.cap * 8, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.first, 0x7F, ((size_t)w.cap + 1) * 4, st));  // 0x7F7F7F7F > any index
  SGB_CUDA_CHECK(cudaMemsetAsync(w.last, 0xFF, ((size_t)w.cap + 1) * 4, st));   // -1
  SGB_CUDA_CHECK(cudaMemsetAsync(w.cnt, 0, ((size_t)w.cap + 1) * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.scalars, 0, 64 * 4, st));
  int nb = div_up(N, 256);
  vox_insert_kernel<<<nb, 256, 0, st>>>((const long long *)d_coords, N, ncol, w);
  SGB_LAUNCH_CHECK();
  vox_flag_kernel<<<nb, 256, 0, st>>>(N, w);
  SGB_LAUNCH_CHECK();
  int rc = exclusive_scan_i32(w.rank, w.rank, (size_t)N, &w.scalars[0], w.scan_tmp, st);
  if (rc) return rc;
  vox_assign_kernel<<<nb, 256, 0, st>>>(N, mode, w);
  SGB_LAUNCH_CHECK();
  vox_inputmap_kernel<<<nb, 256, 0, st>>>(N, d_input_map, w);
  SGB_LAUNCH_CHECK();
  int h[4];
  SGB_CUDA_CHECK(cudaMemcpyAsync(h, w.scalars, sizeof(h), cudaMemcpyDeviceToHost, st));
  SGB_CUDA_CHECK(cudaStreamSynchronize(st));
  SGB_REQUIRE(h[2] == 0, SGB_ERR_RANGE, "voxelize_idx: coordinate outside the packed key range (batch<65536, |xyz|<32768)");
  *h_M = h[0];
  *h_maxActive = std::max(h[1], 1);
  return SGB_OK;
}

int sgb_voxelize_idx_fill(const int64_t *d_coords, int N, int ncol, int mode, int M, int maxActive,
                          int64_t *d_output_coords, int32_t *d_output_map, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0 || M == 0) return SGB_OK;
  SGB_REQUIRE(d_coords && d_output_coords && d_output_map && d_ws, SGB_ERR_ARG, "null pointer");
  VoxWs w;
  SGB_REQUIRE(vox_carve(d_ws, ws_bytes, N, w), SGB_ERR_WORKSPACE, "voxelize_idx workspace too small");
  int W = maxActive + 1;
  SGB_CUDA_CHECK(cudaMemsetAsync(d_output_map, 0, (size_t)M * W * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.fill, 0, ((size_t)N + 1) * 4, st));
  vox_fill_kernel<<<div_up(N, 256), 256, 0, st>>>((const long long *)d_coords, N, ncol, mode, W,
                                                 (long long *)d_output_coords, d_output_map, w);
  SGB_LAUNCH_CHECK();
  if ((mode == 3 || mode == 4) && maxActive > 1) {
    vox_sort_rows_kernel<<<div_up(M, 256), 256, 0, st>>>(M, W, d_output_map);
    SGB_LAUNCH_CHECK();
  }
  return SGB_OK;
}

// ---- CPU path (DataLoader workers; no CUDA calls) ---------------------------------------------
struct VoxCpu {
  int N, ncol, mode, M, maxActive;
  std::vector<int32_t> first, last, count, imap;
};
struct Key4 {
  int32_t k[4];
  bool operator==(const Key4 &o) const { return k[0] == o.k[0] && k[1] == o.k[1] && k[2] == o.k[2] && k[3] == o.k[3]; }
};
struct Key4Hash {
  size_t operator()(const Key4 &p) const {
    uint64_t h = 1469598103934665603ull;
    for (int j = 0; j < 4; j++) { h ^= (uint32_t)p.k[j]; h *= 1099511628211ull; }
    return (size_t)(h ^ (h >> 29));
  }
};

void *sgb_voxelize_idx_cpu_begin(const int64_t *h_coords, int N, int ncol, int mode, int32_t *h_input_map, int *h_M,
                                 int *h_maxActive) {
  if (N < 0 || (ncol != 3 && ncol != 4) || mode < 0 || mode > 4 || !h_M || !h_maxActive) {
    set_error("sgb_voxelize_idx_cpu_begin: bad arguments");
    return nullptr;
  }
  VoxCpu *h = new VoxCpu();
  h->N = N; h->ncol = ncol; h->mode = mode;
  std::unordered_map<Key4, int32_t, Key4Hash> mp;
  mp.reserve((size_t)N * 2 + 16);
  h->imap.resize(N);
  for (int i = 0; i < N; i++) {
    Key4 k;
    const int64_t *c = h_coords + (size_t)i * ncol;
    if (ncol == 4) { k.k[0] = (int32_t)c[0]; k.k[1] = (int32_t)c[1]; k.k[2] = (int32_t)c[2]; k.k[3] = (int32_t)c[3]; }
    else { k.k[0] = 0; k.k[1] = (int32_t)c[0]; k.k[2] = (int32_t)c[1]; k.k[3] = (int32_t)c[2]; }
    auto it = mp.find(k);
    int v;
    if (it == mp.end()) {
      v = (int)h->first.size();
      mp.emplace(k, v);
      h->first.push_back(i); h->last.push_back(i); h->count.push_back(0);
    } else v = it->second;
    h->count[v]++; h->last[v] = i; h->imap[i] = v;
    h_input_map[i] = v;
  }
  h->M = (int)h->first.size();
  int mx = 1;
  if (mode == 3 || mode == 4) for (int c : h->count) mx = std::max(mx, c);
  h->maxActive = mx;
  *h_M = h->M; *h_maxActive = mx;
  return h;
}

int sgb_voxelize_idx_cpu_finish(void *handle, const int64_t *h_coords, int64_t *h_output_coords,
                                int32_t *h_output_map) {
  VoxCpu *h = (VoxCpu *)handle;
  SGB_REQUIRE(h, SGB_ERR_ARG, "null handle");
  int W = h->maxActive + 1;
  std::fill(h_output_map, h_output_map + (size_t)h->M * W, 0);
  if (h->mode == 3 || h->mode == 4) {
    std::vector<int32_t> fill(h->M, 0);
    for (int i = 0; i < h->N; i++) { int v = h->imap[i]; h_output_map[(size_t)v * W + 1 + fill[v]++] = i; }
    for (int v = 0; v < h->M; v++) h_output_map[(size_t)v * W] = h->count[v];
  } else {
    for (int v = 0; v < h->M; v++) {
      h_output_map[(size_t)v * W] = 1;
      h_output_map[(size_t)v * W + 1] = (h->mode == 2) ? h->last[v] : h->first[v];
    }
  }
  for (int v = 0; v < h->M; v++) {
    int p = h_output_map[(size_t)v * W + 1];
    for (int j = 0; j < h->ncol; j++) h_output_coords[(size_t)v * h->ncol + j] = h_coords[(size_t)p * h->ncol + j];
  }
  delete h;
  return SGB_OK;
}

// ---- RLE wire format of the reference (softgroup/util/rle.py:5-19), host side ------------------------------
// ids: ascending point ids of all masks back to back; offs [n_masks+1]; writes "start len start len ..." (1-based
// starts) per mask into out, out_offs [n_masks+1] = byte ranges. Returns bytes written or SGB_ERR_OVERFLOW.
long long sgb_rle_format_ids(const int32_t *h_ids, const long long *h_offs, int n_masks, char *h_out,
                             long long out_cap, long long *h_out_offs) {
  auto put = [](char *p, long long v) -> char * {
    char tmp[24];
    int n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) *p++ = tmp[--n];
    return p;
  };
  char *p = h_out;
  char *end = h_out + out_cap;
  for (int m = 0; m < n_masks; m++) {
    h_out_offs[m] = p - h_out;
    long long a = h_offs[m], b = h_offs[m + 1];
    bool first = true;
    long long i = a;
    while (i < b) {
      long long j = i + 1;
      while (j < b && h_ids[j] == h_ids[j - 1] + 1) j++;
      if (end - p < 48) { set_error("sgb_rle_format_ids: output buffer too small"); return SGB_ERR_OVERFLOW; }
      if (!first) *p++ = ' ';
      p = put(p, (long long)h_ids[i] + 1);
      *p++ = ' ';
      p = put(p, j - i);
      first = false;
      i = j;
    }
  }
  h_out_offs[n_masks] = p - h_out;
  return p - h_out;
}

int sgb_voxelize_fp(const float *d_feats, float *d_out, const int32_t *d_rules, int mode, int M, int maxActive, int C,
                    void *stream) {
  if (M == 0 || C == 0) return SGB_OK;
  SGB_REQUIRE(d_feats && d_out && d_rules && M > 0 && C > 0 && maxActive >= 0, SGB_ERR_ARG, "voxelize_fp arguments");
  long long tot = (long long)M * C;
  voxelize_fp_kernel<<<div_up(tot, 256), 256, 0, (cudaStream_t)stream>>>(d_feats, d_out, d_rules, M, maxActive + 1, C,
                                                                        mode == 4);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_voxelize_bp(const float *d_d_out, float *d_d_feats, const int32_t *d_rules, int mode, int M, int maxActive,
                    int C, void *stream) {
  if (M == 0 || C == 0) return SGB_OK;
  SGB_REQUIRE(d_d_out && d_d_feats && d_rules && M > 0 && C > 0, SGB_ERR_ARG, "voxelize_bp arguments");
  long long tot = (long long)M * C;
  voxelize_bp_kernel<<<div_up(tot, 256), 256, 0, (cudaStream_t)stream>>>(d_d_out, d_d_feats, d_rules, M, maxActive + 1,
                                                                        C, mode == 4);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_bn_relu(const float *d_x, int x_stride, const float *d_scale, const float *d_shift, int relu, float *d_y,
                int y_stride, int M, int C, void *stream) {
  if (M == 0 || C == 0) return SGB_OK;
  SGB_REQUIRE(d_x && d_scale && d_shift && d_y, SGB_ERR_ARG, "bn_relu arguments");
  long long tot = (long long)M * C;
  bn_relu_kernel<<<div_up(tot, 256), 256, 0, (cudaStream_t)stream>>>(d_x, x_stride, d_scale, d_shift, relu, d_y,
                                                                    y_stride, M, C);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_gather_rows(const float *d_in, const int32_t *d_index, float *d_out, int N, int C, void *stream) {
  if (N == 0 || C == 0) return SGB_OK;
  SGB_REQUIRE(d_in && d_index && d_out, SGB_ERR_ARG, "gather_rows arguments");
  bool vec = (C % 4 == 0) && (((uintptr_t)d_in | (uintptr_t)d_out) % 16 == 0);
  if (vec) {
    long long tot = (long long)N * (C / 4);
    gather_rows_kernel<<<div_up(tot, 256), 256, 0, (cudaStream_t)stream>>>(d_in, d_index, d_out, N, C / 4);
  } else {
    long long tot = (long long)N * C;
    gather_rows_scalar_kernel<<<div_up(tot, 256), 256, 0, (cudaStream_t)stream>>>(d_in, d_index, d_out, N, C);
  }
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
}
