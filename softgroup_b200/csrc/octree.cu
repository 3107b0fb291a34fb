// octree.cu -- SoftGroup++ octree ball query on the GPU.
//
// Replaces build_and_export_octree (softgroup/ops/src/octree_ball_query/octree_ball_query.cpp:19-165, pointer tree
// built on the CPU and uploaded on every call, softgroup/ops/functions.py:14-33) and octree_ball_query_cuda
// (octree_ball_query.cu:56-147: one thread per query, int actives[585] + int neighbor_inds[1000] in local memory).
// Same semantics, bit for bit: fixed 3-level octree over the bounding box (585 nodes in BFS order, 512 leaves),
// midpoint splits with `<` going low, leaf point lists in ascending point index, neighbours emitted LEAF-MAJOR
// (leaf 0..511, ascending index inside a leaf), first 1000 kept, box/sphere rejection test in fp32 with the
// compiled contraction order of the reference (pinned against its kernel in tests/test_gpu_vs_reference.py).
//   build : boxes by one thread per node level; leaf id per point; stable counting sort over 512 bins
//           (per-block histograms -> scan -> in-block stable ranks via match_any)
//   query : one warp per query; lane-parallel box tests over the 8/64/512 nodes (a leaf is active iff it and both
//           ancestors intersect), active leaves visited in order with ballot/popc compaction into a staged list.
#include <algorithm>

#include "common.cuh"

namespace sgb {

constexpr int OC_NODES = 585, OC_LEAVES = 512, OC_MIDS = 73;
constexpr int OC_BLK = 512;

__global__ void oc_boxes_kernel(const float *__restrict__ xyzwhl, float *__restrict__ boxes) {
  // one thread: 585 boxes, same arithmetic as get_octant_box (octree_ball_query.cpp:60-84)
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (int j = 0; j < 6; j++) boxes[j] = xyzwhl[j];
  for (int k = 0; k < OC_MIDS; k++) {
    const float *pb = boxes + 6 * k;
    for (int o = 0; o < 8; o++) {
      float *b = boxes + 6 * (8 * k + o + 1);
      float w = __fdiv_rn(pb[3], 2.f), h = __fdiv_rn(pb[4], 2.f), l = __fdiv_rn(pb[5], 2.f);
      b[0] = (o & 1) ? __fadd_rn(pb[0], __fdiv_rn(w, 2.f)) : __fsub_rn(pb[0], __fdiv_rn(w, 2.f));
      b[1] = (o & 2) ? __fadd_rn(pb[1], __fdiv_rn(h, 2.f)) : __fsub_rn(pb[1], __fdiv_rn(h, 2.f));
      b[2] = (o & 4) ? __fadd_rn(pb[2], __fdiv_rn(l, 2.f)) : __fsub_rn(pb[2], __fdiv_rn(l, 2.f));
      b[3] = w; b[4] = h; b[5] = l;
    }
  }
}

__device__ __forceinline__ int oc_leaf_of(const float *__restrict__ boxes, float x, float y, float z) {
  int node = 0;
#pragma unroll
  for (int lvl = 0; lvl < 3; lvl++) {
    const float *b = boxes + 6 * node;
    int ox = x < b[0] ? 0 : 1, oy = y < b[1] ? 0 : 1, oz = z < b[2] ? 0 : 1;  // octree_ball_query.cpp:52-57
    node = 8 * node + ((oz << 2) + (oy << 1) + ox) + 1;
  }
  return node - OC_MIDS;
}

__global__ void __launch_bounds__(OC_BLK) oc_hist_kernel(const float *__restrict__ pts, int n, const float *__restrict__ boxes,
                                                         int32_t *__restrict__ leaf_of, int32_t *__restrict__ hist /*[512][nblk]*/,
                                                         int nblk) {
  __shared__ int h[OC_LEAVES];
  for (int i = threadIdx.x; i < OC_LEAVES; i += OC_BLK) h[i] = 0;
  __syncthreads();
  int i = blockIdx.x * OC_BLK + threadIdx.x;
  if (i < n) {
    int l = oc_leaf_of(boxes, pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]);
    leaf_of[i] = l;
    atomicAdd(&h[l], 1);
  }
  __syncthreads();
  for (int l = threadIdx.x; l < OC_LEAVES; l += OC_BLK) hist[(size_t)l * nblk + blockIdx.x] = h[l];
}

// after the exclusive scan of hist (leaf-major): stable scatter
__global__ void __launch_bounds__(OC_BLK) oc_scatter_kernel(int n, const int32_t *__restrict__ leaf_of,
                                                            const int32_t *__restrict__ hist_scanned, int nblk,
                                                            int32_t *__restrict__ pt_inds) {
  __shared__ int wcnt[OC_BLK / 32][OC_LEAVES + 1];  // per-warp counts per leaf -> exclusive over warps
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < (OC_BLK / 32) * (OC_LEAVES + 1); i += OC_BLK) (&wcnt[0][0])[i] = 0;
  __syncthreads();
  int i = blockIdx.x * OC_BLK + tid;
  int l = (i < n) ? leaf_of[i] : -1;
  unsigned am = __ballot_sync(0xffffffffu, l >= 0);
  int rank_in_warp = 0;
  if (l >= 0) {
    unsigned peers = __match_any_sync(am, l);
    rank_in_warp = __popc(peers & ((1u << lane) - 1u));
    if (rank_in_warp == 0) wcnt[warp][l] = __popc(peers);
  }
  __syncthreads();
  // exclusive prefix over warps, per leaf
  for (int leaf = tid; leaf < OC_LEAVES; leaf += OC_BLK) {
    int acc = 0;
    for (int w = 0; w < OC_BLK / 32; w++) { int c = wcnt[w][leaf]; wcnt[w][leaf] = acc; acc += c; }
  }
  __syncthreads();
  if (l >= 0) pt_inds[hist_scanned[(size_t)l * nblk + blockIdx.x] + wcnt[warp][l] + rank_in_warp] = i;
}

__global__ void oc_leafstart_kernel(const int32_t *__restrict__ hist_scanned, int nblk, int n, int32_t *__restrict__ pt_start_len) {
  int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= OC_LEAVES) return;
  int s = hist_scanned[(size_t)l * nblk];
  int e = (l + 1 < OC_LEAVES) ? hist_scanned[(size_t)(l + 1) * nblk] : n;
  pt_start_len[2 * l] = s;
  pt_start_len[2 * l + 1] = e - s;
}

// is_interection (octree_ball_query.cu:14-44)
__device__ __forceinline__ bool oc_box_hit(const float *__restrict__ box, float cx, float cy, float cz, float r, float r2) {
  float dx = fabsf(__fsub_rn(box[0], cx)), dy = fabsf(__fsub_rn(box[1], cy)), dz = fabsf(__fsub_rn(box[2], cz));
  float hw = __fdiv_rn(box[3], 2.f), hh = __fdiv_rn(box[4], 2.f), hl = __fdiv_rn(box[5], 2.f);
  if (dx > __fadd_rn(hw, r)) return false;
  if (dy > __fadd_rn(hh, r)) return false;
  if (dz > __fadd_rn(hl, r)) return false;
  if (dx <= hw) return true;
  if (dy <= hh) return true;
  if (dz <= hl) return true;
  float ex = __fsub_rn(dx, hw), ey = __fsub_rn(dy, hh), ez = __fsub_rn(dz, hl);
  float d = __fmaf_rn(ez, ez, __fmaf_rn(ex, ex, __fmul_rn(ey, ey)));
  return d <= r2;
}

constexpr int OQ_WARPS = 8;

__global__ void __launch_bounds__(OQ_WARPS * 32) oc_query_kernel(const float *__restrict__ pts, const float *__restrict__ boxes,
                                                                 const int32_t *__restrict__ pt_inds,
                                                                 const int32_t *__restrict__ pt_start_len, int n, float radius,
                                                                 long long capacity, int32_t *__restrict__ out_inds,
                                                                 int32_t *__restrict__ out_start_len, int32_t *__restrict__ total) {
  __shared__ float s_boxes[OC_NODES * 6];
  __shared__ int32_t stage[OQ_WARPS][SGB_MAX_NEIGHBORS];
  __shared__ unsigned int s_act[OQ_WARPS][16];  // 512-bit active-leaf mask per warp
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < OC_NODES * 6; i += blockDim.x) s_boxes[i] = boxes[i];
  __syncthreads();
  const float r2 = __fmul_rn(radius, radius);
  for (int q = blockIdx.x * OQ_WARPS + warp; q < n; q += gridDim.x * OQ_WARPS) {
    const float cx = pts[3 * (size_t)q], cy = pts[3 * (size_t)q + 1], cz = pts[3 * (size_t)q + 2];
    // level 1 (8 nodes), level 2 (64), level 3 = leaves (512): node k active iff box hit and parent active
    unsigned a1 = __ballot_sync(0xffffffffu, lane < 8 && oc_box_hit(s_boxes + 6 * (1 + lane), cx, cy, cz, radius, r2)) & 0xFFu;
    unsigned long long a2 = 0ull;
    for (int h = 0; h < 2; h++) {
      int k = h * 32 + lane;  // level-2 node index 0..63, parent = k/8
      bool act = ((a1 >> (k >> 3)) & 1u) && oc_box_hit(s_boxes + 6 * (9 + k), cx, cy, cz, radius, r2);
      a2 |= (unsigned long long)__ballot_sync(0xffffffffu, act) << (32 * h);
    }
    for (int h = 0; h < 16; h++) {
      int k = h * 32 + lane;  // leaf 0..511, parent level-2 node = k/8
      bool act = ((a2 >> (k >> 3)) & 1ull) && oc_box_hit(s_boxes + 6 * (OC_MIDS + k), cx, cy, cz, radius, r2);
      unsigned m = __ballot_sync(0xffffffffu, act);
      if (lane == 0) s_act[warp][h] = m;
    }
    __syncwarp();
    int cnt = 0;
    for (int h = 0; h < 16 && cnt < SGB_MAX_NEIGHBORS; h++) {
      unsigned m = s_act[warp][h];
      while (m && cnt < SGB_MAX_NEIGHBORS) {
        int leaf = h * 32 + __ffs(m) - 1;
        m &= m - 1;
        const int s = __ldg(&pt_start_len[2 * leaf]), e = s + __ldg(&pt_start_len[2 * leaf + 1]);
        for (int b0 = s; b0 < e && cnt < SGB_MAX_NEIGHBORS; b0 += 32) {
          int t = b0 + lane;
          bool hit = false;
          int pi = 0;
          if (t < e) {
            pi = __ldg(&pt_inds[t]);
            float dx = __fsub_rn(cx, pts[3 * (size_t)pi]), dy = __fsub_rn(cy, pts[3 * (size_t)pi + 1]),
                  dz = __fsub_rn(cz, pts[3 * (size_t)pi + 2]);
            hit = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy))) < r2;  // is_neighbor (:46-54)
          }
          unsigned hm = __ballot_sync(0xffffffffu, hit);
          int pos = cnt + __popc(hm & ((1u << lane) - 1u));
          if (hit && pos < SGB_MAX_NEIGHBORS) stage[warp][pos] = pi;
          cnt = min(cnt + __popc(hm), SGB_MAX_NEIGHBORS);
        }
      }
    }
    __syncwarp();
    int base = 0;
    if (lane == 0) {
      base = atomicAdd(total, cnt);
      out_start_len[2 * (size_t)q] = base;
      out_start_len[2 * (size_t)q + 1] = cnt;
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    if ((long long)base < capacity) {
      int cw = cnt;
      if ((long long)base + cnt >= capacity) cw = (int)(capacity - base);
      for (int k = lane; k < cw; k += 32) out_inds[(size_t)base + k] = stage[warp][k];
    }
    __syncwarp();
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_octree_workspace_bytes(int n) {
  if (n < 0) n = 0;
  size_t nblk = (size_t)div_up(std::max(n, 1), OC_BLK);
  return align_up(64 * 4) + align_up(((size_t)n + 1) * 4) + align_up(nblk * OC_LEAVES * 4 + 4) +
         align_up(scan_temp_elems(nblk * OC_LEAVES + 1) * 4) + 1024;
}

int sgb_octree_build(const float *d_points, int n, const float *d_xyzwhl, float *d_boxes, int32_t *d_pt_inds,
                     int32_t *d_pt_start_len, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n >= 0 && d_xyzwhl && d_boxes && d_pt_start_len && d_ws, SGB_ERR_ARG, "octree_build arguments");
  oc_boxes_kernel<<<1, 32, 0, st>>>(d_xyzwhl, d_boxes);
  SGB_LAUNCH_CHECK();
  if (n == 0) {
    SGB_CUDA_CHECK(cudaMemsetAsync(d_pt_start_len, 0, OC_LEAVES * 2 * 4, st));
    return SGB_OK;
  }
  SGB_REQUIRE(d_points && d_pt_inds, SGB_ERR_ARG, "null pointer");
  Arena a(d_ws, ws_bytes);
  int nblk = div_up(n, OC_BLK);
  a.take<int32_t>(64);
  int32_t *leaf_of = a.take<int32_t>((size_t)n + 1);
  int32_t *hist = a.take<int32_t>((size_t)nblk * OC_LEAVES + 1);
  int32_t *tmp = a.take<int32_t>(scan_temp_elems((size_t)nblk * OC_LEAVES + 1));
  SGB_REQUIRE(tmp, SGB_ERR_WORKSPACE, "octree workspace too small");
  oc_hist_kernel<<<nblk, OC_BLK, 0, st>>>(d_points, n, d_boxes, leaf_of, hist, nblk);
  SGB_LAUNCH_CHECK();
  int rc = exclusive_scan_i32(hist, hist, (size_t)nblk * OC_LEAVES, nullptr, tmp, st);
  if (rc) return rc;
  oc_scatter_kernel<<<nblk, OC_BLK, 0, st>>>(n, leaf_of, hist, nblk, d_pt_inds);
  SGB_LAUNCH_CHECK();
  oc_leafstart_kernel<<<2, 256, 0, st>>>(hist, nblk, n, d_pt_start_len);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

long long sgb_octree_ball_query(const float *d_points, const float *d_boxes, const int32_t *d_pt_inds,
                                const int32_t *d_pt_start_len, int n, int mean_active, float radius, int32_t *d_out_inds,
                                int32_t *d_out_start_len, int32_t *d_total, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  SGB_REQUIRE(d_points && d_boxes && d_pt_inds && d_pt_start_len && d_out_start_len && d_total && mean_active >= 0,
              SGB_ERR_ARG, "octree_ball_query arguments");
  SGB_CURRENT_DEVICE(d);
  SGB_CUDA_CHECK(cudaMemsetAsync(d_total, 0, 4, st));
  int grid = std::min(div_up(n, OQ_WARPS), d->sms * 4);
  oc_query_kernel<<<grid, OQ_WARPS * 32, 0, st>>>(d_points, d_boxes, d_pt_inds, d_pt_start_len, n, radius,
                                                 (long long)n * mean_active, d_out_inds, d_out_start_len, d_total);
  SGB_LAUNCH_CHECK();
  int tot = 0;
  SGB_CUDA_CHECK(cudaMemcpyAsync(&tot, d_total, 4, cudaMemcpyDeviceToHost, st));
  SGB_CUDA_CHECK(cudaStreamSynchronize(st));
  return (long long)tot;
}
}
