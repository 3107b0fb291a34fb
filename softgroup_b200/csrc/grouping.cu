// grouping.cu -- the per-class point selection in front of the ball query, all classes in one pass.
//
// Replaces, for every class of softgroup/model/softgroup.py:427-446 at once,
//     object_idxs = (semantic_scores[:, class_id] > score_thr).nonzero()      (:432)
//     if object_idxs.size(0) < min_npoint: continue                           (:437-439)
//     batch_idxs_ = batch_idxs[object_idxs]; coords_ = coords_float[object_idxs]; pt_offsets_ = pt_offsets[object_idxs]
//     ... ball_query(coords_ + pt_offsets_, batch_idxs_, batch_offsets_, ...)  (:440-452)
// by entry lists in class-major, ascending-point order (the order in which the reference concatenates its per-class
// results): pts[e] = point, seg[e] = rank(class) * B + batch[point], shifted[e] = coords[point] + offsets[point] (one fp32
// add, like the reference), seg_offsets = exclusive scan of the entries per (class, batch item). The PyTorch formulation of
// the same thing was ~30 small launches (index, compare, sum, nonzero, bincount, cumsum, gathers) with two host
// synchronisations and two pageable H2D copies in the middle of the forward; this is 4 launches and none.
// Selection is a strict fp32 comparison on the caller's softmax scores: bit-exact by construction.
#include <algorithm>

#include "common.cuh"

namespace sgb {

constexpr int GE_THREADS = 256;  // one point per thread
constexpr int GE_MAXC = 32;      // classes per call (one bit of a thread's selection mask each)

struct GeArgs {
  const float *scores; int N, C;
  int cls[GE_MAXC]; int nc;
  float thr; int min_npoint;
  const int32_t *batch; int B;
  const float *coords, *offsets;
  int32_t *pts, *seg; float *shifted;
  int32_t *seg_offsets;   // [nc * B + 1]
  int32_t *blk_cnt;       // [nc][nblk] counts, scanned in place to global entry offsets
  int32_t *seg_cnt;       // [nc * B]
  int32_t *total;         // [1 + nc]: entries, then kept count per class
  int nblk;
};

// counts per (class, block of 256 points)
__global__ void ge_count_kernel(GeArgs p) {
  __shared__ int s_cnt[GE_MAXC];
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid < p.nc) s_cnt[tid] = 0;
  __syncthreads();
  const int pt = blockIdx.x * GE_THREADS + tid;
  const float *row = p.scores + (size_t)min(pt, p.N - 1) * p.C;
  for (int j = 0; j < p.nc; j++) {
    const bool f = pt < p.N && row[p.cls[j]] > p.thr;
    const unsigned int b = __ballot_sync(0xffffffffu, f);
    if (lane == 0 && b) atomicAdd(&s_cnt[j], __popc(b));
  }
  __syncthreads();
  if (tid < p.nc) p.blk_cnt[(size_t)tid * p.nblk + blockIdx.x] = s_cnt[tid];
}

// one CTA: class totals -> keep (>= min_npoint) -> class bases -> per-(class, block) entry offsets in place
__global__ void ge_scan_kernel(GeArgs p) {
  __shared__ int s_tot[GE_MAXC], s_base[GE_MAXC];
  __shared__ int s_part[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int j = 0; j < p.nc; j++) {  // exclusive scan of class j's block counts (chunks of blockDim.x)
    int run = 0;
    int32_t *c = p.blk_cnt + (size_t)j * p.nblk;
    for (int b0 = 0; b0 < p.nblk; b0 += blockDim.x) {
      const int i = b0 + tid;
      const int v = i < p.nblk ? c[i] : 0;
      int x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) s_part[warp] = x;
      __syncthreads();
      if (warp == 0) {
        int w = lane < nw ? s_part[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, w, o);
          if (lane >= o) w += y;
        }
        s_part[lane] = w;  // inclusive over warps
      }
      __syncthreads();
      const int before = (warp ? s_part[warp - 1] : 0) + x - v;
      if (i < p.nblk) c[i] = run + before;
      run += s_part[nw - 1];
      __syncthreads();
    }
    if (tid == 0) s_tot[j] = run;
  }
  __syncthreads();
  if (tid == 0) {
    int base = 0;
    for (int j = 0; j < p.nc; j++) {
      const bool keep = s_tot[j] >= p.min_npoint;  // `object_idxs.size(0) < min_npoint -> continue`
      s_base[j] = keep ? base : -1;
      p.total[1 + j] = keep ? s_tot[j] : 0;
      if (keep) base += s_tot[j];
    }
    p.total[0] = base;
  }
  __syncthreads();
  for (int j = 0; j < p.nc; j++) {
    int32_t *c = p.blk_cnt + (size_t)j * p.nblk;
    const int base = s_base[j];
    for (int i = tid; i < p.nblk; i += blockDim.x) c[i] = base < 0 ? -1 : c[i] + base;
  }
  for (int i = tid; i < p.nc * p.B; i += blockDim.x) p.seg_cnt[i] = 0;
}

__global__ void ge_fill_kernel(GeArgs p) {
  __shared__ int s_w[GE_THREADS / 32][GE_MAXC];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int pt = blockIdx.x * GE_THREADS + tid;
  const bool in = pt < p.N;
  const float *row = p.scores + (size_t)min(pt, p.N - 1) * p.C;
  unsigned int mine = 0u;  // bit j: this point is selected for class j
  for (int j = 0; j < p.nc; j++) {
    const bool f = in && row[p.cls[j]] > p.thr;
    const unsigned int b = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_w[warp][j] = __popc(b);
    if (f) mine |= 1u << j;
  }
  __syncthreads();
  int bt = 0;
  float cx = 0.f, cy = 0.f, cz = 0.f;
  if (mine) {
    bt = p.batch[pt];
    cx = p.coords[3 * (size_t)pt] + p.offsets[3 * (size_t)pt];
    cy = p.coords[3 * (size_t)pt + 1] + p.offsets[3 * (size_t)pt + 1];
    cz = p.coords[3 * (size_t)pt + 2] + p.offsets[3 * (size_t)pt + 2];
  }
  for (int j = 0; j < p.nc; j++) {  // every lane stays in the loop: the ballots are full-warp
    const bool f = (mine >> j) & 1u;
    const unsigned int b = __ballot_sync(0xffffffffu, f);
    const int base = p.blk_cnt[(size_t)j * p.nblk + blockIdx.x];
    // one atomic per (warp, batch item) on the segment counter instead of one per entry (131k adds on <= nc*B words
    // serialised in L2)
    const unsigned int peers = __match_any_sync(0xffffffffu, f ? bt : (0x40000000 | lane));
    if (f && base >= 0 && lane == __ffs(peers) - 1) atomicAdd(&p.seg_cnt[j * p.B + bt], __popc(peers));
    if (f && base >= 0) {  // base < 0: class dropped by min_npoint
      int before = 0;
      for (int w = 0; w < warp; w++) before += s_w[w][j];
      const int pos = base + before + __popc(b & ((1u << lane) - 1u));
      p.pts[pos] = pt;
      const int sg = j * p.B + bt;
      p.seg[pos] = sg;
      p.shifted[3 * (size_t)pos] = cx;
      p.shifted[3 * (size_t)pos + 1] = cy;
      p.shifted[3 * (size_t)pos + 2] = cz;
    }
  }
}

__global__ void ge_segoff_kernel(GeArgs p) {  // one warp-sized problem: exclusive scan of the (class, batch) counts
  if (threadIdx.x == 0) {
    int run = 0;
    const int n = p.nc * p.B;
    for (int i = 0; i < n; i++) {
      p.seg_offsets[i] = run;
      run += p.seg_cnt[i];
    }
    p.seg_offsets[n] = run;
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_group_entries_workspace_bytes(int N, int nc, int B) {
  const size_t nblk = (size_t)div_up(std::max(N, 1), GE_THREADS);
  return align_up((size_t)nc * nblk * 4) + align_up((size_t)nc * (size_t)std::max(B, 1) * 4) + 256;
}

int sgb_group_entries(const float *d_scores, int N, int C, const int *h_classes, int nc, float score_thr, int min_npoint,
                      const int32_t *d_batch_idxs, int B, const float *d_coords, const float *d_offsets, int32_t *d_pts,
                      int32_t *d_seg, float *d_shifted, int32_t *d_seg_offsets, int32_t *d_total, void *d_ws, size_t ws_bytes,
                      void *stream) {
  SGB_REQUIRE(N >= 0 && C >= 1 && nc >= 1 && nc <= GE_MAXC && B >= 1 && h_classes, SGB_ERR_ARG, "group_entries arguments (<= 32 classes per call)");
  SGB_REQUIRE(d_seg_offsets && d_total && d_ws, SGB_ERR_ARG, "group_entries outputs");
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) {
    SGB_CUDA_CHECK(cudaMemsetAsync(d_seg_offsets, 0, ((size_t)nc * B + 1) * 4, st));
    SGB_CUDA_CHECK(cudaMemsetAsync(d_total, 0, ((size_t)nc + 1) * 4, st));
    return SGB_OK;
  }
  SGB_REQUIRE(d_scores && d_batch_idxs && d_coords && d_offsets && d_pts && d_seg && d_shifted, SGB_ERR_ARG, "group_entries inputs");
  SGB_REQUIRE(ws_bytes >= sgb_group_entries_workspace_bytes(N, nc, B), SGB_ERR_WORKSPACE, "group_entries workspace too small");
  GeArgs p;
  p.scores = d_scores; p.N = N; p.C = C;
  for (int j = 0; j < nc; j++) {
    SGB_REQUIRE(h_classes[j] >= 0 && h_classes[j] < C, SGB_ERR_RANGE, "group_entries: class id outside the score columns");
    p.cls[j] = h_classes[j];
  }
  p.nc = nc; p.thr = score_thr; p.min_npoint = min_npoint;
  p.batch = d_batch_idxs; p.B = B; p.coords = d_coords; p.offsets = d_offsets;
  p.pts = d_pts; p.seg = d_seg; p.shifted = d_shifted; p.seg_offsets = d_seg_offsets; p.total = d_total;
  p.nblk = div_up(N, GE_THREADS);
  Arena a(d_ws, ws_bytes);
  p.blk_cnt = a.take<int32_t>((size_t)nc * p.nblk);
  p.seg_cnt = a.take<int32_t>((size_t)nc * B);
  SGB_REQUIRE(p.blk_cnt && p.seg_cnt, SGB_ERR_WORKSPACE, "group_entries workspace carve");
  ge_count_kernel<<<p.nblk, GE_THREADS, 0, st>>>(p);
  SGB_LAUNCH_CHECK();
  ge_scan_kernel<<<1, 1024, 0, st>>>(p);
  SGB_LAUNCH_CHECK();
  ge_fill_kernel<<<p.nblk, GE_THREADS, 0, st>>>(p);
  SGB_LAUNCH_CHECK();
  ge_segoff_kernel<<<1, 32, 0, st>>>(p);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
}
