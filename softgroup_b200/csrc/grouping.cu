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
//
// Any number of classes (ScanNet200 groups 198): the selection is kept as one 32-bit word per (tile of 32 points, class
// rank), written once by ge_count_kernel and read by ge_fill_kernel instead of the scores. ge_count_kernel reads the scores
// with one class per lane, so every load instruction takes consecutive columns of one row whatever C is. The class ids
// travel by value in the kernel parameters (GE_SLICE per launch; more classes take one more count launch per slice), so
// there is no host wait and no host-to-device copy.
#include <algorithm>

#include "common.cuh"

namespace sgb {

constexpr int GE_THREADS = 256;               // a block: 256 points = GE_TILES tiles of 32 points, one warp each
constexpr int GE_TILES = GE_THREADS / 32;
constexpr int GE_SLICE = 256;                 // class ids per ge_count_kernel launch (1 KB of kernel parameters)
constexpr int GE_SCAN_THREADS = 1024;

struct GeArgs {
  const float *scores; int N, C;
  int nc;
  float thr; int min_npoint;
  const int32_t *batch; int B;
  const float *coords, *offsets;
  int32_t *pts, *seg; float *shifted;
  int32_t *seg_offsets;   // [nc * B + 1]
  uint32_t *sel;          // [nblk * GE_TILES][nc]: bit q of sel[t][j] = point 32t+q passes class rank j
  int32_t *blk_cnt;       // [nblk][nc] counts, scanned in place to entry offsets within the class
  int32_t *seg_cnt;       // [nc * B]
  int32_t *total;         // [1 + nc]: entries, then kept count per class
  int nblk;
};

struct GeSlice {  // class ranks [j0, j0 + n) and their score columns
  int j0, n;
  int col[GE_SLICE];
};

__device__ __forceinline__ int warp_incl_scan(int x) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x;
}

// exclusive scan of v over the CTA, sum = the CTA's total; every thread calls it (s_part: 32 ints)
__device__ __forceinline__ int block_excl_scan(int v, int *s_part, int &sum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int x = warp_incl_scan(v);
  if (lane == 31) s_part[warp] = x;
  __syncthreads();
  if (warp == 0) {
    const int w = warp_incl_scan(lane < nw ? s_part[lane] : 0);
    s_part[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  const int r = (warp ? s_part[warp - 1] : 0) + x - v;
  sum = s_part[nw - 1];
  __syncthreads();  // s_part is reused by the next call
  return r;
}

// selection words and counts per (class, block of 256 points) for the class ranks of one slice. Lane l takes class rank
// j0 + k0 + l and walks the 32 points of its warp's tile.
__global__ void ge_count_kernel(GeArgs p, GeSlice s) {
  __shared__ int s_cnt[GE_TILES][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = blockIdx.x * GE_TILES + warp;  // tile: points [32t, 32t + 32)
  const int np = min(32, p.N - t * 32);        // <= 0 for the empty tiles of the last block
  for (int k0 = 0; k0 < s.n; k0 += 32) {
    const int r = k0 + lane;
    const bool on = r < s.n;
    uint32_t m = 0u;
    if (on && np > 0) {
      const float *col = p.scores + (size_t)t * 32 * p.C + s.col[r];
      const size_t ld = p.C;
#pragma unroll 1
      for (int q0 = 0; q0 < 32; q0 += 16) {
        float v[16];  // 16 loads in flight before the first compare (rows past N re-read the tile's last row)
#pragma unroll
        for (int q = 0; q < 16; q++) v[q] = __ldg(col + min(q0 + q, np - 1) * ld);
#pragma unroll
        for (int q = 0; q < 16; q++)
          if (q0 + q < np && v[q] > p.thr) m |= 1u << (q0 + q);
      }
    }
    if (on) p.sel[(size_t)t * p.nc + s.j0 + r] = m;
    s_cnt[warp][lane] = __popc(m);
    __syncthreads();
    if (warp == 0 && on) {
      int c = 0;
#pragma unroll
      for (int w = 0; w < GE_TILES; w++) c += s_cnt[w][lane];
      p.blk_cnt[(size_t)blockIdx.x * p.nc + s.j0 + r] = c;
    }
    __syncthreads();
  }
}

// one CTA per class rank j: its block counts -> entry offsets within the class (in place), the class total and the
// `object_idxs.size(0) < min_npoint -> continue` drop; zeroes the class's segment counters for ge_fill_kernel
__global__ void ge_scan_kernel(GeArgs p) {
  __shared__ int s_part[32];
  const int j = blockIdx.x;
  int run = 0;
  for (int b0 = 0; b0 < p.nblk; b0 += blockDim.x) {
    const int i = b0 + threadIdx.x;
    const int v = i < p.nblk ? p.blk_cnt[(size_t)i * p.nc + j] : 0;
    int sum;
    const int e = block_excl_scan(v, s_part, sum);
    if (i < p.nblk) p.blk_cnt[(size_t)i * p.nc + j] = run + e;
    run += sum;
  }
  if (threadIdx.x == 0) p.total[1 + j] = run >= p.min_npoint ? run : 0;
  for (int i = threadIdx.x; i < p.B; i += blockDim.x) p.seg_cnt[(size_t)j * p.B + i] = 0;
}

// ordered compaction, one point per lane: the entry of (class rank j, point) goes to the class base (exclusive scan of the
// kept totals, recomputed per warp 32 classes at a time) + the block's offset in the class + the earlier tiles of the
// block + the earlier lanes of the tile
__global__ void ge_fill_kernel(GeArgs p) {
  __shared__ uint32_t s_sel[GE_TILES][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = blockIdx.x * GE_TILES + warp;
  const int pt = t * 32 + lane;
  int bt = 0;
  float cx = 0.f, cy = 0.f, cz = 0.f;
  if (pt < p.N) {
    bt = p.batch[pt];
    cx = p.coords[3 * (size_t)pt] + p.offsets[3 * (size_t)pt];
    cy = p.coords[3 * (size_t)pt + 1] + p.offsets[3 * (size_t)pt + 1];
    cz = p.coords[3 * (size_t)pt + 2] + p.offsets[3 * (size_t)pt + 2];
  }
  // lanes of the same batch item: one atomic per (warp, class, batch item) on the segment counter instead of one per entry
  // (lanes past N never have a selection bit, so their group does not matter)
  const unsigned int peers = __match_any_sync(0xffffffffu, bt);
  const unsigned int below = (1u << lane) - 1u;
  int run = 0;  // entries of the classes before k0
  for (int k0 = 0; k0 < p.nc; k0 += 32) {
    const int j = k0 + lane;
    const int kept = j < p.nc ? p.total[1 + j] : 0;  // 0 for a class dropped by min_npoint: it gets no entries
    const int incl = warp_incl_scan(kept);
    const uint32_t m = kept ? p.sel[(size_t)t * p.nc + j] : 0u;
    __syncthreads();  // the previous chunk's readers of s_sel are done
    s_sel[warp][lane] = m;
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; w++) before += __popc(s_sel[w][lane]);
    const int base = kept ? run + incl - kept + p.blk_cnt[(size_t)blockIdx.x * p.nc + j] + before : 0;
    run += __shfl_sync(0xffffffffu, incl, 31);
    // only the classes this tile has points of (most words are 0 when there are many classes); every lane stays in the
    // loop: mj and bj are broadcasts
    for (unsigned int nz = __ballot_sync(0xffffffffu, m != 0u); nz; nz &= nz - 1u) {
      const int jj = __ffs(nz) - 1;
      const uint32_t mj = __shfl_sync(0xffffffffu, m, jj);
      const int bj = __shfl_sync(0xffffffffu, base, jj);
      if ((mj >> lane) & 1u) {
        const int pos = bj + __popc(mj & below);
        const int sg = (k0 + jj) * p.B + bt;
        p.pts[pos] = pt;
        p.seg[pos] = sg;
        p.shifted[3 * (size_t)pos] = cx;
        p.shifted[3 * (size_t)pos + 1] = cy;
        p.shifted[3 * (size_t)pos + 2] = cz;
        const unsigned int g = peers & mj;
        if (lane == __ffs(g) - 1) atomicAdd(&p.seg_cnt[sg], __popc(g));
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) p.total[0] = run;
}

__global__ void ge_segoff_kernel(GeArgs p) {  // one CTA: exclusive scan of the (class, batch item) counts
  __shared__ int s_part[32];
  const int n = p.nc * p.B;
  int run = 0;
  for (int i0 = 0; i0 < n; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const int v = i < n ? p.seg_cnt[i] : 0;
    int sum;
    const int e = block_excl_scan(v, s_part, sum);
    if (i < n) p.seg_offsets[i] = run + e;
    run += sum;
  }
  if (threadIdx.x == 0) p.seg_offsets[n] = run;
}

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_group_entries_workspace_bytes(int N, int nc, int B) {
  const size_t nblk = (size_t)div_up(std::max(N, 1), GE_THREADS);
  const size_t c = (size_t)std::max(nc, 1);
  return align_up(nblk * GE_TILES * c * 4) + align_up(nblk * c * 4) + align_up(c * (size_t)std::max(B, 1) * 4) + 256;
}

int sgb_group_entries(const float *d_scores, int N, int C, const int *h_classes, int nc, float score_thr, int min_npoint,
                      const int32_t *d_batch_idxs, int B, const float *d_coords, const float *d_offsets, int32_t *d_pts,
                      int32_t *d_seg, float *d_shifted, int32_t *d_seg_offsets, int32_t *d_total, void *d_ws, size_t ws_bytes,
                      void *stream) {
  SGB_REQUIRE(N >= 0 && C >= 1 && nc >= 1 && B >= 1 && h_classes, SGB_ERR_ARG, "group_entries arguments");
  SGB_REQUIRE((long long)N * nc < (1ll << 31) && (long long)nc * B < (1ll << 31), SGB_ERR_RANGE,
              "group_entries: N * nc entries and nc * B segments must stay below 2^31 (int32 positions)");
  SGB_REQUIRE(d_seg_offsets && d_total && d_ws, SGB_ERR_ARG, "group_entries outputs");
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) {
    SGB_CUDA_CHECK(cudaMemsetAsync(d_seg_offsets, 0, ((size_t)nc * B + 1) * 4, st));
    SGB_CUDA_CHECK(cudaMemsetAsync(d_total, 0, ((size_t)nc + 1) * 4, st));
    return SGB_OK;
  }
  SGB_REQUIRE(d_scores && d_batch_idxs && d_coords && d_offsets && d_pts && d_seg && d_shifted, SGB_ERR_ARG, "group_entries inputs");
  SGB_REQUIRE(ws_bytes >= sgb_group_entries_workspace_bytes(N, nc, B), SGB_ERR_WORKSPACE, "group_entries workspace too small");
  for (int j = 0; j < nc; j++)
    SGB_REQUIRE(h_classes[j] >= 0 && h_classes[j] < C, SGB_ERR_RANGE, "group_entries: class id outside the score columns");
  GeArgs p;
  p.scores = d_scores; p.N = N; p.C = C;
  p.nc = nc; p.thr = score_thr; p.min_npoint = min_npoint;
  p.batch = d_batch_idxs; p.B = B; p.coords = d_coords; p.offsets = d_offsets;
  p.pts = d_pts; p.seg = d_seg; p.shifted = d_shifted; p.seg_offsets = d_seg_offsets; p.total = d_total;
  p.nblk = div_up(N, GE_THREADS);
  Arena a(d_ws, ws_bytes);
  p.sel = a.take<uint32_t>((size_t)p.nblk * GE_TILES * nc);
  p.blk_cnt = a.take<int32_t>((size_t)p.nblk * nc);
  p.seg_cnt = a.take<int32_t>((size_t)nc * B);
  SGB_REQUIRE(p.sel && p.blk_cnt && p.seg_cnt, SGB_ERR_WORKSPACE, "group_entries workspace carve");
  for (int j0 = 0; j0 < nc; j0 += GE_SLICE) {
    GeSlice s;
    s.j0 = j0;
    s.n = std::min(GE_SLICE, nc - j0);
    for (int r = 0; r < s.n; r++) s.col[r] = h_classes[j0 + r];
    ge_count_kernel<<<p.nblk, GE_THREADS, 0, st>>>(p, s);
    SGB_LAUNCH_CHECK();
  }
  ge_scan_kernel<<<nc, GE_SCAN_THREADS, 0, st>>>(p);
  SGB_LAUNCH_CHECK();
  ge_fill_kernel<<<p.nblk, GE_THREADS, 0, st>>>(p);
  SGB_LAUNCH_CHECK();
  ge_segoff_kernel<<<1, GE_SCAN_THREADS, 0, st>>>(p);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
}
