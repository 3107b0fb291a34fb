// instances.cu -- the tail of the forward on the GPU: instance mask selection, run-length encoding, panoptic paste, and
// the prediction/ground-truth intersection matrix of the evaluation.
//
// Replaces (reference file:line):
//   get_instances           softgroup/model/softgroup.py:537-604  18 dense int32 [nProposal, N] masks -> D2H -> numpy RLE
//   rle_encode              softgroup/util/rle.py:5-19            np.where(mask[1:] != mask[:-1]) per instance on the host
//   panoptic_fusion         softgroup/model/softgroup.py:606-639  rle_decode + numpy paste loop per instance
//   assign_instances_for_scan  softgroup/evaluation/instance_eval.py:228-309  np.count_nonzero per (pred, gt) pair
// Masks are bitmaps [instance][W words], W = ceil((N + 1) / 32): bit N is always 0, so the closing transition of a mask
// that ends at point N-1 falls inside the bitmap like the reference's trailing pad (rle.py:14). A transition at point k
// (mask[k] != mask[k-1], mask[-1] = 0) is bit k of  t = x ^ ((x << 1) | carry)  -- one word-parallel pass finds every
// run boundary; the host only formats "start len" pairs from the (already sorted) transition positions.
#include <algorithm>

#include "common.cuh"

namespace sgb {

// npoint[p * nI + i] = #entries e of proposal p with mask_scores[e, i] > thr  (softgroup.py:553, 563-565 `mask_pred.sum(1)`).
// proposals_idx [S, 2] (proposal id, point); entries of one proposal are contiguous (cluster order), so a warp mostly
// holds one proposal: match_any groups + ballot popcounts keep the atomics at one per (warp, proposal, class).
__global__ void inst_count_kernel(const int32_t *__restrict__ pidx, const float *__restrict__ mask_scores, int ms_stride, int S,
                                  int nI, float thr, int32_t *__restrict__ npoint) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool ok = e < S;
  const int p = ok ? pidx[2 * (size_t)e] : -1;
  const unsigned peers = __match_any_sync(0xffffffffu, p);
  const bool leader = (__ffs(peers) - 1) == lane;
  for (int i = 0; i < nI; i++) {
    const bool on = ok && mask_scores[(size_t)e * ms_stride + i] > thr;
    const unsigned b = __ballot_sync(0xffffffffu, on) & peers;
    if (leader && p >= 0 && b) atomicAdd(&npoint[(size_t)p * nI + i], __popc(b));
  }
}

// slot[i * nP + p] (class-major, the order in which the reference appends instances) -> bitmap rows
__global__ void inst_scatter_kernel(const int32_t *__restrict__ pidx, const float *__restrict__ mask_scores, int ms_stride, int S,
                                    int nI, int nP, float thr, const int32_t *__restrict__ slot, uint32_t *__restrict__ bm, int W) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S) return;
  const int p = pidx[2 * (size_t)e], pt = pidx[2 * (size_t)e + 1];
  for (int i = 0; i < nI; i++) {
    const int s = __ldg(&slot[(size_t)i * nP + p]);
    if (s >= 0 && mask_scores[(size_t)e * ms_stride + i] > thr) atomicOr(&bm[(size_t)s * W + (pt >> 5)], 1u << (pt & 31));
  }
}

// generic: set bit `pt` of row `row[e]` for every entry with row[e] >= 0
__global__ void bitmap_set_kernel(const int32_t *__restrict__ row, const int32_t *__restrict__ pt, long long n, uint32_t *__restrict__ bm,
                                  int W) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int r = row[e];
  if (r >= 0) atomicOr(&bm[(size_t)r * W + (pt[e] >> 5)], 1u << (pt[e] & 31));
}

__device__ __forceinline__ uint32_t transitions_of(const uint32_t *__restrict__ bm, int W, long long g) {
  const int w = (int)(g % W);
  const uint32_t x = bm[g];
  const uint32_t carry = (w > 0) ? (bm[g - 1] >> 31) : 0u;
  return x ^ ((x << 1) | carry);
}

__global__ void rle_count_kernel(const uint32_t *__restrict__ bm, int W, long long total, int32_t *__restrict__ cnt) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  cnt[g] = __popc(transitions_of(bm, W, g));
}

// trans[off[g] ...] = 1-based positions of the transitions of word g (ascending): exactly `runs` of rle.py:15 before the
// `runs[1::2] -= runs[::2]` step. inst_off[r] = off[r * W] (first transition of instance r).
__global__ void rle_fill_kernel(const uint32_t *__restrict__ bm, int W, long long total, const int32_t *__restrict__ off,
                                int32_t *__restrict__ trans, int32_t *__restrict__ inst_off, int n_inst, int grand_total) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g == 0) inst_off[n_inst] = grand_total;
  if (g >= total) return;
  const int w = (int)(g % W);
  int o = off[g];
  if (w == 0) inst_off[g / W] = o;
  uint32_t t = transitions_of(bm, W, g);
  while (t) {
    const int b = __ffs(t) - 1;
    t &= t - 1;
    trans[o++] = w * 32 + b + 1;
  }
}

// inter[r * nG + gslot[pt]] += 1 for every set bit (r, pt); vert[r] = popcount; void_inter[r] = set bits with gslot < 0
// marked void (gslot == -2). One warp per (row, 32-word strip).
__global__ void bitmap_hist_kernel(const uint32_t *__restrict__ bm, int W, int n_rows, int N, const int32_t *__restrict__ gslot,
                                   int nG, int32_t *__restrict__ inter, int32_t *__restrict__ vert, int32_t *__restrict__ void_inter) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n_rows * W) return;
  const int r = (int)(g / W), w = (int)(g % W);
  uint32_t x = bm[g];
  if (!x) return;
  atomicAdd(&vert[r], __popc(x));
  int nvoid = 0;
  while (x) {
    const int b = __ffs(x) - 1;
    x &= x - 1;
    const int pt = w * 32 + b;
    if (pt >= N) continue;
    const int s = __ldg(&gslot[pt]);
    if (s >= 0) atomicAdd(&inter[(size_t)r * nG + s], 1);
    else if (s == -2) nvoid++;
  }
  if (nvoid) atomicAdd(&void_inter[r], nvoid);
}

// panoptic_fusion (softgroup.py:606-639): instances in descending confidence (order[] given by the caller), each is
// skipped when intersect / (size + 1e-5) > skip_iou (float64 like numpy), else pasted where nothing was pasted before.
// One CTA walks the instances in order (the loop is sequential by definition); words are spread over the threads.
constexpr int kPanThreads = 1024;
__global__ void __launch_bounds__(kPanThreads) panoptic_paste_kernel(const uint32_t *__restrict__ bm, int W, int N,
                                                                     const int32_t *__restrict__ order, const int32_t *__restrict__ cls,
                                                                     int n_inst, double skip_iou, uint32_t *__restrict__ prev /*[W] zeroed*/,
                                                                     uint32_t *__restrict__ pan_cls, uint32_t *__restrict__ pan_ids) {
  __shared__ int s_red[2][kPanThreads / 32];
  __shared__ int s_tot[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t next_id = 1;
  for (int k = 0; k < n_inst; k++) {
    const int r = order[k];
    const uint32_t *row = bm + (size_t)r * W;
    int inter = 0, size = 0;
    for (int w = tid; w < W; w += kPanThreads) {
      const uint32_t x = row[w];
      inter += __popc(x & prev[w]);
      size += __popc(x);
    }
    inter = warp_sum(inter);
    size = warp_sum(size);
    if (lane == 0) { s_red[0][warp] = inter; s_red[1][warp] = size; }
    __syncthreads();
    if (warp == 0) {
      int a = (lane < kPanThreads / 32) ? s_red[0][lane] : 0, b = (lane < kPanThreads / 32) ? s_red[1][lane] : 0;
      a = warp_sum(a);
      b = warp_sum(b);
      if (lane == 0) { s_tot[0] = a; s_tot[1] = b; }
    }
    __syncthreads();
    const bool skip = (double)s_tot[0] / ((double)s_tot[1] + 1e-5) > skip_iou;
    if (!skip) {
      const uint32_t c = (uint32_t)cls[r];
      for (int w = tid; w < W; w += kPanThreads) {
        uint32_t paste = row[w] & ~prev[w];
        if (paste) {
          prev[w] |= paste;
          while (paste) {
            const int b = __ffs(paste) - 1;
            paste &= paste - 1;
            const int pt = w * 32 + b;
            if (pt < N) { pan_cls[pt] = c; pan_ids[pt] = next_id; }
          }
        }
      }
      next_id++;
    }
    __syncthreads();
  }
}

// Bitmap rows -> ascending point-id lists. A row is cut into segments of kIdSegWords words; the count pass sums the
// popcounts of every (row, segment), a device-wide scan turns them into int64 output offsets, and the fill pass writes
// each segment's ids at its offset. Bits at N and beyond are masked in both passes, so a row never yields an id >= N.
constexpr int kIdThreads = 256;
constexpr int kIdRounds = 4;
constexpr int kIdSegWords = kIdThreads * kIdRounds;  // 1024 words = 32768 points per segment
constexpr int kIdSegsPerCta = kIdThreads / 32;        // count pass: one warp per segment

__device__ __forceinline__ uint32_t row_word(const uint32_t *__restrict__ row, long long w, int W, int N) {
  if (w >= W) return 0u;
  const uint32_t x = row[w];
  const long long left = (long long)N - w * 32;  // valid bits in this word
  return left >= 32 ? x : (left > 0 ? x & ((1u << left) - 1u) : 0u);
}

// seg_cnt[r * B + s] = set bits of segment s of row r (bits < N)
__global__ void __launch_bounds__(kIdThreads) bitmap_ids_count_kernel(const uint32_t *__restrict__ bm, int W, int N, int B,
                                                                      long long n_seg, long long *__restrict__ seg_cnt) {
  const long long seg = (long long)blockIdx.x * kIdSegsPerCta + (threadIdx.x >> 5);
  if (seg >= n_seg) return;
  const long long r = seg / B;
  const long long w0 = (seg - r * B) * (long long)kIdSegWords;
  const uint32_t *row = bm + (size_t)r * W;
  int c = 0;
  for (int k = lane_id(); k < kIdSegWords; k += 32) c += __popc(row_word(row, w0 + k, W, N));
  c = warp_sum(c);
  if (lane_id() == 0) seg_cnt[seg] = c;
}

// offsets[r] = seg_off[r * B] for r <= n_rows (seg_off has n_rows * B + 1 entries, the last one the grand total)
__global__ void bitmap_row_offsets_kernel(const long long *__restrict__ seg_off, int B, int n_rows, long long *__restrict__ offsets) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r <= n_rows) offsets[r] = seg_off[r * B];
}

// One CTA per (row, segment): kIdRounds rounds of kIdThreads words. Per round every thread takes one word, the CTA
// scans the popcounts (warp shuffles, then the warp totals), the ids land in shared memory at their rank and leave in
// one coalesced copy; ids of a word come out ascending, words in order, so the segment's ids are ascending.
__global__ void __launch_bounds__(kIdThreads) bitmap_ids_fill_kernel(const uint32_t *__restrict__ bm, int W, int N, int B,
                                                                     const long long *__restrict__ seg_off,
                                                                     int32_t *__restrict__ ids) {
  __shared__ int32_t s_ids[kIdThreads * 32];
  __shared__ int s_warp[kIdThreads / 32];
  const long long seg = blockIdx.x;
  long long base = seg_off[seg];
  if (seg_off[seg + 1] == base) return;  // an empty segment is not read again
  const long long r = seg / B;
  const long long w0 = (seg - r * B) * (long long)kIdSegWords;
  const uint32_t *row = bm + (size_t)r * W;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int round = 0; round < kIdRounds; round++) {
    const long long w = w0 + (long long)round * kIdThreads + tid;
    uint32_t x = row_word(row, w, W, N);
    const int c = __popc(x);
    int inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    int before = 0, round_total = 0;
#pragma unroll
    for (int k = 0; k < kIdThreads / 32; k++) {
      const int t = s_warp[k];
      before += k < warp ? t : 0;
      round_total += t;
    }
    int pos = before + inc - c;
    while (x) {
      const int b = __ffs(x) - 1;
      x &= x - 1;
      s_ids[pos++] = (int32_t)(w * 32 + b);
    }
    __syncthreads();
    for (int k = tid; k < round_total; k += kIdThreads) ids[base + k] = s_ids[k];
    base += round_total;
    __syncthreads();  // s_ids and s_warp are reused by the next round
  }
}

// Class bitmaps: bit pt of row row_of[labels[pt]] for every point whose label has a row. A warp covers the 32 points of
// one bitmap word, so each (row, word) has a single writer: the lanes with the same row pool their bits with one
// match_any; counts[row] += the bits (one atomic per warp and row).
__global__ void class_bitmaps_kernel(const int64_t *__restrict__ labels, int N, const int32_t *__restrict__ row_of, int n_labels,
                                     uint32_t *__restrict__ bm, int W, long long *__restrict__ counts) {
  const long long pt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int r = -1;
  if (pt < N) {
    const int64_t l = labels[pt];
    if (l >= 0 && l < n_labels) r = __ldg(&row_of[l]);
  }
  const unsigned peers = __match_any_sync(0xffffffffu, r);
  if (r >= 0 && lane_id() == __ffs(peers) - 1) {
    bm[(size_t)r * W + (pt >> 5)] = peers;
    if (counts) atomicAdd((unsigned long long *)&counts[r], (unsigned long long)__popc(peers));
  }
}

// ---- per-list reductions and the point map over int64-offset id lists ----------------------------------------------
// The id space [0, total) is cut into chunks of kListChunk ids, one warp per chunk, so the work per warp is the same
// whatever the list lengths. A list inside one chunk is finished by that warp. A list that crosses a chunk boundary
// leaves one partial per chunk it touches: in the chunk where it starts, the "tail" slot (2c + 1); in every later chunk,
// the "head" slot (2c). Those lists are finished by id_reduce_lists_kernel, which combines the partials in chunk order.
// Sums are float64 and every combination order is fixed, so a mean has the same bits on every run.
constexpr int kListThreads = 256;
constexpr int kListWarps = kListThreads / 32;
constexpr int kListChunk = 256;
constexpr int kListCtasPerSm = 6;  // 40 registers, no spills (ptxas -v): 48 of 64 warps per multiprocessor

__device__ __forceinline__ int pow2_lanes(int C) {  // channel lanes: pow2 >= min(C, 32)
  int cw = 1;
  while (cw < C && cw < 32) cw <<= 1;
  return cw;
}

// last k in [0, n) with off[k] <= i (0 if none)
__device__ __forceinline__ int list_of(const long long *__restrict__ off, int n, long long i) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kListThreads, kListCtasPerSm) id_reduce_chunks_kernel(
    const long long *__restrict__ off, int n, const int32_t *__restrict__ ids, long long total, int N,
    const float *__restrict__ vals, long long ld, int C, int ops, float *__restrict__ omin, float *__restrict__ omax,
    float *__restrict__ omean, long long *__restrict__ ocnt, double *__restrict__ psum, float *__restrict__ pmin,
    float *__restrict__ pmax, int32_t *__restrict__ pcnt) {
  const int lane = lane_id(), Cw = pow2_lanes(C), rows = 32 / Cw;
  const int tx = lane % Cw, ty = lane / Cw;
  const long long nch = (total + kListChunk - 1) / kListChunk;
  for (long long ch = (long long)blockIdx.x * kListWarps + (threadIdx.x >> 5); ch < nch; ch += (long long)gridDim.x * kListWarps) {
    const long long cs = ch * kListChunk, ce = min(cs + kListChunk, total);
    int k = list_of(off, n, cs);
    long long r0 = cs;
    while (r0 < ce) {
      while (k < n - 1 && off[k + 1] <= r0) k++;  // empty lists have no ids
      const long long start = off[k], end = min(off[k + 1], total);
      const long long e = min(end, ce);
      r0 = max(r0, start);  // ids below offsets[0] belong to no list
      if (e <= r0) break;   // nor do ids at offsets[n] and beyond
      const bool whole = start >= cs && end <= ce;
      const long long slot = 2 * ch + (start < cs ? 0 : 1);
      for (int c0 = 0; c0 < C; c0 += Cw) {
        const int c = c0 + tx;
        double sum = 0.0;
        float mn = INFINITY, mx = -INFINITY;
        int cnt = 0;
        for (long long i = r0 + ty; i < e; i += rows) {
          const int id = __ldg(&ids[i]);
          if ((unsigned)id >= (unsigned)N) continue;  // outside [0, N): never read
          cnt++;
          if (c < C) {
            const float x = __ldg(&vals[(size_t)id * ld + c]);
            mn = (x < mn) ? x : mn;  // the comparisons of seg_minmax_kernel: NaN never wins
            mx = (x > mx) ? x : mx;
            sum += (double)x;
          }
        }
        for (int o = Cw; o < 32; o <<= 1) {  // across the row lanes; lane ty == 0 holds a fixed-order result
          sum += __shfl_xor_sync(0xffffffffu, sum, o);
          const float a = __shfl_xor_sync(0xffffffffu, mn, o), b = __shfl_xor_sync(0xffffffffu, mx, o);
          mn = (a < mn) ? a : mn;
          mx = (b > mx) ? b : mx;
          cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        }
        if (ty == 0 && c < C) {
          if (whole) {
            const size_t o = (size_t)k * C + c;
            if (ops & SGB_REDUCE_MIN) omin[o] = mn;
            if (ops & SGB_REDUCE_MAX) omax[o] = mx;
            if (ops & SGB_REDUCE_MEAN) omean[o] = (float)(sum / (double)cnt);  // 0 / 0 = NaN for no id in [0, N)
            if (c == 0) ocnt[k] = cnt;
          } else {
            const size_t o = (size_t)slot * C + c;
            psum[o] = sum;
            pmin[o] = mn;
            pmax[o] = mx;
            if (c == 0) pcnt[slot] = cnt;
          }
        }
      }
      r0 = e;
    }
  }
}

// Lists the chunk pass did not finish: empty ones, and those spanning chunks (partials tail[c0], head[c0 + 1 .. c1]).
// One CTA per list; per channel, a thread sums every rows_par-th partial in order, then a fixed shared-memory tree.
__global__ void __launch_bounds__(kListThreads) id_reduce_lists_kernel(
    const long long *__restrict__ off, int n, long long total, int C, int ops, const double *__restrict__ psum,
    const float *__restrict__ pmin, const float *__restrict__ pmax, const int32_t *__restrict__ pcnt,
    float *__restrict__ omin, float *__restrict__ omax, float *__restrict__ omean, long long *__restrict__ ocnt) {
  __shared__ double s_sum[kListThreads];
  __shared__ float s_min[kListThreads], s_max[kListThreads];
  __shared__ long long s_cnt[kListWarps];
  const int Cw = pow2_lanes(C), rows_par = kListThreads / Cw;
  const int tx = threadIdx.x % Cw, ty = threadIdx.x / Cw;
  for (int k = blockIdx.x; k < n; k += gridDim.x) {
    const long long s = min(off[k], total), e = min(off[k + 1], total);
    const long long c0 = s / kListChunk, c1 = (e - 1) / kListChunk;
    if (e > s && c0 == c1) continue;  // finished by the chunk pass
    const long long m = e > s ? c1 - c0 + 1 : 0;  // partials, in chunk order
    long long cnt = 0;
    for (long long j = threadIdx.x; j < m; j += kListThreads) cnt += pcnt[j == 0 ? 2 * c0 + 1 : 2 * (c0 + j)];
    cnt = warp_sum(cnt);
    if (lane_id() == 0) s_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    cnt = 0;
    for (int w = 0; w < kListWarps; w++) cnt += s_cnt[w];
    for (int cb = 0; cb < C; cb += Cw) {
      const int c = cb + tx;
      double sum = 0.0;
      float mn = INFINITY, mx = -INFINITY;
      if (c < C)
        for (long long j = ty; j < m; j += rows_par) {
          const size_t o = (size_t)(j == 0 ? 2 * c0 + 1 : 2 * (c0 + j)) * C + c;
          sum += psum[o];
          const float a = pmin[o], b = pmax[o];
          mn = (a < mn) ? a : mn;
          mx = (b > mx) ? b : mx;
        }
      s_sum[threadIdx.x] = sum;
      s_min[threadIdx.x] = mn;
      s_max[threadIdx.x] = mx;
      __syncthreads();
      for (int h = rows_par >> 1; h > 0; h >>= 1) {
        if (ty < h) {
          const int t = threadIdx.x + h * Cw;
          s_sum[threadIdx.x] += s_sum[t];
          s_min[threadIdx.x] = (s_min[t] < s_min[threadIdx.x]) ? s_min[t] : s_min[threadIdx.x];
          s_max[threadIdx.x] = (s_max[t] > s_max[threadIdx.x]) ? s_max[t] : s_max[threadIdx.x];
        }
        __syncthreads();
      }
      if (ty == 0 && c < C) {
        const size_t o = (size_t)k * C + c;
        if (ops & SGB_REDUCE_MIN) omin[o] = s_min[tx];
        if (ops & SGB_REDUCE_MAX) omax[o] = s_max[tx];
        if (ops & SGB_REDUCE_MEAN) omean[o] = (float)(s_sum[tx] / (double)cnt);
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) ocnt[k] = cnt;
  }
}

// (ordered confidence, ~k): the larger key is the higher confidence, then the smaller k. NaN orders below -inf and -0.0
// equals +0.0. Key 0 is no list (~k >= 2^31 for every k < 2^31).
__device__ __forceinline__ unsigned long long point_key(float conf, int k) {
  uint32_t o = 0u;
  if (!isnan(conf)) {
    const uint32_t u = __float_as_uint(conf == 0.f ? 0.f : conf);
    o = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  }
  return ((unsigned long long)o << 32) | (unsigned long long)(~(uint32_t)k);
}

__global__ void __launch_bounds__(kListThreads, kListCtasPerSm) id_map_keys_kernel(const long long *__restrict__ off, int n,
                                                                   const int32_t *__restrict__ ids, long long total, int N,
                                                                   const float *__restrict__ conf,
                                                                   unsigned long long *__restrict__ key) {
  const int lane = lane_id();
  const long long nch = (total + kListChunk - 1) / kListChunk;
  for (long long ch = (long long)blockIdx.x * kListWarps + (threadIdx.x >> 5); ch < nch; ch += (long long)gridDim.x * kListWarps) {
    const long long cs = ch * kListChunk, ce = min(cs + kListChunk, total);
    int k = list_of(off, n, cs);
    for (long long i = cs + lane; i < ce; i += 32) {
      while (k < n - 1 && off[k + 1] <= i) k++;
      if (i < off[k] || i >= off[k + 1]) continue;  // ids outside [offsets[0], offsets[n]) belong to no list
      const int id = __ldg(&ids[i]);
      if ((unsigned)id < (unsigned)N) atomicMax(&key[id], point_key(__ldg(&conf[k]), k));
    }
  }
}

__global__ void id_map_decode_kernel(const unsigned long long *__restrict__ key, int N, int32_t *__restrict__ map) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < N) {
    const unsigned long long v = key[p];
    map[p] = v ? (int32_t)~(uint32_t)v : -1;
  }
}

// ---- farthest-point sampling per id list (sgb_id_lists_fps) ----------------------------------------------------------
// A bin pass sorts the lists by length into three queues; a persistent kernel per queue pulls lists from it: one warp,
// one CTA or one 8-CTA cluster per list. A thread keeps kFpsR positions (x, y, z, d) in registers, and a float4
// (x, y, z, id) copy of each in shared memory broadcasts the chosen point. Each step is one argmax of fps_key over the
// list, so the result does not depend on the reduction order. Lists beyond the cluster's capacity stream their points
// from global memory every step and keep d in the workspace.
constexpr int kFpsR = 16;            // positions per thread
constexpr int kFpsCtaThreads = 512;  // CTA and cluster paths
constexpr int kFpsCtaWarps = kFpsCtaThreads / 32;
constexpr int kFpsWarpLists = 8;     // warp path: lists in flight per CTA
constexpr int kFpsCl = 8;            // CTAs per cluster (portable maximum)
static_assert(SGB_FPS_WARP_MAX == 32 * kFpsR, "warp path capacity");
static_assert(SGB_FPS_CTA_MAX == kFpsCtaThreads * kFpsR, "CTA path capacity");
static_assert(SGB_FPS_CLUSTER_MAX == kFpsCl * SGB_FPS_CTA_MAX, "cluster path on-chip capacity");

// (0 for NaN, else the bits of d + 1 : 0xFFFFFFFF - position): the larger key is the larger d, then the smaller position.
// d is never negative, so its bits order like its value. A valid position's key is never 0 (positions < 2^31).
__device__ __forceinline__ unsigned long long fps_key(float d, int pos) {
  const uint32_t hi = isnan(d) ? 0u : __float_as_uint(d) + 1u;
  return ((unsigned long long)hi << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)pos);
}
__device__ __forceinline__ int fps_pos(unsigned long long key) { return (int)(0xFFFFFFFFu - (uint32_t)key); }
// The chosen point's d is 0 or NaN: every d is then 0 or NaN, the d of a point with d = 0 stays 0 (its coordinates and
// the chosen point's are finite) and NaN stays NaN, so every later step chooses the same position.
__device__ __forceinline__ bool fps_settled(unsigned long long key) { return (key >> 32) <= 1ull; }

__device__ __forceinline__ float fps_dist(float x, float y, float z, float sx, float sy, float sz) {
  const float dx = __fsub_rn(x, sx), dy = __fsub_rn(y, sy), dz = __fsub_rn(z, sz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
__device__ __forceinline__ float fps_min(float d, float t) { return (t < d || t != t) ? t : d; }  // np.minimum: NaN wins
__device__ __forceinline__ unsigned long long umax64(unsigned long long a, unsigned long long b) { return a > b ? a : b; }

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = umax64(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// every thread of the CTA gets the CTA's largest key; one barrier (s_cand is double-buffered by `phase`)
__device__ __forceinline__ unsigned long long cta_max_u64(unsigned long long v, unsigned long long (*s_cand)[kFpsCtaWarps],
                                                          int &phase) {
  v = warp_max_u64(v);
  unsigned long long *c = s_cand[phase++ & 1];
  if (lane_id() == 0) c[threadIdx.x >> 5] = v;
  __syncthreads();
  return warp_max_u64(lane_id() < kFpsCtaWarps ? c[lane_id()] : 0ull);
}

// list k clamped to the id array; a negative length or one beyond 2^31 - 1 positions counts as no position
__device__ __forceinline__ int fps_list(const long long *__restrict__ off, int k, long long total, long long &start) {
  start = min(off[k], total);
  const long long len = min(off[k + 1], total) - start;
  return (len < 0 || len > 0x7FFFFFFFll) ? 0 : (int)len;
}

struct FpsRegs {
  float x[kFpsR], y[kFpsR], z[kFpsR], d[kFpsR];
  uint32_t valid;
};

// positions first + r * STRIDE below `end` into registers (d = +inf) and into s_pts[lfirst + r * STRIDE]; returns the
// largest key of those, i.e. the smallest valid position (0 if none)
template <int STRIDE>
__device__ __forceinline__ unsigned long long fps_load(FpsRegs &p, const int32_t *__restrict__ ids, long long start, int first,
                                                       int end, int N, const float *__restrict__ xyz, long long ld,
                                                       float4 *s_pts, int lfirst) {
  unsigned long long best = 0;
  p.valid = 0;
#pragma unroll
  for (int r = 0; r < kFpsR; r++) {
    const int pos = first + r * STRIDE;
    p.x[r] = p.y[r] = p.z[r] = 0.f;
    p.d[r] = INFINITY;
    const int id = pos < end ? __ldg(&ids[start + pos]) : -1;
    if ((unsigned)id < (unsigned)N) {
      const float *q = xyz + (size_t)id * ld;
      p.x[r] = __ldg(q);
      p.y[r] = __ldg(q + 1);
      p.z[r] = __ldg(q + 2);
      p.valid |= 1u << r;
      s_pts[lfirst + r * STRIDE] = make_float4(p.x[r], p.y[r], p.z[r], __int_as_float(id));
      best = umax64(best, fps_key(INFINITY, pos));
    }
  }
  return best;
}

// one step over the registers: d = min(d, dist to s), returns the largest key
template <int STRIDE>
__device__ __forceinline__ unsigned long long fps_sweep(FpsRegs &p, int first, float sx, float sy, float sz) {
  unsigned long long best = 0;
#pragma unroll
  for (int r = 0; r < kFpsR; r++) {
    if (p.valid & (1u << r)) {
      p.d[r] = fps_min(p.d[r], fps_dist(p.x[r], p.y[r], p.z[r], sx, sy, sz));
      best = umax64(best, fps_key(p.d[r], first + r * STRIDE));
    }
  }
  return best;
}

// Warp path (T = 32: kFpsWarpLists lists per CTA, one per warp, shuffles only) and CTA path (T = kFpsCtaThreads: one list
// per CTA, one barrier per step). Positions are t + r * T, so a position's shared-memory slot is the position itself.
template <int T>
__global__ void __launch_bounds__(T == 32 ? 32 * kFpsWarpLists : T, T == 32 ? 2 : 1)
    fps_lists_kernel(const long long *__restrict__ off, const int32_t *__restrict__ ids, long long total, int N,
                     const float *__restrict__ xyz, long long ld, int K, const int32_t *__restrict__ queue,
                     const int *__restrict__ count, int *head, int32_t *__restrict__ out) {
  extern __shared__ float4 s_pts_all[];  // [lists per CTA][T * kFpsR]
  __shared__ unsigned long long s_cand[2][kFpsCtaWarps];
  __shared__ int s_item;
  const int t = threadIdx.x % T;
  float4 *s_pts = s_pts_all + (threadIdx.x / T) * (T * kFpsR);
  const int n_items = *count;
  int phase = 0;
  FpsRegs p;
  auto group_max = [&](unsigned long long v) {
    if constexpr (T == 32) {
      __syncwarp();  // s_pts stores before the broadcast read
      return warp_max_u64(v);
    } else {
      return cta_max_u64(v, s_cand, phase);
    }
  };
  while (true) {
    int item;
    if constexpr (T == 32) {
      __syncwarp();  // the previous list's s_pts reads before this list's stores
      item = __shfl_sync(0xffffffffu, t == 0 ? atomicAdd(head, 1) : 0, 0);
    } else {
      if (t == 0) s_item = atomicAdd(head, 1);
      __syncthreads();
      item = s_item;
    }
    if (item >= n_items) break;
    const int k = queue[item];
    long long start;
    const int len = fps_list(off, k, total, start);
    int32_t *row = out + (size_t)k * K;
    unsigned long long best = group_max(fps_load<T>(p, ids, start, t, len, N, xyz, ld, s_pts, t));
    if (best == 0) {  // no valid position
      for (int j = t; j < K; j += T) row[j] = -1;
      continue;
    }
    for (int j = 0;; j++) {
      const float4 s = s_pts[fps_pos(best)];
      const int id = __float_as_int(s.w);
      if (j == K - 1 || fps_settled(best)) {
        for (int jj = j + t; jj < K; jj += T) row[jj] = id;
        break;
      }
      if (t == 0) row[j] = id;
      best = group_max(fps_sweep<T>(p, t, s.x, s.y, s.z));
    }
  }
}

// streaming: positions first, first + kFpsCtaThreads, ... below `end`, points read from global memory, d from dws
// (written, not read, on the first update, where the old d is +inf)
__device__ __forceinline__ unsigned long long fps_stream_sweep(const int32_t *__restrict__ ids, long long start, int first, int end,
                                                               int N, const float *__restrict__ xyz, long long ld,
                                                               float *__restrict__ dws, bool first_update, float sx, float sy,
                                                               float sz) {
  constexpr int B = 4;  // loads in flight per thread
  unsigned long long best = 0;
  for (int pos0 = first; pos0 < end; pos0 += B * kFpsCtaThreads) {
    int id[B];
    float x[B], y[B], z[B], d[B];
#pragma unroll
    for (int b = 0; b < B; b++) {
      const int pos = pos0 + b * kFpsCtaThreads;
      id[b] = pos < end ? __ldg(&ids[start + pos]) : -1;
    }
#pragma unroll
    for (int b = 0; b < B; b++) {
      x[b] = y[b] = z[b] = 0.f;
      d[b] = INFINITY;
      if ((unsigned)id[b] < (unsigned)N) {
        const float *q = xyz + (size_t)id[b] * ld;
        x[b] = __ldg(q);
        y[b] = __ldg(q + 1);
        z[b] = __ldg(q + 2);
        if (!first_update) d[b] = __ldcg(&dws[start + pos0 + b * kFpsCtaThreads]);
      }
    }
#pragma unroll
    for (int b = 0; b < B; b++) {
      if ((unsigned)id[b] < (unsigned)N) {
        const int pos = pos0 + b * kFpsCtaThreads;
        d[b] = fps_min(d[b], fps_dist(x[b], y[b], z[b], sx, sy, sz));
        __stcg(&dws[start + pos], d[b]);
        best = umax64(best, fps_key(d[b], pos));
      }
    }
  }
  return best;
}

// the smallest valid position of first, first + kFpsCtaThreads, ... below `end`, as a key with d = +inf (0 if none)
__device__ __forceinline__ unsigned long long fps_stream_first(const int32_t *__restrict__ ids, long long start, int first, int end,
                                                               int N) {
  for (int pos = first; pos < end; pos += kFpsCtaThreads)
    if ((unsigned)__ldg(&ids[start + pos]) < (unsigned)N) return fps_key(INFINITY, pos);
  return 0ull;
}

__device__ __forceinline__ void fps_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t fps_cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t fps_mapa(const void *p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(rank));
  return r;
}

struct alignas(16) FpsPick {
  float x, y, z;
  int id;
  unsigned long long key;
};

// Cluster path: one list per 8-CTA cluster, CTA r owns the positions [r * slice, (r + 1) * slice). Per step each CTA
// publishes its best (key, x, y, z, id) in its own shared memory (double-buffered), one barrier.cluster, then lanes 0..7
// of every warp read the 8 candidates through distributed shared memory and reduce them identically.
__global__ void __cluster_dims__(kFpsCl, 1, 1) __launch_bounds__(kFpsCtaThreads, 1)
    fps_cluster_kernel(const long long *__restrict__ off, const int32_t *__restrict__ ids, long long total, int N,
                       const float *__restrict__ xyz, long long ld, int K, const int32_t *__restrict__ queue,
                       const int *__restrict__ count, int *head, float *__restrict__ dws, int32_t *__restrict__ out) {
  extern __shared__ float4 s_pts[];  // [SGB_FPS_CTA_MAX]
  __shared__ unsigned long long s_cand[2][kFpsCtaWarps];
  __shared__ FpsPick s_pub[2];
  __shared__ int s_item;
  const int t = threadIdx.x, lane = lane_id();
  const uint32_t crank = fps_cluster_rank();
  const int n_items = *count;
  int phase = 0, cphase = 0;
  FpsRegs p;
  while (true) {
    if (crank == 0 && t == 0) s_item = atomicAdd(head, 1);
    fps_cluster_sync();
    int item;
    asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(item) : "r"(fps_mapa(&s_item, 0)) : "memory");
    if (item >= n_items) break;
    const int k = queue[item];
    long long start;
    const int len = fps_list(off, k, total, start);
    const int slice = (len + kFpsCl - 1) / kFpsCl;
    const int a = (int)crank * slice, b = min(a + slice, len);
    const bool stream = len > SGB_FPS_CLUSTER_MAX;
    int32_t *row = out + (size_t)k * K;
    auto pick = [&](unsigned long long v) {
      v = cta_max_u64(v, s_cand, phase);
      FpsPick *pub = &s_pub[cphase++ & 1];
      if (t == 0) {
        FpsPick m{0.f, 0.f, 0.f, -1, v};
        if (v) {
          const int pos = fps_pos(v);
          if (!stream) {
            const float4 s = s_pts[pos - a];
            m.x = s.x, m.y = s.y, m.z = s.z, m.id = __float_as_int(s.w);
          } else {
            m.id = __ldg(&ids[start + pos]);
            const float *q = xyz + (size_t)m.id * ld;
            m.x = __ldg(q), m.y = __ldg(q + 1), m.z = __ldg(q + 2);
          }
        }
        *pub = m;
      }
      fps_cluster_sync();
      unsigned long long key = 0ull;
      float x = 0.f, y = 0.f, z = 0.f, id = 0.f;
      if (lane < kFpsCl) {
        const uint32_t r = fps_mapa(pub, lane);
        asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x), "=f"(y), "=f"(z), "=f"(id) : "r"(r) : "memory");
        asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(key) : "r"(r + 16) : "memory");
      }
      const unsigned long long top = warp_max_u64(key);
      const int src = __ffs(__ballot_sync(0xffffffffu, lane < kFpsCl && key == top)) - 1;
      return FpsPick{__shfl_sync(0xffffffffu, x, src), __shfl_sync(0xffffffffu, y, src), __shfl_sync(0xffffffffu, z, src),
                     __float_as_int(__shfl_sync(0xffffffffu, id, src)), top};
    };
    FpsPick s = pick(stream ? fps_stream_first(ids, start, a + t, b, N)
                            : fps_load<kFpsCtaThreads>(p, ids, start, a + t, b, N, xyz, ld, s_pts, t));
    const int ct = (int)crank * kFpsCtaThreads + t;  // thread rank in the cluster
    if (s.key == 0) {
      for (int j = ct; j < K; j += kFpsCl * kFpsCtaThreads) row[j] = -1;
      continue;
    }
    for (int j = 0;; j++) {
      if (j == K - 1 || fps_settled(s.key)) {
        for (int jj = j + ct; jj < K; jj += kFpsCl * kFpsCtaThreads) row[jj] = s.id;
        break;
      }
      if (ct == 0) row[j] = s.id;
      s = pick(stream ? fps_stream_sweep(ids, start, a + t, b, N, xyz, ld, dws, j == 0, s.x, s.y, s.z)
                      : fps_sweep<kFpsCtaThreads>(p, a + t, s.x, s.y, s.z));
    }
  }
  fps_cluster_sync();  // no CTA leaves while another may still read its shared memory
}

// lists -> queues[q][0 .. counts[q]): q = 0 for lengths up to SGB_FPS_WARP_MAX (and lengths with no position), 1 up to
// SGB_FPS_CTA_MAX, 2 beyond. One atomic per warp and queue.
__global__ void fps_bin_kernel(const long long *__restrict__ off, int n, long long total, int *__restrict__ counts,
                               int32_t *__restrict__ queues) {
  const int lane = lane_id();
  for (long long base = (long long)blockIdx.x * blockDim.x; base < n; base += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(base + threadIdx.x);
    int q = -1;
    if (k < n) {
      long long start;
      const int len = fps_list(off, k, total, start);
      q = len <= SGB_FPS_WARP_MAX ? 0 : (len <= SGB_FPS_CTA_MAX ? 1 : 2);
    }
    const unsigned peers = __match_any_sync(0xffffffffu, q);
    const int leader = __ffs(peers) - 1;
    int slot = 0;
    if (lane == leader && q >= 0) slot = atomicAdd(&counts[q], __popc(peers));
    slot = __shfl_sync(0xffffffffu, slot, leader) + __popc(peers & ((1u << lane) - 1u));
    if (q >= 0) queues[(size_t)q * n + slot] = k;
  }
}

// per device: dynamic shared memory of the three list kernels and their resident grids
static DeviceOnce g_fps_once;
static int g_fps_grid[kMaxDevices][3];
constexpr size_t kFpsWarpSmem = (size_t)kFpsWarpLists * SGB_FPS_WARP_MAX * sizeof(float4);
constexpr size_t kFpsCtaSmem = (size_t)SGB_FPS_CTA_MAX * sizeof(float4);

static int fps_setup(Device *d) {
  return once_per_device(g_fps_once, d->ordinal, [d] {
    SGB_CUDA_CHECK(cudaFuncSetAttribute(fps_lists_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFpsWarpSmem));
    SGB_CUDA_CHECK(cudaFuncSetAttribute(fps_lists_kernel<kFpsCtaThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)kFpsCtaSmem));
    SGB_CUDA_CHECK(cudaFuncSetAttribute(fps_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFpsCtaSmem));
    int b0 = 0, b1 = 0, nc = 0;
    SGB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b0, fps_lists_kernel<32>, 32 * kFpsWarpLists, kFpsWarpSmem));
    SGB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b1, fps_lists_kernel<kFpsCtaThreads>, kFpsCtaThreads,
                                                                 kFpsCtaSmem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(d->sms / kFpsCl * kFpsCl);
    cfg.blockDim = dim3(kFpsCtaThreads);
    cfg.dynamicSmemBytes = kFpsCtaSmem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kFpsCl;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    SGB_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&nc, fps_cluster_kernel, &cfg));
    SGB_REQUIRE(b0 >= 1 && b1 >= 1 && nc >= 1, SGB_ERR_CUDA, "id_lists_fps kernels do not fit on this device");
    g_fps_grid[d->ordinal][0] = b0 * d->sms;
    g_fps_grid[d->ordinal][1] = b1 * d->sms;
    g_fps_grid[d->ordinal][2] = nc * kFpsCl;
    return SGB_OK;
  });
}

}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_inst_count(const int32_t *d_proposals_idx, const float *d_mask_scores, int ms_stride, int S, int nI, float thr,
                   int32_t *d_npoint, int nP, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(S >= 0 && nI >= 0 && nP >= 0 && d_npoint, SGB_ERR_ARG, "inst_count arguments");
  SGB_CUDA_CHECK(cudaMemsetAsync(d_npoint, 0, (size_t)nP * nI * 4, st));
  if (S == 0 || nI == 0) return SGB_OK;
  SGB_REQUIRE(d_proposals_idx && d_mask_scores && ms_stride >= nI, SGB_ERR_ARG, "inst_count pointers");
  inst_count_kernel<<<div_up(S, 256), 256, 0, st>>>(d_proposals_idx, d_mask_scores, ms_stride, S, nI, thr, d_npoint);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

size_t sgb_bitmap_words(int N) { return (size_t)(N + 1 + 31) / 32; }

int sgb_inst_scatter(const int32_t *d_proposals_idx, const float *d_mask_scores, int ms_stride, int S, int nI, int nP, float thr,
                     const int32_t *d_slot, uint32_t *d_bitmaps, int n_inst, int N, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int W = (int)sgb_bitmap_words(N);
  SGB_REQUIRE(S >= 0 && n_inst >= 0 && N >= 0, SGB_ERR_ARG, "inst_scatter arguments");
  if (n_inst == 0) return SGB_OK;
  SGB_REQUIRE(d_bitmaps, SGB_ERR_ARG, "null bitmaps");
  SGB_CUDA_CHECK(cudaMemsetAsync(d_bitmaps, 0, (size_t)n_inst * W * 4, st));
  if (S == 0 || nI == 0) return SGB_OK;
  SGB_REQUIRE(d_proposals_idx && d_mask_scores && d_slot, SGB_ERR_ARG, "inst_scatter pointers");
  inst_scatter_kernel<<<div_up(S, 256), 256, 0, st>>>(d_proposals_idx, d_mask_scores, ms_stride, S, nI, nP, thr, d_slot, d_bitmaps, W);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_bitmap_set(const int32_t *d_row, const int32_t *d_pt, long long n, uint32_t *d_bitmaps, int n_rows, int N, int clear,
                   void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int W = (int)sgb_bitmap_words(N);
  SGB_REQUIRE(n >= 0 && n_rows >= 0 && (n_rows == 0 || d_bitmaps), SGB_ERR_ARG, "bitmap_set arguments");
  if (clear && n_rows) SGB_CUDA_CHECK(cudaMemsetAsync(d_bitmaps, 0, (size_t)n_rows * W * 4, st));
  if (n == 0) return SGB_OK;
  SGB_REQUIRE(d_row && d_pt, SGB_ERR_ARG, "bitmap_set pointers");
  bitmap_set_kernel<<<div_up(n, 256), 256, 0, st>>>(d_row, d_pt, n, d_bitmaps, W);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

size_t sgb_rle_workspace_bytes(int n_inst, int N) {
  const size_t tot = (size_t)std::max(n_inst, 0) * sgb_bitmap_words(N) + 1;
  return align_up(tot * 4) + align_up(scan_temp_elems(tot) * 4) + align_up(64) + 1024;
}

// count (blocking): returns the number of transitions of all masks (2 per run), or < 0.
long long sgb_rle_count(const uint32_t *d_bitmaps, int n_inst, int N, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n_inst == 0) return 0;
  const int W = (int)sgb_bitmap_words(N);
  const long long total = (long long)n_inst * W;
  SGB_REQUIRE(total < (1ll << 31), SGB_ERR_RANGE, "rle: n_inst * words must stay below 2^31");
  Arena a(d_ws, ws_bytes);
  int32_t *cnt = a.take<int32_t>((size_t)total + 1);
  int32_t *tmp = a.take<int32_t>(scan_temp_elems((size_t)total + 1));
  int32_t *tot_d = a.take<int32_t>(16);
  SGB_REQUIRE(d_bitmaps && cnt && tmp && tot_d, SGB_ERR_WORKSPACE, "rle workspace too small");
  rle_count_kernel<<<div_up(total, 256), 256, 0, st>>>(d_bitmaps, W, total, cnt);
  SGB_LAUNCH_CHECK();
  int rc = exclusive_scan_i32(cnt, cnt, (size_t)total, tot_d, tmp, st);
  if (rc) return rc;
  int h = 0;
  SGB_CUDA_CHECK(cudaMemcpyAsync(&h, tot_d, 4, cudaMemcpyDeviceToHost, st));
  SGB_CUDA_CHECK(cudaStreamSynchronize(st));
  return h;
}

// fill: after sgb_rle_count on the same workspace. d_trans int32 [total], d_inst_off int32 [n_inst + 1].
int sgb_rle_fill(const uint32_t *d_bitmaps, int n_inst, int N, int total_trans, int32_t *d_trans, int32_t *d_inst_off, void *d_ws,
                 size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(d_inst_off, SGB_ERR_ARG, "null inst_off");
  if (n_inst == 0) { SGB_CUDA_CHECK(cudaMemsetAsync(d_inst_off, 0, 4, st)); return SGB_OK; }
  const int W = (int)sgb_bitmap_words(N);
  const long long total = (long long)n_inst * W;
  Arena a(d_ws, ws_bytes);
  int32_t *off = a.take<int32_t>((size_t)total + 1);
  SGB_REQUIRE(d_bitmaps && off && (total_trans == 0 || d_trans), SGB_ERR_WORKSPACE, "rle workspace too small");
  rle_fill_kernel<<<div_up(total, 256), 256, 0, st>>>(d_bitmaps, W, total, off, d_trans, d_inst_off, n_inst, total_trans);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

// Host-side formatter: transitions (1-based positions, ascending per mask; offsets int32 [n+1]) -> "start len ..." strings.
long long sgb_rle_format_runs(const int32_t *h_trans, const int32_t *h_offs, int n_masks, char *h_out, long long out_cap,
                              long long *h_out_offs) {
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
    const int a = h_offs[m], b = h_offs[m + 1];
    if ((b - a) & 1) { set_error("sgb_rle_format_runs: odd number of transitions in mask %d", m); return SGB_ERR_ARG; }
    for (int i = a; i < b; i += 2) {
      if (end - p < 48) { set_error("sgb_rle_format_runs: output buffer too small"); return SGB_ERR_OVERFLOW; }
      if (i > a) *p++ = ' ';
      p = put(p, (long long)h_trans[i]);
      *p++ = ' ';
      p = put(p, (long long)h_trans[i + 1] - h_trans[i]);
    }
  }
  h_out_offs[n_masks] = p - h_out;
  return p - h_out;
}

// Prediction x ground-truth intersections (instance_eval.py:262-293). d_gslot int32 [N]: column of the point's gt
// instance (>= 0), -2 = void label (counted in d_void), -1 = neither. Outputs are zeroed here.
int sgb_bitmap_intersections(const uint32_t *d_bitmaps, int n_rows, int N, const int32_t *d_gslot, int nG, int32_t *d_inter,
                             int32_t *d_vert, int32_t *d_void, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n_rows >= 0 && N >= 0 && nG >= 0, SGB_ERR_ARG, "bitmap_intersections arguments");
  if (n_rows == 0) return SGB_OK;
  SGB_REQUIRE(d_bitmaps && d_gslot && d_vert && d_void && (nG == 0 || d_inter), SGB_ERR_ARG, "bitmap_intersections pointers");
  if (nG) SGB_CUDA_CHECK(cudaMemsetAsync(d_inter, 0, (size_t)n_rows * nG * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(d_vert, 0, (size_t)n_rows * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(d_void, 0, (size_t)n_rows * 4, st));
  const int W = (int)sgb_bitmap_words(N);
  bitmap_hist_kernel<<<div_up((long long)n_rows * W, 256), 256, 0, st>>>(d_bitmaps, W, n_rows, N, d_gslot, nG, d_inter, d_vert, d_void);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

// panoptic_fusion on bitmaps. d_order int32 [n_inst]: instance rows in descending confidence (the caller sorts: numpy
// argsort()[::-1] order must be reproduced by the caller); d_cls int32 [n_rows]: class value to paste (label_id + offset).
// d_pan_cls must hold the semantic predictions on entry (uint32 [N]), d_pan_ids zeros; d_prev uint32 [W] scratch.
int sgb_panoptic_paste(const uint32_t *d_bitmaps, int N, const int32_t *d_order, const int32_t *d_cls, int n_inst, double skip_iou,
                       uint32_t *d_prev, uint32_t *d_pan_cls, uint32_t *d_pan_ids, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n_inst >= 0 && N >= 0, SGB_ERR_ARG, "panoptic_paste arguments");
  if (n_inst == 0 || N == 0) return SGB_OK;
  SGB_REQUIRE(d_bitmaps && d_order && d_cls && d_prev && d_pan_cls && d_pan_ids, SGB_ERR_ARG, "panoptic_paste pointers");
  const int W = (int)sgb_bitmap_words(N);
  SGB_CUDA_CHECK(cudaMemsetAsync(d_prev, 0, (size_t)W * 4, st));
  panoptic_paste_kernel<<<1, kPanThreads, 0, st>>>(d_bitmaps, W, N, d_order, d_cls, n_inst, skip_iou, d_prev, d_pan_cls, d_pan_ids);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

static long long id_segments(int n_rows, int N) {
  return (long long)std::max(n_rows, 0) * div_up((long long)sgb_bitmap_words(N), kIdSegWords);
}

size_t sgb_bitmap_ids_workspace_bytes(int n_rows, int N) {
  const size_t n = (size_t)id_segments(n_rows, N) + 1;
  return align_up(n * 8) + align_up(scan_temp_elems(n) * 8) + 1024;
}

// Count pass: d_offsets int64 [n_rows + 1] = exclusive prefix of the rows' set bits (bits < N); d_offsets[n_rows] is the
// total. No host wait. The per-segment offsets stay in the workspace for sgb_bitmap_ids_fill.
int sgb_bitmap_ids_count(const uint32_t *d_bitmaps, int n_rows, int N, long long *d_offsets, void *d_ws, size_t ws_bytes,
                         void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n_rows >= 0 && N >= 0 && d_offsets, SGB_ERR_ARG, "bitmap_ids_count arguments");
  if (n_rows == 0) { SGB_CUDA_CHECK(cudaMemsetAsync(d_offsets, 0, 8, st)); return SGB_OK; }
  const int W = (int)sgb_bitmap_words(N);
  const int B = div_up(W, kIdSegWords);
  const long long n_seg = id_segments(n_rows, N);
  SGB_REQUIRE(n_seg < (1ll << 31), SGB_ERR_RANGE, "bitmap_ids: rows * segments must stay below 2^31");
  Arena a(d_ws, ws_bytes);
  long long *seg = a.take<long long>((size_t)n_seg + 1);
  long long *tmp = a.take<long long>(scan_temp_elems((size_t)n_seg + 1));
  SGB_REQUIRE(d_bitmaps && seg && tmp, SGB_ERR_WORKSPACE, "bitmap_ids workspace too small");
  bitmap_ids_count_kernel<<<div_up(n_seg, kIdSegsPerCta), kIdThreads, 0, st>>>(d_bitmaps, W, N, B, n_seg, seg);
  SGB_LAUNCH_CHECK();
  const int rc = exclusive_scan_i64(seg, seg, (size_t)n_seg, seg + n_seg, tmp, st);
  if (rc) return rc;
  bitmap_row_offsets_kernel<<<div_up((long long)n_rows + 1, 256), 256, 0, st>>>(seg, B, n_rows, d_offsets);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

// Fill pass, after sgb_bitmap_ids_count on the same workspace and stream: d_ids int32 [total], the ids of row r
// ascending at [offsets[r], offsets[r + 1]).
int sgb_bitmap_ids_fill(const uint32_t *d_bitmaps, int n_rows, int N, int32_t *d_ids, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n_rows >= 0 && N >= 0, SGB_ERR_ARG, "bitmap_ids_fill arguments");
  if (n_rows == 0) return SGB_OK;
  const int W = (int)sgb_bitmap_words(N);
  const int B = div_up(W, kIdSegWords);
  const long long n_seg = id_segments(n_rows, N);
  SGB_REQUIRE(n_seg < (1ll << 31), SGB_ERR_RANGE, "bitmap_ids: rows * segments must stay below 2^31");
  Arena a(d_ws, ws_bytes);
  const long long *seg = a.take<long long>((size_t)n_seg + 1);
  SGB_REQUIRE(d_bitmaps && d_ids && seg, SGB_ERR_WORKSPACE, "bitmap_ids workspace too small");
  bitmap_ids_fill_kernel<<<(unsigned)n_seg, kIdThreads, 0, st>>>(d_bitmaps, W, N, B, seg, d_ids);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

// Class bitmaps (zeroed here): d_bitmaps uint32 [n_rows][W]; row d_row_of_label[l] (or -1) for label l in [0, n_labels);
// labels outside that range set no bit. d_counts int64 [n_rows] (may be null) receives the rows' set bits.
int sgb_class_bitmaps(const int64_t *d_labels, int N, const int32_t *d_row_of_label, int n_labels, uint32_t *d_bitmaps, int n_rows,
                      long long *d_counts, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(N >= 0 && n_labels >= 0 && n_rows >= 0, SGB_ERR_ARG, "class_bitmaps arguments");
  if (n_rows == 0) return SGB_OK;
  SGB_REQUIRE(d_bitmaps, SGB_ERR_ARG, "null bitmaps");
  const int W = (int)sgb_bitmap_words(N);
  SGB_CUDA_CHECK(cudaMemsetAsync(d_bitmaps, 0, (size_t)n_rows * W * 4, st));
  if (d_counts) SGB_CUDA_CHECK(cudaMemsetAsync(d_counts, 0, (size_t)n_rows * 8, st));
  if (N == 0 || n_labels == 0) return SGB_OK;
  SGB_REQUIRE(d_labels && d_row_of_label, SGB_ERR_ARG, "class_bitmaps pointers");
  class_bitmaps_kernel<<<div_up(N, 256), 256, 0, st>>>(d_labels, N, d_row_of_label, n_labels, d_bitmaps, W, d_counts);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

static long long list_chunks(long long total) { return (std::max(total, 0ll) + kListChunk - 1) / kListChunk; }

// grid of the chunk passes: one warp per chunk, as many CTAs as are resident at once (the warps loop over the rest)
static int list_chunk_grid(long long total, int sms) {
  return (int)std::min<long long>(div_up(list_chunks(total), kListWarps), (long long)kListCtasPerSm * sms);
}

size_t sgb_id_lists_reduce_workspace_bytes(long long total, int C) {
  const size_t slots = 2 * (size_t)list_chunks(total), sc = slots * (size_t)std::max(C, 0);
  return align_up(sc * 8) + 2 * align_up(sc * 4) + align_up(slots * 4) + 1024;
}

int sgb_id_lists_reduce(const long long *d_offsets, const int32_t *d_ids, int n, long long total, int N, const float *d_values,
                        long long ld, int C, int ops, float *d_min, float *d_max, float *d_mean, long long *d_counts, void *d_ws,
                        size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n >= 0 && total >= 0 && N >= 0 && C >= 1 && ld >= C, SGB_ERR_ARG, "id_lists_reduce sizes");
  SGB_REQUIRE(ops > 0 && (ops & ~(SGB_REDUCE_MIN | SGB_REDUCE_MAX | SGB_REDUCE_MEAN)) == 0, SGB_ERR_ARG, "id_lists_reduce ops");
  if (n == 0) return SGB_OK;
  SGB_REQUIRE((!(ops & SGB_REDUCE_MIN) || d_min) && (!(ops & SGB_REDUCE_MAX) || d_max) && (!(ops & SGB_REDUCE_MEAN) || d_mean),
              SGB_ERR_ARG, "id_lists_reduce: null output for a requested op");
  SGB_REQUIRE(d_offsets && d_counts && (total == 0 || (d_ids && (N == 0 || d_values))), SGB_ERR_ARG, "id_lists_reduce pointers");
  SGB_CURRENT_DEVICE(d);
  const size_t sc = 2 * (size_t)list_chunks(total) * C;
  Arena a(d_ws, ws_bytes);
  double *psum = a.take<double>(sc);
  float *pmin = a.take<float>(sc), *pmax = a.take<float>(sc);
  int32_t *pcnt = a.take<int32_t>(2 * (size_t)list_chunks(total));
  SGB_REQUIRE(psum && pmin && pmax && pcnt, SGB_ERR_WORKSPACE, "id_lists_reduce workspace too small");
  if (total > 0) {
    id_reduce_chunks_kernel<<<list_chunk_grid(total, d->sms), kListThreads, 0, st>>>(
        d_offsets, n, d_ids, total, N, d_values, ld, C, ops, d_min, d_max, d_mean, d_counts, psum, pmin, pmax, pcnt);
    SGB_LAUNCH_CHECK();
  }
  id_reduce_lists_kernel<<<std::min(n, 8 * d->sms), kListThreads, 0, st>>>(d_offsets, n, total, C, ops, psum, pmin, pmax, pcnt,
                                                                          d_min, d_max, d_mean, d_counts);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

size_t sgb_id_lists_point_map_workspace_bytes(int N) { return align_up((size_t)std::max(N, 0) * 8) + 1024; }

int sgb_id_lists_point_map(const long long *d_offsets, const int32_t *d_ids, int n, long long total, int N, const float *d_conf,
                           int32_t *d_map, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n >= 0 && total >= 0 && N >= 0, SGB_ERR_ARG, "id_lists_point_map sizes");
  if (N == 0) return SGB_OK;
  SGB_REQUIRE(d_map && (n == 0 || total == 0 || (d_offsets && d_ids && d_conf)), SGB_ERR_ARG, "id_lists_point_map pointers");
  SGB_CURRENT_DEVICE(d);
  Arena a(d_ws, ws_bytes);
  unsigned long long *key = a.take<unsigned long long>((size_t)N);
  SGB_REQUIRE(key, SGB_ERR_WORKSPACE, "id_lists_point_map workspace too small");
  SGB_CUDA_CHECK(cudaMemsetAsync(key, 0, (size_t)N * 8, st));
  if (n > 0 && total > 0) {
    id_map_keys_kernel<<<list_chunk_grid(total, d->sms), kListThreads, 0, st>>>(d_offsets, n, d_ids, total, N, d_conf, key);
    SGB_LAUNCH_CHECK();
  }
  id_map_decode_kernel<<<div_up(N, 256), 256, 0, st>>>(key, N, d_map);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

size_t sgb_id_lists_fps_workspace_bytes(int n, long long total) {
  return align_up(16 * 4) + align_up(3 * (size_t)std::max(n, 0) * 4) + align_up((size_t)std::max(total, 0ll) * 4);
}

int sgb_id_lists_fps(const long long *d_offsets, const int32_t *d_ids, int n, long long total, int N, const float *d_xyz,
                     long long ld, int K, int32_t *d_out, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(n >= 0 && total >= 0 && N >= 0 && K >= 1 && ld >= 3, SGB_ERR_ARG, "id_lists_fps sizes");
  if (n == 0) return SGB_OK;
  SGB_REQUIRE(d_offsets && d_out && (total == 0 || d_ids) && (N == 0 || d_xyz), SGB_ERR_ARG, "id_lists_fps pointers");
  SGB_CURRENT_DEVICE(d);
  if (const int rc = fps_setup(d)) return rc;
  Arena a(d_ws, ws_bytes);
  int *counters = a.take<int>(16);  // counts[3], heads[3]
  int32_t *queues = a.take<int32_t>(3 * (size_t)n);
  float *dws = a.take<float>((size_t)total);
  SGB_REQUIRE(counters && queues && dws, SGB_ERR_WORKSPACE, "id_lists_fps workspace too small");
  const int *g = g_fps_grid[d->ordinal];
  SGB_CUDA_CHECK(cudaMemsetAsync(counters, 0, 6 * 4, st));
  fps_bin_kernel<<<std::min(div_up(n, 256), 4 * d->sms), 256, 0, st>>>(d_offsets, n, total, counters, queues);
  SGB_LAUNCH_CHECK();
  fps_cluster_kernel<<<g[2], kFpsCtaThreads, kFpsCtaSmem, st>>>(d_offsets, d_ids, total, N, d_xyz, ld, K, queues + 2 * (size_t)n,
                                                              counters + 2, counters + 5, dws, d_out);
  SGB_LAUNCH_CHECK();
  fps_lists_kernel<kFpsCtaThreads><<<g[1], kFpsCtaThreads, kFpsCtaSmem, st>>>(d_offsets, d_ids, total, N, d_xyz, ld, K,
                                                                             queues + (size_t)n, counters + 1, counters + 4, d_out);
  SGB_LAUNCH_CHECK();
  fps_lists_kernel<32><<<g[0], 32 * kFpsWarpLists, kFpsWarpSmem, st>>>(d_offsets, d_ids, total, N, d_xyz, ld, K, queues,
                                                                        counters, counters + 3, d_out);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
}
