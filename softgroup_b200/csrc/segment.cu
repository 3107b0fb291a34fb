// segment.cu -- segmented reductions over contiguous row segments and the mask-IoU ops.
//
// Replaces sec_mean/sec_min/sec_max (softgroup/ops/src/sec_mean/sec_mean.cu:13-93: one 32-thread block per
// proposal, serial loop), global_avg_pool_fp/bp (roipool/roipool.cu:12-72) and get_mask_iou_* / get_mask_label
// (cal_iou_and_masklabel/cal_iou_and_masklabel.cu:9-164: O(nInstance * len) rescans per proposal).
// Here: reads are coalesced over the channel dimension. min/max (order independent, exact): the ROW SPACE is cut into
// 2048-row chunks spread over a machine-filling grid, a chunk is split at proposal boundaries, and the per-chunk partial
// of every (proposal, channel) is combined with one atomic min/max on the sign-aware integer image of the float
// (seg_minmax_kernel) -- 40 long proposals no longer mean 40 busy SMs. mean/avg: one CTA per proposal, shared-memory
// tree (error bound in include/sgb200.h).
#include <float.h>

#include "common.cuh"

namespace sgb {

enum { OP_MEAN = 0, OP_MIN = 1, OP_MAX = 2, OP_AVG = 3 };

constexpr int kSegThreads = 256;

// One CTA per proposal. Threads: tx = channel lane (Cw = pow2 >= min(C,32)), ty = row lane.
template <int OP>
__global__ void __launch_bounds__(kSegThreads) seg_reduce_kernel(const float *__restrict__ inp,
                                                                 const int32_t *__restrict__ offsets,
                                                                 float *__restrict__ out, int nProposal, int C, int Cw) {
  __shared__ float red[kSegThreads];
  const int rows_par = kSegThreads / Cw;
  const int tx = threadIdx.x % Cw, ty = threadIdx.x / Cw;
  for (int p = blockIdx.x; p < nProposal; p += gridDim.x) {
    const int s = offsets[p], e = offsets[p + 1];
    const float count = (float)(e - s);
    for (int c0 = 0; c0 < C; c0 += Cw) {
      const int c = c0 + tx;
      float acc = (OP == OP_MIN) ? INFINITY : (OP == OP_MAX) ? -INFINITY : 0.f;
      if (c < C) {
        for (int i = s + ty; i < e; i += rows_par) {
          float x = __ldg(&inp[(size_t)i * C + c]);
          if (OP == OP_MIN) acc = (x < acc) ? x : acc;
          else if (OP == OP_MAX) acc = (x > acc) ? x : acc;
          else if (OP == OP_MEAN) acc += __fdiv_rn(x, count);  // sec_mean.cu:23-25 divides every term
          else acc += x;                                       // roipool.cu:23-29 divides after the sum
        }
      }
      red[threadIdx.x] = acc;
      __syncthreads();
      for (int h = rows_par >> 1; h > 0; h >>= 1) {
        if (ty < h) {
          float a = red[threadIdx.x], b = red[threadIdx.x + h * Cw];
          if (OP == OP_MIN) a = (b < a) ? b : a;
          else if (OP == OP_MAX) a = (b > a) ? b : a;
          else a += b;
          red[threadIdx.x] = a;
        }
        __syncthreads();
      }
      if (ty == 0 && c < C) {
        float r = red[tx];
        if (OP == OP_AVG) r = __fdiv_rn(r, count);
        out[(size_t)p * C + c] = r;
      }
      __syncthreads();
    }
  }
}

// ---- chunked min / max -------------------------------------------------------------------------------------------
constexpr int kSegChunk = 2048;

// The branch is chosen by the sign BIT, not by `v >= 0.f` (true for -0.0, whose int image is INT_MIN): floats with the
// sign bit clear are ordered like their int images, floats with it set are ordered inversely to their unsigned images,
// and every sign-clear image is below every sign-set one as unsigned and above it as signed. So a signed atomicMin /
// atomicMax for sign-clear values and an unsigned atomicMax / atomicMin for sign-set values order any mix correctly
// (-0.0 sorts just below +0.0, which only decides the sign of a zero result).
__device__ __forceinline__ void atomic_min_f32(float *addr, float v) {  // *addr starts at +inf; NaN never gets here
  if (__float_as_int(v) >= 0) atomicMin(reinterpret_cast<int *>(addr), __float_as_int(v));
  else atomicMax(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_f32(float *addr, float v) {  // *addr starts at -inf
  if (__float_as_int(v) >= 0) atomicMax(reinterpret_cast<int *>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v));
}

__global__ void seg_fill_kernel(float *__restrict__ out, long long n, float v) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v;
}

template <int OP>
__global__ void __launch_bounds__(kSegThreads) seg_minmax_kernel(const float *__restrict__ inp, const int32_t *__restrict__ offsets,
                                                                 float *__restrict__ out, int nProposal, int C, int Cw) {
  __shared__ float red[kSegThreads];
  const int rows_par = kSegThreads / Cw;
  const int tx = threadIdx.x % Cw, ty = threadIdx.x / Cw;
  const int S = offsets[nProposal];
  const int first = offsets[0];  // rows below offsets[0] belong to no proposal
  for (long long r0l = (long long)blockIdx.x * kSegChunk; r0l < S; r0l += (long long)gridDim.x * kSegChunk) {
    const int r1 = min((int)r0l + kSegChunk, S);
    int r0 = max((int)r0l, first);
    // proposal holding row r0: last p with offsets[p] <= r0
    int lo = 0, hi = nProposal;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (offsets[mid] <= r0) lo = mid; else hi = mid;
    }
    int p = lo;
    while (r0 < r1) {
      while (offsets[p + 1] <= r0) p++;  // skip empty proposals
      const int e = min(offsets[p + 1], r1);
      for (int c0 = 0; c0 < C; c0 += Cw) {
        const int c = c0 + tx;
        float acc = (OP == OP_MIN) ? INFINITY : -INFINITY;
        if (c < C)
          for (int i = r0 + ty; i < e; i += rows_par) {
            const float x = __ldg(&inp[(size_t)i * C + c]);
            if (OP == OP_MIN) acc = (x < acc) ? x : acc;  // same comparison as sec_mean.cu:50 / :76 (NaN never wins)
            else acc = (x > acc) ? x : acc;
          }
        red[threadIdx.x] = acc;
        __syncthreads();
        for (int h = rows_par >> 1; h > 0; h >>= 1) {
          if (ty < h) {
            float a = red[threadIdx.x];
            const float b = red[threadIdx.x + h * Cw];
            if (OP == OP_MIN) a = (b < a) ? b : a; else a = (b > a) ? b : a;
            red[threadIdx.x] = a;
          }
          __syncthreads();
        }
        if (ty == 0 && c < C) {
          const float r = red[tx];
          if (OP == OP_MIN) { if (r < INFINITY) atomic_min_f32(&out[(size_t)p * C + c], r); }
          else { if (r > -INFINITY) atomic_max_f32(&out[(size_t)p * C + c], r); }
        }
        __syncthreads();
      }
      r0 = e;
    }
  }
}

__global__ void avg_pool_bp_kernel(float *__restrict__ d_feats, const int32_t *__restrict__ offsets,
                                   const float *__restrict__ d_out, int nProposal, int C) {
  for (int p = blockIdx.x; p < nProposal; p += gridDim.x) {
    int s = offsets[p], e = offsets[p + 1];
    float n = (float)(e - s);
    long long tot = (long long)(e - s) * C;
    for (long long t = threadIdx.x; t < tot; t += blockDim.x) {
      int i = s + (int)(t / C), c = (int)(t % C);
      d_feats[(size_t)i * C + c] += __fdiv_rn(d_out[(size_t)p * C + c], n);  // roipool.cu:54-57
    }
  }
}

// IoU: one CTA per proposal, shared-memory histogram of instance labels over the proposal's points.
__global__ void mask_iou_kernel(const int32_t *__restrict__ pidx, const int32_t *__restrict__ poff,
                                const long long *__restrict__ inst_labels, const int32_t *__restrict__ inst_pointnum,
                                const float *__restrict__ mask_sig, float *__restrict__ iou, int nInstance,
                                int nProposal) {
  extern __shared__ int hist[];
  __shared__ int s_total;
  for (int p = blockIdx.x; p < nProposal; p += gridDim.x) {
    for (int q = threadIdx.x; q < nInstance; q += blockDim.x) hist[q] = 0;
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    int s = poff[p], e = poff[p + 1];
    int local_total = 0;
    for (int i = s + threadIdx.x; i < e; i += blockDim.x) {
      bool on = mask_sig ? (mask_sig[i] > 0.5f) : true;  // `> 0.5` double literal == float compare for 0.5
      if (on) {
        local_total++;
        int lab = (int)inst_labels[pidx[i]];
        if (lab >= 0 && lab < nInstance) atomicAdd(&hist[lab], 1);
      }
    }
    if (local_total) atomicAdd(&s_total, local_total);
    __syncthreads();
    int total = s_total;
    for (int q = threadIdx.x; q < nInstance; q += blockDim.x) {
      int inter = hist[q];
      // fp64 divide, `+ 1e-5` is a double literal (cal_iou_and_masklabel.cu:29-31)
      double v = (double)(float)inter / ((double)(float)(total + inst_pointnum[q] - inter) + 1e-5);
      iou[(size_t)p * nInstance + q] = (float)v;
    }
    __syncthreads();
  }
}

__global__ void mask_label_kernel(const int32_t *__restrict__ pidx, const int32_t *__restrict__ poff,
                                  const long long *__restrict__ inst_labels, const long long *__restrict__ inst_cls,
                                  const float *__restrict__ iou, int nInstance, int nProposal, float iou_thr,
                                  float *__restrict__ mask_label) {
  __shared__ float s_val[32];
  __shared__ int s_ind[32];
  for (int p = blockIdx.x; p < nProposal; p += gridDim.x) {
    // first instance (lowest index) attaining the strict maximum > 0 among non-ignored classes (:80-89)
    float best = 0.f;
    int bi = 0x7fffffff;
    for (int q = threadIdx.x; q < nInstance; q += blockDim.x) {
      float v = iou[(size_t)p * nInstance + q];
      if (inst_cls[q] != -100 && (v > best || (v == best && v > 0.f && q < bi))) { best = v; bi = q; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_val[warp] = best; s_ind[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      int nw = blockDim.x >> 5;
      best = (lane < nw) ? s_val[lane] : 0.f;
      bi = (lane < nw) ? s_ind[lane] : 0x7fffffff;
      for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (lane == 0) { s_val[0] = best; s_ind[0] = (best > 0.f) ? bi : 0; }
    }
    __syncthreads();
    float max_iou = s_val[0];
    int max_ind = s_ind[0];
    if (max_iou >= iou_thr) {
      int s = poff[p], e = poff[p + 1];
      for (int i = s + threadIdx.x; i < e; i += blockDim.x)
        mask_label[i] = ((int)inst_labels[pidx[i]] == max_ind) ? 1.f : 0.f;
    }
    __syncthreads();
  }
}

static int pow2_cw(int C) {
  int cw = 1;
  while (cw < C && cw < 32) cw <<= 1;
  return cw;
}

template <int OP>
static int seg_launch(const float *inp, const int32_t *off, float *out, int nP, int C, void *stream) {
  if (nP == 0 || C == 0) return SGB_OK;
  SGB_REQUIRE(inp && off && out && nP > 0 && C > 0, SGB_ERR_ARG, "segment reduce arguments");
  if (OP == OP_MIN || OP == OP_MAX) {
    SGB_CURRENT_DEVICE(d);
    // an empty proposal keeps the initial value: +inf / -inf, what `1e50` / `-1e50` become as float (sec_mean.cu:47,73)
    const long long n = (long long)nP * C;
    seg_fill_kernel<<<div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(out, n, OP == OP_MIN ? INFINITY : -INFINITY);
    SGB_LAUNCH_CHECK();
    seg_minmax_kernel<OP><<<d->sms * 4, kSegThreads, 0, (cudaStream_t)stream>>>(inp, off, out, nP, C, pow2_cw(C));
    SGB_LAUNCH_CHECK();
    return SGB_OK;
  }
  seg_reduce_kernel<OP><<<std::min(nP, 65535), kSegThreads, 0, (cudaStream_t)stream>>>(inp, off, out, nP, C, pow2_cw(C));
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_sec_mean(const float *d_inp, const int32_t *d_offsets, float *d_out, int nProposal, int C, void *stream) {
  return seg_launch<OP_MEAN>(d_inp, d_offsets, d_out, nProposal, C, stream);
}
int sgb_sec_min(const float *d_inp, const int32_t *d_offsets, float *d_out, int nProposal, int C, void *stream) {
  return seg_launch<OP_MIN>(d_inp, d_offsets, d_out, nProposal, C, stream);
}
int sgb_sec_max(const float *d_inp, const int32_t *d_offsets, float *d_out, int nProposal, int C, void *stream) {
  return seg_launch<OP_MAX>(d_inp, d_offsets, d_out, nProposal, C, stream);
}
int sgb_global_avg_pool_fp(const float *d_feats, const int32_t *d_offsets, float *d_out, int nProposal, int C,
                           void *stream) {
  return seg_launch<OP_AVG>(d_feats, d_offsets, d_out, nProposal, C, stream);
}
int sgb_global_avg_pool_bp(float *d_d_feats, const int32_t *d_offsets, const float *d_d_out, int nProposal, int C,
                           void *stream) {
  if (nProposal == 0 || C == 0) return SGB_OK;
  SGB_REQUIRE(d_d_feats && d_offsets && d_d_out, SGB_ERR_ARG, "global_avg_pool_bp arguments");
  avg_pool_bp_kernel<<<std::min(nProposal, 65535), 256, 0, (cudaStream_t)stream>>>(d_d_feats, d_offsets, d_d_out,
                                                                                  nProposal, C);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_get_mask_iou(const int32_t *d_proposals_idx, const int32_t *d_proposals_offset,
                     const int64_t *d_instance_labels, const int32_t *d_instance_pointnum,
                     const float *d_mask_scores_sigmoid, float *d_proposals_iou, int nInstance, int nProposal,
                     void *stream) {
  if (nProposal == 0 || nInstance == 0) return SGB_OK;
  SGB_REQUIRE(d_proposals_idx && d_proposals_offset && d_instance_labels && d_instance_pointnum && d_proposals_iou,
              SGB_ERR_ARG, "get_mask_iou arguments");
  SGB_REQUIRE(nInstance <= 12000, SGB_ERR_RANGE, "get_mask_iou: nInstance > 12000 does not fit the shared histogram");
  mask_iou_kernel<<<std::min(nProposal, 65535), 256, (size_t)nInstance * 4, (cudaStream_t)stream>>>(
      d_proposals_idx, d_proposals_offset, (const long long *)d_instance_labels, d_instance_pointnum,
      d_mask_scores_sigmoid, d_proposals_iou, nInstance, nProposal);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_get_mask_label(const int32_t *d_proposals_idx, const int32_t *d_proposals_offset,
                       const int64_t *d_instance_labels, const int64_t *d_instance_cls,
                       const float *d_proposals_iou, int nInstance, int nProposal, float iou_thr,
                       float *d_mask_label, void *stream) {
  if (nProposal == 0) return SGB_OK;
  SGB_REQUIRE(d_proposals_idx && d_proposals_offset && d_instance_labels && d_instance_cls && d_proposals_iou &&
                  d_mask_label,
              SGB_ERR_ARG, "get_mask_label arguments");
  mask_label_kernel<<<std::min(nProposal, 65535), 256, 0, (cudaStream_t)stream>>>(
      d_proposals_idx, d_proposals_offset, (const long long *)d_instance_labels, (const long long *)d_instance_cls,
      d_proposals_iou, nInstance, nProposal, iou_thr, d_mask_label);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
}
