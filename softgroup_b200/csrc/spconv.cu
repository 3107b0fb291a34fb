// spconv.cu -- rulebook construction and sparse convolution, replacing the spconv 2.x dependency of the
// reference (softgroup/model/blocks.py:31-41,50-70,96-129; softgroup/model/softgroup.py:60-65,73-74).
//
// Rulebook: one 64-bit-key hash of the active voxel coordinates per level (atomicCAS open addressing).
//   subm3  -> int32 map[27][M]   (output-stationary: no atomics in the convolution, deterministic sums)
//   down2  -> parents numbered by first occurrence (flags + scan), map[8][Mout] children, inv_map[8][M]
// Convolution: out tile 128 rows x 32 channels per CTA; for every kernel offset the 128 input rows are gathered
// (eval-BatchNorm + ReLU applied on the fly) into a K-major shared tile, the 32x32 weight slice into another,
// and each thread accumulates an 8x4 register block with fp32 FFMA. Offsets with no active pair in the tile are
// skipped (warp vote). Residual add / bias / strided output (for the U-Net concat) are fused in the epilogue.
#include <algorithm>

#include "common.cuh"

namespace sgb {

// key: [b:16][x+1:16][y+1:16][z+1:16]; coordinates in [-1, 32766]
__device__ __forceinline__ unsigned long long vkey(int b, int x, int y, int z) {
  return ((unsigned long long)(unsigned)(b & 0xFFFF) << 48) | ((unsigned long long)(unsigned)((x + 1) & 0xFFFF) << 32) |
         ((unsigned long long)(unsigned)((y + 1) & 0xFFFF) << 16) | (unsigned long long)(unsigned)((z + 1) & 0xFFFF);
}

struct RbWs {
  unsigned long long *keys;  // [cap]
  int32_t *vals;             // [cap] row (subm) or first child (down)
  int32_t *slot_of;          // [M]
  int32_t *rank;             // [M]
  int32_t *scalars;          // 0: Mout, 2: range error
  int32_t *scan_tmp;
  uint32_t cap;
};

static size_t rb_cap(int M) { return pow2_at_least((size_t)std::max(M, 1) * 2); }

static bool rb_carve(void *ws, size_t bytes, int M, RbWs &w) {
  Arena a(ws, bytes);
  w.cap = (uint32_t)rb_cap(M);
  w.scalars = a.take<int32_t>(64);
  w.keys = a.take<unsigned long long>(w.cap);
  w.vals = a.take<int32_t>(w.cap);
  w.slot_of = a.take<int32_t>((size_t)M + 1);
  w.rank = a.take<int32_t>((size_t)M + 1);
  w.scan_tmp = a.take<int32_t>(scan_temp_elems((size_t)M + 1));
  return w.scan_tmp != nullptr;
}

__device__ __forceinline__ bool idx_ok(int b, int x, int y, int z) {
  return b >= 0 && b < 65536 && x >= 0 && x < 32767 && y >= 0 && y < 32767 && z >= 0 && z < 32767;
}

__global__ void rb_insert_kernel(const int32_t *__restrict__ indices, int M, RbWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
  if (!idx_ok(c.x, c.y, c.z, c.w)) { w.scalars[2] = 1; return; }
  uint32_t s = hash_insert(w.keys, w.cap - 1, vkey(c.x, c.y, c.z, c.w));
  w.vals[s] = i;
}

__global__ void rb_subm3_kernel(const int32_t *__restrict__ indices, int M, int32_t *__restrict__ map, RbWs w) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)M * 27) return;
  int k = (int)(t / M), j = (int)(t % M);
  int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + j);
  int dx = k / 9 - 1, dy = (k / 3) % 3 - 1, dz = k % 3 - 1;
  int r = -1;
  if (k == 13) r = j;
  else if (idx_ok(c.x, c.y, c.z, c.w)) {  // a rejected row's key could alias another row or equal kEmptyKey
    uint32_t s = hash_find(w.keys, w.cap - 1, vkey(c.x, c.y + dx, c.z + dy, c.w + dz));
    if (s != 0xFFFFFFFFu) r = w.vals[s];
  }
  map[(size_t)k * M + j] = r;
}

__global__ void rb_down_insert_kernel(const int32_t *__restrict__ indices, int M, int ox, int oy, int oz, RbWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
  if (!idx_ok(c.x, c.y, c.z, c.w)) { w.scalars[2] = 1; w.slot_of[i] = -1; return; }
  int px = c.y >> 1, py = c.z >> 1, pz = c.w >> 1;
  if (px >= ox || py >= oy || pz >= oz) { w.slot_of[i] = -1; return; }  // max plane of an odd dim is dropped
  uint32_t s = hash_insert(w.keys, w.cap - 1, vkey(c.x, px, py, pz));
  w.slot_of[i] = (int32_t)s;
  atomicMin(&w.vals[s], i);
}

__global__ void rb_down_flag_kernel(int M, RbWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  int s = w.slot_of[i];
  w.rank[i] = (s >= 0 && w.vals[s] == i) ? 1 : 0;
}

// after scan: for first children, publish parent id into vals' companion (reuse keys? no: separate pass)
__global__ void rb_down_pid_kernel(int M, int32_t *__restrict__ pid_of_slot, RbWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  int s = w.slot_of[i];
  if (s >= 0 && w.vals[s] == i) pid_of_slot[s] = w.rank[i];
}

__global__ void rb_down_fill_kernel(const int32_t *__restrict__ indices, int M, int Mout,
                                    const int32_t *__restrict__ pid_of_slot, int32_t *__restrict__ out_indices,
                                    int32_t *__restrict__ map, int32_t *__restrict__ inv_map, RbWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  int s = w.slot_of[i];
  if (s < 0) return;
  int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
  int pid = pid_of_slot[s];
  int k = ((c.y & 1) * 2 + (c.z & 1)) * 2 + (c.w & 1);
  map[(size_t)k * Mout + pid] = i;
  inv_map[(size_t)k * M + i] = pid;
  if (w.vals[s] == i) reinterpret_cast<int4 *>(out_indices)[pid] = make_int4(c.x, c.y >> 1, c.z >> 1, c.w >> 1);
}

// ---------------------------------------------------------------------------------------------
// convolution
// ---------------------------------------------------------------------------------------------
constexpr int TM = 128, TN = 32, KC = 32, CONV_THREADS = 128;

struct ConvArgs {
  const float *in; int in_stride, in_off;
  const int32_t *map; int K, Mout;
  const float *W; int Cin, Cout;
  const float *in_scale, *in_shift;
  const float *residual; int res_stride, res_off;
  const float *bias;
  float *out; int out_stride, out_off;
};

__global__ void __launch_bounds__(CONV_THREADS) spconv_kernel(ConvArgs p) {
  __shared__ __align__(16) float As[KC][TM];
  __shared__ __align__(16) float Bs[KC][TN];
  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * TM, n0 = blockIdx.y * TN;
  const int tr = tid >> 3, tc = tid & 7;
  const int my_row = row0 + tid;
  const bool row_ok = my_row < p.Mout;
  const bool has_act = p.in_scale != nullptr;
  const bool vec_ok = ((p.in_stride & 3) == 0) && ((p.in_off & 3) == 0) && ((((uintptr_t)p.in) & 15) == 0);

  float acc[8][4];
#pragma unroll
  for (int r = 0; r < 8; r++)
#pragma unroll
    for (int c = 0; c < 4; c++) acc[r][c] = 0.f;

  const int nkc = (p.Cin + KC - 1) / KC;
  for (int o = 0; o < p.K; o++) {
    int src = -1;
    if (row_ok) src = p.map ? __ldg(&p.map[(size_t)o * p.Mout + my_row]) : my_row;
    if (!__syncthreads_or(src >= 0)) continue;
    for (int kc = 0; kc < nkc; kc++) {
      const int c0 = kc * KC;
      // ---- A: gather one input row per thread, transpose into As[k][row] -------------------------
      if (src >= 0) {
        const float *rp = p.in + (size_t)src * p.in_stride + p.in_off + c0;
        if (vec_ok && c0 + KC <= p.Cin) {
#pragma unroll
          for (int q = 0; q < KC / 4; q++) {
            float4 v = __ldg(reinterpret_cast<const float4 *>(rp) + q);
            if (has_act) {
              float4 sc = __ldg(reinterpret_cast<const float4 *>(p.in_scale + c0) + q);
              float4 sh = __ldg(reinterpret_cast<const float4 *>(p.in_shift + c0) + q);
              v.x = fmaxf(fmaf(v.x, sc.x, sh.x), 0.f);
              v.y = fmaxf(fmaf(v.y, sc.y, sh.y), 0.f);
              v.z = fmaxf(fmaf(v.z, sc.z, sh.z), 0.f);
              v.w = fmaxf(fmaf(v.w, sc.w, sh.w), 0.f);
            }
            As[4 * q + 0][tid] = v.x;
            As[4 * q + 1][tid] = v.y;
            As[4 * q + 2][tid] = v.z;
            As[4 * q + 3][tid] = v.w;
          }
        } else {
#pragma unroll 8
          for (int k = 0; k < KC; k++) {
            float v = 0.f;
            if (c0 + k < p.Cin) {
              v = __ldg(rp + k);
              if (has_act) v = fmaxf(fmaf(v, __ldg(&p.in_scale[c0 + k]), __ldg(&p.in_shift[c0 + k])), 0.f);
            }
            As[k][tid] = v;
          }
        }
      } else {
#pragma unroll 8
        for (int k = 0; k < KC; k++) As[k][tid] = 0.f;
      }
      // ---- B: weight slice W[o][c0+k][n0+c] ----------------------------------------------------------
      {
        const int k = tid >> 2, cb = (tid & 3) * 8;
        const float *wp = p.W + ((size_t)o * p.Cin + c0 + k) * p.Cout + n0 + cb;
        const bool kin = (c0 + k) < p.Cin;
#pragma unroll
        for (int c = 0; c < 8; c++) Bs[k][cb + c] = (kin && n0 + cb + c < p.Cout) ? __ldg(wp + c) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < KC; k++) {
        float4 a0 = *reinterpret_cast<const float4 *>(&As[k][tr * 8]);
        float4 a1 = *reinterpret_cast<const float4 *>(&As[k][tr * 8 + 4]);
        float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tc * 4]);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int r = 0; r < 8; r++)
#pragma unroll
          for (int c = 0; c < 4; c++) acc[r][c] = fmaf(av[r], bv[c], acc[r][c]);
      }
      __syncthreads();
    }
  }
  // ---- epilogue -----------------------------------------------------------------------------------
#pragma unroll
  for (int r = 0; r < 8; r++) {
    int row = row0 + tr * 8 + r;
    if (row >= p.Mout) continue;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      int n = n0 + tc * 4 + c;
      if (n >= p.Cout) continue;
      float v = acc[r][c];
      if (p.bias) v += __ldg(&p.bias[n]);
      if (p.residual) v += __ldg(&p.residual[(size_t)row * p.res_stride + p.res_off + n]);
      p.out[(size_t)row * p.out_stride + p.out_off + n] = v;
    }
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_rulebook_workspace_bytes(int M) {
  if (M < 0) M = 0;
  size_t cap = rb_cap(M);
  // + pid_of_slot [cap] for down2
  size_t b = align_up(64 * 4) + align_up(cap * 8) + 2 * align_up(cap * 4) + 2 * align_up(((size_t)M + 1) * 4) +
             align_up(scan_temp_elems((size_t)M + 1) * 4);
  return b + 1024;
}

int sgb_rulebook_subm3(const int32_t *d_indices, int M, int32_t *d_map, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (M == 0) return SGB_OK;
  SGB_REQUIRE(d_indices && d_map && d_ws && M > 0, SGB_ERR_ARG, "rulebook_subm3 arguments");
  SGB_REQUIRE(((uintptr_t)d_indices & 15) == 0, SGB_ERR_ARG, "indices must be 16-byte aligned");
  RbWs w;
  SGB_REQUIRE(rb_carve(d_ws, ws_bytes, M, w), SGB_ERR_WORKSPACE, "rulebook workspace too small");
  SGB_CUDA_CHECK(cudaMemsetAsync(w.keys, 0xFF, (size_t)w.cap * 8, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.scalars, 0, 64 * 4, st));
  rb_insert_kernel<<<div_up(M, 256), 256, 0, st>>>(d_indices, M, w);
  SGB_LAUNCH_CHECK();
  rb_subm3_kernel<<<div_up((long long)M * 27, 256), 256, 0, st>>>(d_indices, M, d_map, w);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_rulebook_down2_count(const int32_t *d_indices, int M, const int32_t *h_spatial_shape, void *d_ws,
                             size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (M == 0) return 0;
  SGB_REQUIRE(d_indices && h_spatial_shape && d_ws && M > 0, SGB_ERR_ARG, "rulebook_down2 arguments");
  SGB_REQUIRE(((uintptr_t)d_indices & 15) == 0, SGB_ERR_ARG, "indices must be 16-byte aligned");
  RbWs w;
  SGB_REQUIRE(rb_carve(d_ws, ws_bytes, M, w), SGB_ERR_WORKSPACE, "rulebook workspace too small");
  SGB_CUDA_CHECK(cudaMemsetAsync(w.keys, 0xFF, (size_t)w.cap * 8, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.vals, 0x7F, (size_t)w.cap * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.scalars, 0, 64 * 4, st));
  int nb = div_up(M, 256);
  // spconv: out = floor((D + 2*0 - 2) / 2) + 1 = floor(D / 2) for D >= 2
  rb_down_insert_kernel<<<nb, 256, 0, st>>>(d_indices, M, h_spatial_shape[0] / 2, h_spatial_shape[1] / 2,
                                            h_spatial_shape[2] / 2, w);
  SGB_LAUNCH_CHECK();
  rb_down_flag_kernel<<<nb, 256, 0, st>>>(M, w);
  SGB_LAUNCH_CHECK();
  int rc = exclusive_scan_i32(w.rank, w.rank, (size_t)M, &w.scalars[0], w.scan_tmp, st);
  if (rc) return rc;
  int h[4];
  SGB_CUDA_CHECK(cudaMemcpyAsync(h, w.scalars, sizeof(h), cudaMemcpyDeviceToHost, st));
  SGB_CUDA_CHECK(cudaStreamSynchronize(st));
  SGB_REQUIRE(h[2] == 0, SGB_ERR_RANGE, "rulebook: index outside the packed key range (b<65536, 0<=xyz<32767)");
  return h[0];
}

int sgb_rulebook_down2_fill(const int32_t *d_indices, int M, int Mout, int32_t *d_out_indices, int32_t *d_map,
                            int32_t *d_inv_map, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (M == 0) return SGB_OK;
  // with no parents (an axis of extent 1) the outputs of Mout rows are empty and may be null
  SGB_REQUIRE(d_indices && (Mout == 0 || (d_out_indices && d_map)) && d_inv_map && d_ws, SGB_ERR_ARG,
              "rulebook_down2_fill arguments");
  SGB_REQUIRE(((uintptr_t)d_out_indices & 15) == 0, SGB_ERR_ARG, "out_indices must be 16-byte aligned");
  RbWs w;
  SGB_REQUIRE(rb_carve(d_ws, ws_bytes, M, w), SGB_ERR_WORKSPACE, "rulebook workspace too small");
  // pid_of_slot lives right after the carved region
  Arena a(d_ws, ws_bytes);
  a.off = (size_t)((char *)w.scan_tmp - (char *)d_ws) + align_up(scan_temp_elems((size_t)M + 1) * 4);
  int32_t *pid_of_slot = a.take<int32_t>(w.cap);
  SGB_REQUIRE(pid_of_slot, SGB_ERR_WORKSPACE, "rulebook workspace too small");
  if (Mout > 0) SGB_CUDA_CHECK(cudaMemsetAsync(d_map, 0xFF, (size_t)8 * Mout * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(d_inv_map, 0xFF, (size_t)8 * M * 4, st));
  int nb = div_up(M, 256);
  rb_down_pid_kernel<<<nb, 256, 0, st>>>(M, pid_of_slot, w);
  SGB_LAUNCH_CHECK();
  rb_down_fill_kernel<<<nb, 256, 0, st>>>(d_indices, M, Mout, pid_of_slot, d_out_indices, d_map, d_inv_map, w);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int sgb_spconv_forward(const float *d_in, int in_stride, int in_off, const int32_t *d_map, int K, int Mout,
                       const float *d_W, int Cin, int Cout, const float *d_in_scale, const float *d_in_shift,
                       const float *d_residual, int res_stride, int res_off, const float *d_bias, float *d_out,
                       int out_stride, int out_off, void *stream) {
  if (Mout == 0 || Cout == 0) return SGB_OK;
  SGB_REQUIRE(d_in && d_W && d_out && K >= 1 && Mout > 0 && Cin > 0 && Cout > 0, SGB_ERR_ARG, "spconv_forward arguments");
  SGB_REQUIRE(d_map || K == 1, SGB_ERR_ARG, "identity map requires K == 1");
  SGB_REQUIRE((d_in_scale == nullptr) == (d_in_shift == nullptr), SGB_ERR_ARG, "scale/shift must come together");
  SGB_REQUIRE(in_stride >= in_off + Cin && out_stride >= out_off + Cout, SGB_ERR_ARG, "row strides");
  ConvArgs p;
  p.in = d_in; p.in_stride = in_stride; p.in_off = in_off;
  p.map = d_map; p.K = K; p.Mout = Mout;
  p.W = d_W; p.Cin = Cin; p.Cout = Cout;
  p.in_scale = d_in_scale; p.in_shift = d_in_shift;
  p.residual = d_residual; p.res_stride = res_stride; p.res_off = res_off;
  p.bias = d_bias;
  p.out = d_out; p.out_stride = out_stride; p.out_off = out_off;
  dim3 grid(div_up(Mout, TM), div_up(Cout, TN));
  spconv_kernel<<<grid, CONV_THREADS, 0, (cudaStream_t)stream>>>(p);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
}
