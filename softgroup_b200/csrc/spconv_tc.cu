// spconv_tc.cu -- sparse convolution on the Hopper tensor cores (wgmma, fp32 accumulators in registers), sm_90a.
//
// One CTA (two warpgroups, 64 output rows each) owns a work item of 128 output rows x NT <= 128 output columns (and,
// with split-K, a contiguous share of the item's (kernel offset, 32-channel slice) iterations). For every kernel offset
// with at least one active pair in the tile and every 32-channel slice of Cin:
//   * all threads gather the tile's input row slices with cp.async (16 B per copy, zero-fill for absent neighbours)
//     straight into the SWIZZLE_128B K-major tile the MMA reads. Inputs are PACKED rows: activated (the consumer's
//     BatchNorm(eval)+ReLU) and split once by the PRODUCING convolution's epilogue or by sgb_act_pack. A value x is
//     carried as two fp16 numbers hi = fp16(x), lo = fp16((x - hi) * 2^kLoShift): one 128-byte line per row and slice
//     holds 32 hi values then 32 lo values;
//   * the pre-packed weight slice (same split, core-matrix order, done once on the host side) is copied next to it;
//     several stages are in flight, so the L2 latency of the gather overlaps the MMAs of the stages before;
//   * each warpgroup issues the error-compensated products as wgmma.mma_async m64nNTk16 (fp16 in, fp32 accumulate)
//         main += A_hi * B_hi      corr += A_hi * B_lo      corr += A_lo * B_hi
//     and the epilogue forms main + corr * 2^-kLoShift, adds bias / residual and writes strided fp32 rows (the U-Net
//     concat buffer) and/or the PACKED rows its consumer reads (that consumer's BatchNorm+ReLU folded in: an
//     intermediate with a single consumer never exists in fp32).
// Two launch forms of the same kernel (bit-identical results without split-K, see sgb_spconv_kernel_choice):
//   * kernel 0, one CTA per work item. With few row tiles (deep U-Net levels: a handful of tiles, megabytes of weights)
//     the columns are split and the CTAs of one thread-block cluster share a tile's iterations (split-K); ranks > 0
//     park their partial tiles in their own shared memory and rank 0 sums them in rank order over distributed shared
//     memory -- deterministic, no workspace, no atomics;
//   * kernel 1, persistent: as many CTAs as fit on the GPU at once walk the work items round-robin.
// Dropping lo*lo leaves a relative error of ~2^-22 per product, i.e. fp32-grade (1e-4 end to end over ~40 sequential
// convolutions rules out plain TF32/fp16; see DESIGN.md).
#include <algorithm>
#include <cstdlib>

#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace sgb {

constexpr int TC_ROWS = 128;
constexpr int TC_KC = 32;        // channels per iteration: one 128-byte packed line per row
constexpr int TC_THREADS = 256;  // two warpgroups
constexpr int TC_STAGES = 4;     // gather ring depth
constexpr int TC_A_BYTES = TC_ROWS * 128;  // 16 KB of rows per stage
// The remainder lo = x - fp16(x) is carried as fp16(lo * 2^kLoShift); the correction products are scaled back by
// 2^-kLoShift when they are added to the main product. 11 keeps lo a normal fp16 number down to |x| = 2^-14 (with
// shift 0 the per-element 1e-4 bar was missed at C = 224); sgb_spconv_lo_shift() tells the host weight packer.
constexpr int kLoShift = 11;
constexpr float kLoScale = (float)(1 << kLoShift), kLoInv = 1.0f / kLoScale;

struct TcArgs {
  const uint32_t *in; int in_stride;     // packed rows [Min][in_stride words]
  const int32_t *map; int K, Mout;       // map [K][Mout] (nullptr: identity, K == 1)
  const float *Wp;                       // packed fp16 [K][nkc][4 chunks][2 (hi,lo)][N][8 halves]
  int Cin, N, Cout;                      // N = Cout rounded up to 16
  int nparts;                            // column parts of NT (the last may be shorter)
  int items;                             // row tiles x column parts
  int ksplit;                            // CTAs per cluster along z sharing one item's iterations (1 = no split)
  const float *residual; int res_stride, res_off;
  const float *bias;
  float *out; int out_stride, out_off;   // optional fp32 rows
  uint32_t *pk; int pk_stride, pk_coff;  // optional packed rows: row stride in words, first channel (multiple of 8)
  const float *pk_scale, *pk_shift; int pk_relu;  // per OUTPUT channel (nullptr: identity): the consumer's BatchNorm+ReLU
  int pk_fill;                           // zero the rest of the 32-channel chunk the written channels end in
  int *oflow;                            // device flag: a packed value beyond the fp16 range
};

template <int NT>
constexpr size_t tc_stage_bytes() { return (size_t)TC_A_BYTES + (size_t)NT * 128; }  // rows + [4 chunks][hi|lo][NT][16 B]
template <int NT>
constexpr int tc_min_blocks() { return NT <= 64 ? 2 : 1; }  // register file: 2 x NT / 2 fp32 accumulators per thread

template <int NT>
__global__ void __launch_bounds__(TC_THREADS, tc_min_blocks<NT>()) spconv_tc_kernel(TcArgs p) {
  constexpr int R = NT / 2;  // accumulator registers per thread and product
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ unsigned int s_mask;
  __shared__ int s_list[32];
  __shared__ int s_nact;

  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, wq = (tid >> 5) & 3;
  unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // SWIZZLE_128B: 1024-aligned
  unsigned char *a_ring = smem;
  unsigned char *b_ring = a_ring + (size_t)TC_STAGES * TC_A_BYTES;
  int32_t *map_s = reinterpret_cast<int32_t *>(b_ring + (size_t)TC_STAGES * NT * 128);  // [K][128]
  const uint32_t a_base = smem_u32(a_ring), b_base = smem_u32(b_ring);
  const int nkc = (p.Cin + TC_KC - 1) / TC_KC;
  const int ks_last = (p.Cin - (nkc - 1) * TC_KC + 15) >> 4;  // 16-channel k-steps of the last slice (1 or 2)
  const int S = p.ksplit, z = blockIdx.z;
  const bool split = S > 1;

  for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
    const int tile = item / p.nparts, part = item - tile * p.nparts;
    const int row0 = tile * TC_ROWS, n0 = part * NT;
    const int nt = min(NT, p.N - n0);  // columns of this item (multiple of 16)
    __syncthreads();  // the previous item is done with the rulebook slice and the ring
    if (tid == 0) s_mask = 0u;
    __syncthreads();
    // ---- rulebook slice of this tile -> shared memory; which kernel offsets have any active pair ----------------
    {
      const int r = tid & (TC_ROWS - 1), row = row0 + r;
      unsigned int flags = 0u;
      if (p.map) {
        for (int ob = tid >> 7; ob < p.K; ob += 16) {  // up to 8 entries of this row in flight
          int v[8];
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const int o = ob + 2 * j;
            v[j] = (o < p.K && row < p.Mout) ? __ldg(&p.map[(size_t)o * p.Mout + row]) : -1;
          }
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const int o = ob + 2 * j;
            if (o < p.K) {
              map_s[o * TC_ROWS + r] = v[j];
              if (v[j] >= 0) flags |= 1u << o;
            }
          }
        }
      } else if (tid < TC_ROWS) {
        map_s[r] = row < p.Mout ? row : -1;
        flags = 1u;
      }
      flags = __reduce_or_sync(0xffffffffu, flags);
      if (lane == 0 && flags) atomicOr(&s_mask, flags);
    }
    __syncthreads();
    if (tid < 32) {  // compact the active offsets in ascending order
      const unsigned int m = s_mask;
      if (tid < p.K && (m >> tid & 1u)) s_list[__popc(m & ((1u << tid) - 1u))] = tid;
      if (tid == 0) s_nact = __popc(m);
    }
    __syncthreads();
    // split-K: the cluster's CTAs take contiguous shares of the item's (offset, slice) iterations
    const int total_all = s_nact * nkc;
    const int i_beg = (int)((long long)total_all * z / S), i_end = (int)((long long)total_all * (z + 1) / S);
    const int total = i_end - i_beg;

    // ---- gather of iteration `it` (CTA-local) into ring stage it % TC_STAGES: 1024 row chunks + 8 NT weight chunks
    auto load = [&](int it) {
      if (it < total) {
        const int gi = i_beg + it, a = gi / nkc, kc = gi - a * nkc;
        const int o = s_list[a];
        const int s = it % TC_STAGES;
        const uint32_t sa = a_base + (uint32_t)s * TC_A_BYTES;
        const int32_t *ms = map_s + o * TC_ROWS;
#pragma unroll
        for (int q = 0; q < TC_ROWS * 8 / TC_THREADS; q++) {
          const int c = tid + q * TC_THREADS, row = c >> 3, ch = c & 7;
          const int src = ms[row];
          const uint32_t *gp = p.in + (size_t)max(src, 0) * p.in_stride + kc * TC_KC + ch * 4;
          cp_async16(sa + (uint32_t)(row * 128 + ((ch ^ (row & 7)) << 4)), gp, src >= 0 ? 16 : 0);
        }
        const uint32_t sb = b_base + (uint32_t)s * (NT * 128);
        const float4 *g = reinterpret_cast<const float4 *>(p.Wp) + ((size_t)o * nkc + kc) * (size_t)p.N * 8;
        for (int c = tid; c < 8 * NT; c += TC_THREADS) {
          const int seg = c / NT, n = c - seg * NT;  // seg = chunk * 2 + (hi, lo)
          const bool ok = n < nt;
          cp_async16(sb + (uint32_t)c * 16u, g + (size_t)seg * p.N + n0 + (ok ? n : 0), ok ? 16 : 0);
        }
      }
      cp_async_commit();  // (an empty group past the end keeps the group count in step)
    };

    float acc[R], cor[R];
#pragma unroll
    for (int i = 0; i < R; i++) acc[i] = cor[i] = 0.f;
#pragma unroll
    for (int s = 0; s < TC_STAGES - 1; s++) load(s);
    const uint32_t b_lbo = (uint32_t)NT * 32u;  // distance between the two 8-channel chunks of a k-step: [hi NT | lo NT] x 16 B
    for (int it = 0; it < total; it++) {
      cp_async_wait<TC_STAGES - 2>();
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy (cp.async) writes -> visible to wgmma
      __syncthreads();  // every thread's copies of stage it landed; every warpgroup is done with stage it - 1
      load(it + TC_STAGES - 1);
      const int s = it % TC_STAGES;
      const int kc = (i_beg + it) % nkc;
      const int ksteps = (kc + 1 < nkc) ? 2 : ks_last;
      const uint32_t sa = a_base + (uint32_t)s * TC_A_BYTES + (uint32_t)wg * (64 * 128);
      const uint32_t sb = b_base + (uint32_t)s * (NT * 128);
      wgmma_fence_regs(acc);
      wgmma_fence_regs(cor);
      wgmma_fence();
      for (int ks = 0; ks < ksteps; ks++) {
        const uint64_t ah = desc_sw128(sa + 32u * ks), al = desc_sw128(sa + 64u + 32u * ks);
        const uint32_t bk = sb + (uint32_t)ks * 2u * b_lbo;  // chunks 2 ks, 2 ks + 1
        const uint64_t bh = desc_plain(bk, b_lbo, 128), bl = desc_plain(bk + (uint32_t)NT * 16u, b_lbo, 128);
        wgmma_f16<NT>(acc, ah, bh);
        wgmma_f16<NT>(cor, ah, bl);
        wgmma_f16<NT>(cor, al, bh);
      }
      wgmma_commit();
      wgmma_wait0();
      wgmma_fence_regs(acc);
      wgmma_fence_regs(cor);
    }
    cp_async_wait<0>();
#pragma unroll
    for (int i = 0; i < R; i++) acc[i] = fmaf(cor[i], kLoInv, acc[i]);

    // ---- epilogue: thread holds rows rb, rb + 8 and columns 8 j + 2 (lane & 3) + {0, 1} of its warpgroup's 64 rows --
    const int rl = wg * 64 + wq * 16 + (lane >> 2);  // tile-local row of acc[4 j + 0, 1]; acc[4 j + 2, 3] is rl + 8
    const int cl = 2 * (lane & 3);
    if (split) {
      const uint32_t pbuf = a_base;  // partial tile [NT columns][128 rows] f32 (the ring is idle by now)
      __syncthreads();
      if (z > 0) {
#pragma unroll
        for (int i = 0; i < R; i++) {
          const int col = 8 * (i >> 2) + cl + (i & 1), row = rl + 8 * ((i >> 1) & 1);
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(pbuf + (uint32_t)((col * TC_ROWS + row) * 4)), "f"(acc[i]) : "memory");
        }
      }
      asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
      if (z == 0) {  // add the other ranks' partial tiles in rank order (distributed shared memory)
        for (int zz = 1; zz < S; zz++) {
          uint32_t rbase;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbase) : "r"(pbuf), "r"(zz));
#pragma unroll
          for (int i = 0; i < R; i++) {
            const int col = 8 * (i >> 2) + cl + (i & 1), row = rl + 8 * ((i >> 1) & 1);
            float t;
            asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(t) : "r"(rbase + (uint32_t)((col * TC_ROWS + row) * 4)) : "memory");
            acc[i] += t;
          }
        }
      }
      // ranks > 0 keep their shared memory alive until rank 0 has read it
      asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    }
    if (!split || z == 0) {
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = row0 + rl + 8 * h;
        if (row >= p.Mout) continue;
#pragma unroll
        for (int j = 0; j < NT / 8; j++) {
          const int cj = 8 * j + cl;  // item-local column of this pair
          if (cj >= nt) continue;
          const int col = n0 + cj;
          float x[2] = {acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]};
          const bool full = col + 2 <= p.Cout;
          if (p.bias) {
#pragma unroll
            for (int e = 0; e < 2; e++)
              if (col + e < p.Cout) x[e] += __ldg(&p.bias[col + e]);
          }
          if (p.residual) {
            const float *rp = p.residual + (size_t)row * p.res_stride + p.res_off + col;
#pragma unroll
            for (int e = 0; e < 2; e++)
              if (col + e < p.Cout) x[e] += __ldg(rp + e);
          }
          if (p.out) {
            float *op = p.out + (size_t)row * p.out_stride + p.out_off + col;
            if (full && ((reinterpret_cast<uintptr_t>(op) & 7) == 0)) {
              *reinterpret_cast<float2 *>(op) = make_float2(x[0], x[1]);
            } else {
#pragma unroll
              for (int e = 0; e < 2; e++)
                if (col + e < p.Cout) op[e] = x[e];
            }
          }
          if (p.pk) {
            // the consumer's BatchNorm(eval)+ReLU, then the fp16 hi/lo split: 2 channels -> 1 word hi + 1 word lo
            float y[2];
            bool big = false;
#pragma unroll
            for (int e = 0; e < 2; e++) {
              float t = x[e];
              if (col + e >= p.Cout) t = 0.f;  // padding channels stay exactly zero
              else if (p.pk_scale) t = fmaf(t, __ldg(&p.pk_scale[col + e]), __ldg(&p.pk_shift[col + e]));
              if (p.pk_relu) t = fmaxf(t, 0.f);
              big |= !(fabsf(t) <= 65504.f);
              y[e] = t;
            }
            if (big) *p.oflow = 1;
            const __half2 hh = f2h2_sat(y[0], y[1]);
            const float2 hf = __half22float2(hh);
            const __half2 ll = f2h2_sat((y[0] - hf.x) * kLoScale, (y[1] - hf.y) * kLoScale);
            const int ch = p.pk_coff + col;  // channel in the packed tensor (even)
            uint32_t *dst = p.pk + (size_t)row * p.pk_stride + (ch >> 5) * 32 + ((ch & 31) >> 1);
            dst[0] = *reinterpret_cast<const uint32_t *>(&hh);
            dst[16] = *reinterpret_cast<const uint32_t *>(&ll);
          }
        }
        if (p.pk && p.pk_fill && n0 + nt == p.N && ((p.pk_coff + p.N) & 31)) {
          // the written channels end in the middle of a 32-channel chunk: the consumer reads whole chunks, so channels
          // [pk_coff + N, round_up32(pk_coff + N)) -- 8, 16 or 24 of them, hi and lo words -- must be zero (not stale
          // memory: 0 * NaN would poison the sums); the 4 threads of the row share the words
          const int ch2 = p.pk_coff + p.N;
          uint32_t *zp = p.pk + (size_t)row * p.pk_stride + (ch2 >> 5) * 32;
          for (int w = ((ch2 & 31) >> 1) + (lane & 3); w < 16; w += 4) { zp[w] = 0u; zp[w + 16] = 0u; }
        }
      }
    }
  }
}

// y = BatchNorm(eval)+ReLU(x) (or x when scale == nullptr) -> packed rows (see the header of this file). One thread per
// (row, word pair); channels past C are zero up to Cfill. Used where a tensor has no producing convolution to fuse into
// (network input, the concat half written by the encoder, gathered point rows).
__global__ void act_pack_kernel(const float *__restrict__ x, int x_stride, int x_off, const float *__restrict__ scale,
                                const float *__restrict__ shift, int relu, uint32_t *__restrict__ y, int y_stride, int y_coff,
                                int M, int C, int Cfill, int *__restrict__ oflow) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int wpr = Cfill >> 1;  // word pairs (2 channels) per row
  if (t >= (long long)M * wpr) return;
  const int row = (int)(t / wpr), pr = (int)(t % wpr);
  const int c = 2 * pr;
  float a = 0.f, b = 0.f;
  if (c < C) a = x[(size_t)row * x_stride + x_off + c];
  if (c + 1 < C) b = x[(size_t)row * x_stride + x_off + c + 1];
  if (scale) {
    if (c < C) a = fmaf(a, __ldg(&scale[c]), __ldg(&shift[c]));
    if (c + 1 < C) b = fmaf(b, __ldg(&scale[c + 1]), __ldg(&shift[c + 1]));
  }
  if (relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
  if (!(fabsf(a) <= 65504.f) || !(fabsf(b) <= 65504.f)) *oflow = 1;
  const __half2 h = f2h2_sat(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = f2h2_sat((a - hf.x) * kLoScale, (b - hf.y) * kLoScale);
  const int ch = y_coff + c;
  uint32_t *yr = y + (size_t)row * y_stride + (ch >> 5) * 32 + ((ch & 31) >> 1);
  yr[0] = *reinterpret_cast<const uint32_t *>(&h);
  yr[16] = *reinterpret_cast<const uint32_t *>(&l);
}

}  // namespace sgb

using namespace sgb;

namespace {

constexpr int kNumSMs = 132;  // H100 SXM: what the pure plan functions assume when the caller gives no SM count

// per NT / 16: the kernel's shared-memory attribute is set and its CTAs per SM are known, per device
DeviceOnce g_tc_once[9];
int g_tc_per_sm[kMaxDevices][9];

// Columns per work item of the persistent launch: all of N up to 128, else N cut into equal parts (multiple of 16).
int persistent_nt(int N) { return N <= 128 ? N : (div_up(N, div_up(N, 128)) + 15) / 16 * 16; }

// Shared memory of a CTA: the gather ring, the rulebook slice of the largest kernel (27 offsets) and the alignment slack.
size_t tc_smem_bytes(int NT) { return (size_t)TC_STAGES * ((size_t)TC_A_BYTES + (size_t)NT * 128) + 27 * TC_ROWS * 4 + 1024; }

// Which launch runs a problem. The persistent form takes the levels with many row tiles (Cout >= 64 from 16 row tiles
// upwards, and the big 32-channel levels); one CTA per work item keeps the deep levels (a handful of row tiles: column
// split + split-K clusters) and the 32-channel tiny U-Net (a few hundred tiles).
bool use_persistent(int K, int Mout, int Cin, int Cout, int sms) {
  if ((Cout + 15) / 16 * 16 > 256 || Cin > 512 || K > 27) return false;
  const int tiles = div_up(Mout, TC_ROWS);
  return tiles >= 16 && (Cout >= 64 || tiles >= 4 * sms);
}

template <int NT>
int launch_nt(const TcArgs &p, bool persistent, const Device &d, cudaStream_t stream) {
  const size_t smem = tc_smem_bytes(NT);
  int *per_sm = &g_tc_per_sm[d.ordinal][NT / 16];
  int rc = once_per_device(g_tc_once[NT / 16], d.ordinal, [&] {
    SGB_CUDA_CHECK(cudaFuncSetAttribute(spconv_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int n = 0;
    SGB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, spconv_tc_kernel<NT>, TC_THREADS, smem));
    *per_sm = std::max(n, 1);
    return SGB_OK;
  });
  if (rc) return rc;
  if (persistent) {
    const int grid = std::min(p.items, d.sms * *per_sm);
    spconv_tc_kernel<NT><<<grid, TC_THREADS, smem, stream>>>(p);
  } else if (p.ksplit == 1) {
    spconv_tc_kernel<NT><<<p.items, TC_THREADS, smem, stream>>>(p);
  } else {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.items, 1, p.ksplit);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = p.ksplit;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    SGB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, spconv_tc_kernel<NT>, p));
  }
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

int launch(int NT, const TcArgs &p, bool persistent, const Device &d, cudaStream_t stream) {
  switch (NT) {
    case 16: return launch_nt<16>(p, persistent, d, stream);
    case 32: return launch_nt<32>(p, persistent, d, stream);
    case 48: return launch_nt<48>(p, persistent, d, stream);
    case 64: return launch_nt<64>(p, persistent, d, stream);
    case 80: return launch_nt<80>(p, persistent, d, stream);
    case 96: return launch_nt<96>(p, persistent, d, stream);
    case 112: return launch_nt<112>(p, persistent, d, stream);
    case 128: return launch_nt<128>(p, persistent, d, stream);
  }
  SGB_REQUIRE(false, SGB_ERR_RANGE, "spconv_forward_tc: columns per CTA not a multiple of 16 in [16, 128]");
}

}  // namespace

extern "C" {

// log2 of the factor the fp16 remainders (weights AND activations) are scaled by; the host weight packer uses the same.
int sgb_spconv_lo_shift(void) { return sgb::kLoShift; }

// Reads (and clears) the overflow flag raised by the packing code paths: blocking 4-byte read on `stream`.
int sgb_spconv_overflow(int *h_flag, void *stream) {
  SGB_REQUIRE(h_flag, SGB_ERR_ARG, "null flag");
  *h_flag = 0;
  SGB_CURRENT_DEVICE(d);
  cudaStream_t st = (cudaStream_t)stream;
  SGB_CUDA_CHECK(cudaMemcpyAsync(h_flag, d->oflow, 4, cudaMemcpyDeviceToHost, st));
  SGB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (*h_flag) SGB_CUDA_CHECK(cudaMemsetAsync(d->oflow, 0, 4, st));
  return SGB_OK;
}

int sgb_act_pack(const float *d_x, int x_stride, int x_off, const float *d_scale, const float *d_shift, int relu,
                 float *d_pk, int pk_stride, int pk_coff, int M, int C, int Cfill, void *stream) {
  if (M == 0 || C == 0) return SGB_OK;
  SGB_REQUIRE(d_x && d_pk && M > 0 && C > 0 && (d_scale == nullptr) == (d_shift == nullptr), SGB_ERR_ARG, "act_pack arguments");
  SGB_REQUIRE((pk_stride & 31) == 0 && (pk_coff & 1) == 0 && (Cfill & 1) == 0 && Cfill >= C && pk_stride >= pk_coff + Cfill,
              SGB_ERR_ARG, "act_pack: row stride multiple of 32 words, channel offset and fill width even, fill inside the row");
  SGB_CURRENT_DEVICE(d);
  long long tot = (long long)M * (Cfill / 2);
  act_pack_kernel<<<div_up(tot, 256), 256, 0, (cudaStream_t)stream>>>(d_x, x_stride, x_off, d_scale, d_shift, relu,
                                                                    (uint32_t *)d_pk, pk_stride, pk_coff, M, C, Cfill, d->oflow);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

// Packed weight size in floats for sgb_spconv_forward_tc: K * ceil(Cin/32) * 8 * N * 4 with N = Cout rounded to 16.
long long sgb_spconv_tc_packed_floats(int K, int Cin, int Cout) {
  int N = (Cout + 15) / 16 * 16;
  int nkc = (Cin + 31) / 32;
  return (long long)K * nkc * 4 * 2 * N * 4;  // fp16: 4 chunks of 8 halves, counted in 32-bit words
}

// Tile configuration of the one-CTA-per-item launch for a problem (pure function of the sizes; also what the launch
// uses): for tests and tools. out[0] = NT, [1] = column parts, [2] = split-K ranks, [3] = shared memory per CTA (bytes),
// [4] = gather ring stages, [5] = row tiles
int sgb_spconv_tc_plan(int K, int Mout, int Cin, int Cout, int has_map, int sms, int *out) {
  SGB_REQUIRE(out && K >= 1 && Mout >= 1 && Cin >= 1 && Cout >= 1, SGB_ERR_ARG, "spconv_tc_plan arguments");
  if (sms <= 0) sms = kNumSMs;
  const int N = (Cout + 15) / 16 * 16;
  // Column split: few row tiles (deep U-Net levels) would leave most SMs idle and make one CTA stream all the
  // weights, so N is cut into NT-column CTAs until the grid covers the machine (NT multiple of 16, >= 32).
  const int tiles = div_up(Mout, TC_ROWS);
  int NT = std::min(N, 128);
  if (N > 128) NT = (N / 2 + 15) / 16 * 16;
  while (NT > 32 && tiles * div_up(N, NT) < sms) {
    int nxt = (NT / 2 + 15) / 16 * 16;
    if (nxt >= NT) break;
    NT = nxt;
  }
  // split-K: when even the narrowest column split leaves most SMs idle, a cluster of S CTAs shares each tile's
  // iterations (S <= 8, the portable cluster size) and reduces through distributed shared memory.
  const int nkc = (Cin + TC_KC - 1) / TC_KC;
  const int ctas = tiles * div_up(N, NT);
  int S = 1;
  if (ctas * 2 <= sms) S = std::max(1, std::min({8, 2 * sms / ctas, std::max(1, K * nkc / 4)}));
  out[0] = NT; out[1] = div_up(N, NT); out[2] = S; out[3] = (int)tc_smem_bytes(NT); out[4] = TC_STAGES; out[5] = tiles;
  (void)has_map;
  return SGB_OK;
}

// 1 = the persistent launch would run this problem, 0 = one CTA per work item (pure function).
int sgb_spconv_kernel_choice(int K, int Mout, int Cin, int Cout, int sms) {
  if (K < 1 || Mout < 1 || Cin < 1 || Cout < 1) return 0;
  return use_persistent(K, Mout, Cin, Cout, sms > 0 ? sms : kNumSMs) ? 1 : 0;
}

int sgb_spconv_forward_tc(const float *d_in_pk, int in_stride, int Min, const int32_t *d_map, int K, int Mout,
                          const float *d_Wp, int Cin, int Cout, const float *d_residual, int res_stride, int res_off,
                          const float *d_bias, float *d_out, int out_stride, int out_off, float *d_pk_out, int pk_stride,
                          int pk_coff, const float *d_pk_scale, const float *d_pk_shift, int pk_relu, int pk_fill,
                          void *stream) {
  return sgb_spconv_forward_tc_ex(d_in_pk, in_stride, Min, d_map, K, Mout, d_Wp, Cin, Cout, d_residual, res_stride, res_off, d_bias,
                                  d_out, out_stride, out_off, d_pk_out, pk_stride, pk_coff, d_pk_scale, d_pk_shift, pk_relu, pk_fill,
                                  -1, stream);
}

int sgb_spconv_forward_tc_ex(const float *d_in_pk, int in_stride, int Min, const int32_t *d_map, int K, int Mout,
                             const float *d_Wp, int Cin, int Cout, const float *d_residual, int res_stride, int res_off,
                             const float *d_bias, float *d_out, int out_stride, int out_off, float *d_pk_out, int pk_stride,
                             int pk_coff, const float *d_pk_scale, const float *d_pk_shift, int pk_relu, int pk_fill, int kernel,
                             void *stream) {
  if (Mout == 0 || Cout == 0) return SGB_OK;
  SGB_REQUIRE(kernel >= -1 && kernel <= 1, SGB_ERR_ARG, "kernel: -1 (choose), 0 (one CTA per work item), 1 (persistent)");
  SGB_REQUIRE(d_in_pk && d_Wp && (d_out || d_pk_out) && K >= 1 && K <= 27 && Mout > 0 && Min > 0 && Cin > 0 && Cout > 0, SGB_ERR_ARG,
              "spconv_forward_tc arguments");
  SGB_REQUIRE(d_map || (K == 1 && Min >= Mout), SGB_ERR_ARG, "identity map requires K == 1");
  SGB_REQUIRE((in_stride & 31) == 0 && in_stride >= (Cin + 31) / 32 * 32, SGB_ERR_ARG, "packed input row stride (words, multiple of 32)");
  SGB_REQUIRE((((uintptr_t)d_in_pk) & 31) == 0, SGB_ERR_ARG, "packed input must be 32-byte aligned");
  SGB_REQUIRE(!d_out || out_stride >= out_off + Cout, SGB_ERR_ARG, "fp32 output row stride");
  SGB_REQUIRE(!d_pk_out || ((pk_stride & 31) == 0 && (pk_coff & 7) == 0 && pk_stride >= pk_coff + (Cout + 15) / 16 * 16), SGB_ERR_ARG,
              "packed output: row stride multiple of 32 words, channel offset multiple of 8");
  SGB_REQUIRE((d_pk_scale == nullptr) == (d_pk_shift == nullptr), SGB_ERR_ARG, "scale/shift must come together");
  const int N = (Cout + 15) / 16 * 16;
  SGB_REQUIRE(N <= 256 && Cin <= 512, SGB_ERR_RANGE, "spconv_forward_tc: Cout > 256 or Cin > 512 is not tiled");
  SGB_CURRENT_DEVICE(d);
  const bool persistent = kernel == 1 || (kernel == -1 && use_persistent(K, Mout, Cin, Cout, d->sms));
  TcArgs p;
  p.in = (const uint32_t *)d_in_pk; p.in_stride = in_stride;
  p.map = d_map; p.K = K; p.Mout = Mout;
  p.Wp = d_Wp; p.Cin = Cin; p.N = N; p.Cout = Cout;
  p.residual = d_residual; p.res_stride = res_stride; p.res_off = res_off;
  p.bias = d_bias;
  p.out = d_out; p.out_stride = out_stride; p.out_off = out_off;
  p.pk = (uint32_t *)d_pk_out; p.pk_stride = pk_stride; p.pk_coff = pk_coff;
  p.pk_scale = d_pk_scale; p.pk_shift = d_pk_shift; p.pk_relu = pk_relu; p.pk_fill = pk_fill;
  p.oflow = d->oflow;
  const int tiles = div_up(Mout, TC_ROWS);
  int NT;
  if (persistent) {
    NT = persistent_nt(N);
    p.ksplit = 1;
  } else {
    int plan[6];
    int rc = sgb_spconv_tc_plan(K, Mout, Cin, Cout, d_map != nullptr, d->sms, plan);
    if (rc) return rc;
    NT = plan[0];
    p.ksplit = plan[2];
  }
  p.nparts = div_up(N, NT);
  p.items = tiles * p.nparts;
  return launch(NT, p, persistent, *d, (cudaStream_t)stream);
}
}
