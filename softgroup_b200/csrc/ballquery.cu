// ballquery.cu -- ballquery_batch_p on a uniform-grid hash.
//
// Replaces the O(n * n_b) brute force of softgroup/ops/src/bfs_cluster/bfs_cluster.cu:15-66 with
//   (1) cell hash:   cell = floor(p / h), h = radius*(1+1e-4) in fp64; 64-bit key (segment, cx, cy, cz) ->
//                    open-addressing hash (atomicCAS); counts per cell; exclusive scan; scatter of
//                    (x,y,z,idx) records so every cell is one contiguous run of 16-byte records;
//   (2) query:       a persistent grid (one 1024-thread CTA per SM) pulls work items = (occupied cell, chunk of
//                    <= 128 queries of that cell). The <= 27 neighbouring runs are staged in shared memory and put
//                    in ascending point-index order in LINEAR time: a bitmap over the stencil's id range plus
//                    per-word prefix popcounts gives every record its rank (bitonic sort only when the id range
//                    does not fit the bitmap). Each query (one warp) then streams the staged candidates in index
//                    order in two passes: count (the ballot masks are kept in shared memory), one atomicAdd on
//                    the global cursor like the reference (:52), then a coalesced write of the hits -- the
//                    "first 1000 by index" cap (:43-48) is a loop exit. Stencils larger than the staging area
//                    fall back to an exact index-order scan of the whole segment.
// Routing of a work item (total_s = points in the stencil, nwords = its id range in 32-bit words):
//    pass 0, bitmap    total_s <= 5120    nwords <= 4096
//    pass 0, bitonic   total_s <= 4096    nwords >  4096
//    pass 1, bitmap    total_s <= 10240   nwords <= 8192   (items pass 0 did not take)
//    pass 1, bitonic   total_s <= 8192    nwords >  8192
//    exact scan        everything else
// The bitonic sort pads the stencil to P = pow2 >= total_s records, so it runs only where P fits the staging area
// (total_s <= kSortMax); a wider stencil goes on to the next configuration. tests/neighbour_cases.py restates this
// routing on the CPU.
// Exactness: the distance is evaluated with the reference's compiled contraction order
//   d2 = fma(dz,dz, fma(dx,dx, dy*dy)),  hit iff d2 < radius*radius   (strict, fp32)
// and any pair with d2 < r^2 differs by < h in every coordinate, so it lies in the 27-cell stencil.
// List placement uses an atomic cursor like the reference (:52) -- per-point lists are deterministic,
// the global layout is not.
#include <algorithm>

#include "common.cuh"

namespace sgb {

// Two 512-thread CTAs per SM (round 1 ran one 1024-thread CTA with a 160 KB staging area): the CTA-wide barriers of the
// staging / ordering phases were the largest stall reason -- with two CTAs one stages while the other queries, and each
// barrier spans half as many warps.
// Pass 0 of the query: 512-thread CTAs, two per SM, 5120 staged candidates (80 KB) each. Work items whose stencil is
// larger (the core cells of collapsed objects: several thousand candidates) are only NOTED in pass 0 and processed by
// pass 1: one 1024-thread CTA per SM with a 10240-candidate staging area (the round-1 configuration). The small
// configuration alone is faster on fragmented predictions but slower on the clean 40-object scan, whose cores overflow
// into the exact-scan path.
template <int PASS> struct BqCfg;
// kSortMax: the largest power of two <= kSMax, the most records the bitonic fallback can pad and sort in S[].
template <> struct BqCfg<0> { static constexpr int kThreads = 512, kSMax = 5120, kSortMax = 4096, kBmWords = 4096, kPerSM = 2; };
template <> struct BqCfg<1> { static constexpr int kThreads = 1024, kSMax = 10240, kSortMax = 8192, kBmWords = 8192, kPerSM = 1; };
template <int PASS> constexpr bool bq_sort_max_ok() {
  constexpr int m = BqCfg<PASS>::kSortMax, s = BqCfg<PASS>::kSMax;
  return (m & (m - 1)) == 0 && m <= s && 2 * m > s;
}
static_assert(bq_sort_max_ok<0>() && bq_sort_max_ok<1>(), "kSortMax must be the largest power of two <= kSMax");
constexpr int kCellBias = 131072;
constexpr int kMaxSeg = 1023;

struct BqWs {
  unsigned long long *keys;  // [cap]
  int32_t *slot_cnt;         // [cap]
  int32_t *slot_start;       // [cap]
  int32_t *slot_fill;        // [cap]
  int32_t *slot_lo, *slot_hi;  // [cap] smallest / largest point index of the cell (the id range of a stencil without a pass over it)
  int32_t *cell_slot;        // [n] cell id -> slot
  int32_t *cell_cnt;         // [n] -> scanned in place to starts
  int32_t *slot_of;          // [n]
  float4 *sorted;            // [n] (x,y,z,idx)
  int32_t *chunk_cell;       // [2n] work item -> cell id
  int32_t *chunk_q0;         // [2n] work item -> first query of the cell handled by this item
  int32_t *big_items;        // [2n] work items pass 0 left to pass 1 (count in scalars[5])
  int32_t *scalars;          // 0: ncells, 1: work counter, 2: error flag, 3: total, 4: items, 5: big items, 6: pass-1 counter
  int32_t *scan_tmp;
  uint32_t cap;
};

static size_t bq_cap(int n) { return pow2_at_least((size_t)std::max(n, 1) * 2); }

static bool bq_carve(void *ws, size_t bytes, int n, BqWs &w) {
  Arena a(ws, bytes);
  w.cap = (uint32_t)bq_cap(n);
  w.scalars = a.take<int32_t>(64);
  w.keys = a.take<unsigned long long>(w.cap);
  w.slot_cnt = a.take<int32_t>(w.cap);
  w.slot_start = a.take<int32_t>(w.cap);
  w.slot_fill = a.take<int32_t>(w.cap);
  w.slot_lo = a.take<int32_t>(w.cap);
  w.slot_hi = a.take<int32_t>(w.cap);
  w.cell_slot = a.take<int32_t>((size_t)n + 1);
  w.cell_cnt = a.take<int32_t>((size_t)n + 1);
  w.slot_of = a.take<int32_t>((size_t)n + 1);
  w.sorted = a.take<float4>((size_t)n + 1);
  w.chunk_cell = a.take<int32_t>(2 * (size_t)n + 2);
  w.chunk_q0 = a.take<int32_t>(2 * (size_t)n + 2);
  w.big_items = a.take<int32_t>(2 * (size_t)n + 2);
  w.scan_tmp = a.take<int32_t>(scan_temp_elems((size_t)n + 1));
  return w.scan_tmp != nullptr;
}

__device__ __forceinline__ unsigned long long cell_key(int seg, int cx, int cy, int cz) {
  return ((unsigned long long)seg << 54) | ((unsigned long long)(cx + kCellBias) << 36) |
         ((unsigned long long)(cy + kCellBias) << 18) | (unsigned long long)(cz + kCellBias);
}

// A point that is not hashed (NaN / Inf coordinate, or outside the addressable cell range) gets the empty list
// start_len = (0, 0) here and is never a candidate of anybody else. For NaN / Inf that IS the reference's result:
// every distance to or from such a point is NaN or +Inf, so `d2 < r2` never holds, not even with itself
// (bfs_cluster.cu:38-44). A finite coordinate beyond +-131070 cells, or a segment id outside [0, 1023], is a limit of
// this implementation: it raises the error flag scalars[2], reported as SGB_ERR_RANGE at the caller's next sync.
__global__ void bq_insert_kernel(const float *__restrict__ xyz, const int32_t *__restrict__ batch_idxs, int n,
                                 double inv_h, int32_t *__restrict__ start_len, BqWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
  double fx = floor((double)x * inv_h);
  double fy = floor((double)y * inv_h);
  double fz = floor((double)z * inv_h);
  int seg = batch_idxs[i];
  const double lim = (double)(kCellBias - 2);
  if (!(fabs(fx) < lim && fabs(fy) < lim && fabs(fz) < lim) || seg < 0 || seg > kMaxSeg) {
    const bool nonfinite = !(isfinite(x) && isfinite(y) && isfinite(z));
    if (!nonfinite || seg < 0 || seg > kMaxSeg) w.scalars[2] = 1;
    w.slot_of[i] = -1;
    start_len[2 * (size_t)i] = 0;
    start_len[2 * (size_t)i + 1] = 0;
    return;
  }
  unsigned long long key = cell_key(seg, (int)fx, (int)fy, (int)fz);
  uint32_t mask = w.cap - 1;
  uint32_t s = hash64(key) & mask;
  while (true) {
    unsigned long long cur = w.keys[s];
    if (cur == key) break;
    if (cur == kEmptyKey) {
      unsigned long long old = atomicCAS(&w.keys[s], kEmptyKey, key);
      if (old == kEmptyKey) {
        int id = atomicAdd(&w.scalars[0], 1);
        w.cell_slot[id] = (int32_t)s;
        break;
      }
      if (old == key) break;
    }
    s = (s + 1) & mask;
  }
  w.slot_of[i] = (int32_t)s;
  atomicAdd(&w.slot_cnt[s], 1);
  atomicMin(&w.slot_lo[s], i);
  atomicMax(&w.slot_hi[s], i);
}

__global__ void bq_cellcnt_kernel(int n, BqWs w) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  w.cell_cnt[c] = (c < w.scalars[0]) ? w.slot_cnt[w.cell_slot[c]] : 0;
}

constexpr int kBqChunk = 128;  // queries per work item: dense cells (hundreds to thousands of queries sharing one
                              // stencil) are cut into several items so a single SM never owns a whole object core

__global__ void bq_cellstart_kernel(int n, BqWs w) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= w.scalars[0]) return;
  const int slot = w.cell_slot[c];
  w.slot_start[slot] = w.cell_cnt[c];
  const int q = w.slot_cnt[slot];
  const int nch = (q + kBqChunk - 1) / kBqChunk;
  const int base = atomicAdd(&w.scalars[4], nch);
  for (int k = 0; k < nch; k++) {
    w.chunk_cell[base + k] = c;
    w.chunk_q0[base + k] = k * kBqChunk;
  }
}

__global__ void bq_scatter_kernel(const float *__restrict__ xyz, int n, BqWs w) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int s = w.slot_of[i];
  if (s < 0) return;
  int pos = w.slot_start[s] + atomicAdd(&w.slot_fill[s], 1);
  w.sorted[pos] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], __int_as_float(i));
}

__device__ __forceinline__ bool bq_hit(float qx, float qy, float qz, float x, float y, float z, float r2) {
  float dx = __fsub_rn(qx, x), dy = __fsub_rn(qy, y), dz = __fsub_rn(qz, z);
  float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
  return d2 < r2;
}

// The list cursor w.scalars[3] is int32 like the reference's. A neighbour total beyond 2^31 - 1 wraps it: the list that
// crosses 2^31 - 1 raises bit 2 of the error flag, and every later (negative) base writes nothing -- the lists are then
// incomplete, and the flag makes the caller's next synchronisation fail instead of clustering them. Below the limit
// nothing changes: a base is never negative and the crossing never happens.
__device__ __forceinline__ void bq_check_cursor(int base, int cnt, const BqWs &w) {
  if (base < 0 || (long long)base + cnt > 0x7fffffffll) atomicOr(&w.scalars[2], 2);
}

// Emit one query's list: staged hits (ascending) -> global, reference truncation rules (bfs_cluster.cu:52-65).
__device__ __forceinline__ void bq_emit(int qi, int cnt, const int32_t *stage, int32_t *__restrict__ idx,
                                        int32_t *__restrict__ start_len, int32_t *total, long long capacity, int lane) {
  int base = 0;
  if (lane == 0) {
    base = atomicAdd(total, cnt);
    start_len[2 * (size_t)qi] = base;
    start_len[2 * (size_t)qi + 1] = cnt;
  }
  base = __shfl_sync(0xffffffffu, base, 0);
  if ((long long)base >= capacity) return;
  int cw = cnt;
  if ((long long)base + cnt >= capacity) cw = (int)(capacity - base);
  for (int k = lane; k < cw; k += 32) idx[(size_t)base + k] = stage[k];
}

template <int PASS>
__global__ void __launch_bounds__(BqCfg<PASS>::kThreads, BqCfg<PASS>::kPerSM) bq_query_kernel(const float *__restrict__ xyz,
                                                              const int32_t *__restrict__ batch_idxs,
                                                              const int32_t *__restrict__ batch_offsets, int n,
                                                              float radius, long long capacity,
                                                              int32_t *__restrict__ idx,
                                                              int32_t *__restrict__ start_len, BqWs w) {
  constexpr int kBqThreads = BqCfg<PASS>::kThreads, kBqWarps = kBqThreads / 32, kBqSMax = BqCfg<PASS>::kSMax;
  constexpr int kBmWords = BqCfg<PASS>::kBmWords;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float4 *S = reinterpret_cast<float4 *>(smem_raw);  // [kBqSMax]
  uint32_t *bm = reinterpret_cast<uint32_t *>(smem_raw + sizeof(float4) * kBqSMax);                      // [kBmWords]
  unsigned short *pre = reinterpret_cast<unsigned short *>(smem_raw + sizeof(float4) * kBqSMax + 4 * kBmWords);  // [kBmWords]
  __shared__ int s_lo, s_hi, s_wsum[kBqThreads / 32];
  __shared__ int nb_start[27], nb_cnt[27], nb_off[28];
  __shared__ int s_cell;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float r2 = __fmul_rn(radius, radius);
  // pass 0 walks all work items; pass 1 the items pass 0 noted as too large for its staging area
  const int nitems = (PASS == 0) ? w.scalars[4] : w.scalars[5];

  while (true) {
    __syncthreads();
    if (tid == 0) s_cell = atomicAdd(&w.scalars[PASS == 0 ? 1 : 6], 1);
    __syncthreads();
    if (s_cell >= nitems) break;
    const int item = (PASS == 0) ? s_cell : w.big_items[s_cell];
    const int cell = w.chunk_cell[item];
    const int cslot = w.cell_slot[cell];
    const unsigned long long ckey = w.keys[cslot];
    if (tid < 27) {
      int seg = (int)(ckey >> 54);
      int cx = (int)((ckey >> 36) & 0x3FFFF) + (tid % 3) - 1;
      int cy = (int)((ckey >> 18) & 0x3FFFF) + ((tid / 3) % 3) - 1;
      int cz = (int)(ckey & 0x3FFFF) + (tid / 9) - 1;
      int st = 0, ct = 0, lo = 0x7fffffff, hi = -1;
      if (cx >= 0 && cy >= 0 && cz >= 0 && cx < 2 * kCellBias && cy < 2 * kCellBias && cz < 2 * kCellBias) {
        unsigned long long key = ((unsigned long long)seg << 54) | ((unsigned long long)cx << 36) |
                                 ((unsigned long long)cy << 18) | (unsigned long long)cz;
        uint32_t s = hash_find(w.keys, w.cap - 1, key);
        if (s != 0xFFFFFFFFu) { st = w.slot_start[s]; ct = w.slot_cnt[s]; lo = w.slot_lo[s]; hi = w.slot_hi[s]; }
      }
      nb_start[tid] = st;
      nb_cnt[tid] = ct;
      // id range of the whole stencil from the per-cell ranges kept by bq_insert_kernel (this used to be a pass over the
      // stencil's records in global memory between two CTA barriers, for every work item)
      lo = __reduce_min_sync(0x07ffffffu, lo);
      hi = __reduce_max_sync(0x07ffffffu, hi);
      if (tid == 0) { s_lo = lo; s_hi = hi; }
    }
    __syncthreads();
    if (tid == 0) {
      int acc = 0;
      for (int k = 0; k < 27; k++) { nb_off[k] = acc; acc += nb_cnt[k]; }
      nb_off[27] = acc;
    }
    __syncthreads();
    const int total_s = nb_off[27];
    const int q_first = w.chunk_q0[item];
    const int q_start = w.slot_start[cslot] + q_first, q_cnt = min(kBqChunk, w.slot_cnt[cslot] - q_first);
    const int lo = s_lo;
    const int nwords = (s_hi - lo + 32) >> 5;
    const bool use_bitmap = nwords <= kBmWords;
    // the bitonic fallback pads the stencil to a power of two >= total_s, which has to fit S[] too
    const bool staged = total_s <= (use_bitmap ? kBqSMax : BqCfg<PASS>::kSortMax);
    if (PASS == 0 && !staged) {  // too large for this configuration's staging area: left to pass 1
      if (tid == 0) w.big_items[atomicAdd(&w.scalars[5], 1)] = item;
      continue;
    }

    if (staged) {
      // ---- order the stencil by point index. Point indices are distinct, so the sorted position of a record is
      //      the number of stencil members with a smaller index: one bit per index in a shared-memory bitmap +
      //      prefix popcounts gives it in O(|S| + range/32) instead of an O(|S| log^2 |S|) bitonic sort.
      bool ordered = false;
      if (use_bitmap) {
        for (int t = tid; t < nwords; t += kBqThreads) bm[t] = 0u;
        __syncthreads();
        for (int k = 0; k < 27; k++) {
          int c = nb_cnt[k], st = nb_start[k];
          for (int t = tid; t < c; t += kBqThreads) {
            int d = __float_as_int(__ldg(&reinterpret_cast<const float *>(w.sorted + st + t)[3])) - lo;
            atomicOr(&bm[d >> 5], 1u << (d & 31));
          }
        }
        __syncthreads();
        {  // exclusive prefix of popcounts: 8 consecutive words per thread
          const int w0 = tid * 8;
          int loc[8], sum = 0;
#pragma unroll
          for (int e = 0; e < 8; e++) { loc[e] = sum; sum += (w0 + e < nwords) ? __popc(bm[w0 + e]) : 0; }
          int inc = sum;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            int t2 = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t2;
          }
          if (lane == 31) s_wsum[warp] = inc;
          __syncthreads();
          int woff = 0;
          for (int q = 0; q < warp; q++) woff += s_wsum[q];
          const int basep = woff + inc - sum;
#pragma unroll
          for (int e = 0; e < 8; e++)
            if (w0 + e < nwords) pre[w0 + e] = (unsigned short)(basep + loc[e]);
        }
        __syncthreads();
        for (int k = 0; k < 27; k++) {
          int c = nb_cnt[k], st = nb_start[k];
          for (int t = tid; t < c; t += kBqThreads) {
            float4 rec = w.sorted[st + t];
            int d = __float_as_int(rec.w) - lo;
            int pos = (int)pre[d >> 5] + __popc(bm[d >> 5] & ((1u << (d & 31)) - 1u));
            S[pos] = rec;
          }
        }
        __syncthreads();
        ordered = true;
      }
      if (!ordered) {
      // ---- index range too wide for the bitmap: stage the stencil and bitonic-sort it (P <= kSortMax) ----
      int P = 32;
      while (P < total_s) P <<= 1;
      for (int k = 0; k < 27; k++) {
        int c = nb_cnt[k], st = nb_start[k], o = nb_off[k];
        for (int t = tid; t < c; t += kBqThreads) S[o + t] = w.sorted[st + t];
      }
      for (int t = total_s + tid; t < P; t += kBqThreads) S[t] = make_float4(0.f, 0.f, 0.f, __int_as_float(0x7fffffff));
      __syncthreads();
      // bitonic sort by point index; every thread owns compare-exchange pairs (no idle half)
      for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
          for (int q = tid; q < (P >> 1); q += kBqThreads) {
            const int t = ((q & ~(j - 1)) << 1) | (q & (j - 1));
            const int u = t | j;
            float4 a = S[t], b = S[u];
            const bool asc = ((t & k) == 0);
            const bool gt = __float_as_int(a.w) > __float_as_int(b.w);
            if (gt == asc) { S[t] = b; S[u] = a; }
          }
          __syncthreads();
        }
      }
      }  // !ordered
      // ---- queries of this cell: one warp each ----------------------------------------------------
      // The two loops below are most of the kernel's instructions: they run on raw
      // 32-bit shared-memory addresses (the generic-pointer form re-derived the shared window base in every iteration) and
      // without a bounds test -- the staged stencil is padded to a multiple of 32 with records that can never hit (NaN).
      const int total_pad = (total_s + 31) & ~31;
      for (int t = total_s + tid; t < total_pad; t += kBqThreads)
        S[t] = make_float4(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fffffff));
      __syncthreads();
      const uint32_t s_addr = (uint32_t)__cvta_generic_to_shared(S);
      const uint32_t m_addr = (uint32_t)__cvta_generic_to_shared(bm + warp * (kBqSMax / 32));  // this warp's ballot masks
      const unsigned lt_mask = (1u << lane) - 1u;
      const int nblk = total_pad >> 5;
      for (int q = warp; q < q_cnt; q += kBqWarps) {
        const float4 qp = w.sorted[q_start + q];
        const int qi = __float_as_int(qp.w);
        // pass 1: count (first 1000 by index); pass 2: write straight to the reserved global range. The candidates
        // sit in shared memory, so scanning twice is cheaper than staging 4 KB per warp (which would cap the CTA at
        // 8 warps and quadruple the per-cell sort time). The ballot masks of pass 1 are kept in the (now idle) bitmap
        // area, one word per 32 candidates, so pass 2 does not recompute distances and only touches the index word of
        // actual hits.
        int cnt = 0, nb = 0;
        uint32_t ca = s_addr + (uint32_t)lane * 16u;
        // two blocks of 32 candidates per trip (a block counted beyond the cap only leaves an unused mask behind: pass 2
        // stops after `cnt` hits)
        while (nb + 1 < nblk && cnt < SGB_MAX_NEIGHBORS) {
          float ax, ay, az, aw, bx, by, bz, bw;
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(ax), "=f"(ay), "=f"(az), "=f"(aw) : "r"(ca));
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(bx), "=f"(by), "=f"(bz), "=f"(bw) : "r"(ca + 512u));
          const unsigned m0 = __ballot_sync(0xffffffffu, bq_hit(qp.x, qp.y, qp.z, ax, ay, az, r2));
          const unsigned m1 = __ballot_sync(0xffffffffu, bq_hit(qp.x, qp.y, qp.z, bx, by, bz, r2));
          if (lane == 0) asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(m_addr + (uint32_t)nb * 4u), "r"(m0), "r"(m1) : "memory");
          cnt = min(cnt + __popc(m0) + __popc(m1), SGB_MAX_NEIGHBORS);
          nb += 2;
          ca += 1024u;
        }
        while (nb < nblk && cnt < SGB_MAX_NEIGHBORS) {
          float cx, cy, cz, cwv;
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(cx), "=f"(cy), "=f"(cz), "=f"(cwv) : "r"(ca));
          const unsigned m = __ballot_sync(0xffffffffu, bq_hit(qp.x, qp.y, qp.z, cx, cy, cz, r2));
          if (lane == 0) asm volatile("st.shared.u32 [%0], %1;" ::"r"(m_addr + (uint32_t)nb * 4u), "r"(m) : "memory");
          cnt = min(cnt + __popc(m), SGB_MAX_NEIGHBORS);
          nb++;
          ca += 512u;
        }
        __syncwarp();
        int base = 0;
        if (lane == 0) {
          base = atomicAdd(&w.scalars[3], cnt);
          start_len[2 * (size_t)qi] = base;
          start_len[2 * (size_t)qi + 1] = cnt;
        }
        base = __shfl_sync(0xffffffffu, base, 0);
        if (lane == 0) bq_check_cursor(base, cnt, w);
        const long long room = capacity - (long long)base;  // reference truncation (bfs_cluster.cu:55-61)
        const int cw = (base < 0 || room <= 0) ? 0 : (((long long)base + cnt >= capacity) ? (int)room : cnt);
        int32_t *__restrict__ out = idx + base;
        int done = 0;
        uint32_t wa = s_addr + (uint32_t)lane * 16u + 12u;  // the index word of this lane's candidate
        for (int b = 0; b < nb && done < cw; b++) {
          unsigned m;
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(m) : "r"(m_addr + (uint32_t)b * 4u));
          const int pos = done + __popc(m & lt_mask);
          if (((m >> lane) & 1u) && pos < cw) {
            int id;
            asm volatile("ld.shared.s32 %0, [%1];" : "=r"(id) : "r"(wa));
            out[pos] = id;
          }
          done += __popc(m);
          wa += 512u;
        }
        __syncwarp();
      }
    } else {
      // ---- stencil beyond pass 1's staging area: exact index-order scan of the segment ---------------
      for (int q = warp; q < q_cnt; q += kBqWarps) {
        float4 qp = w.sorted[q_start + q];
        int qi = __float_as_int(qp.w);
        int b = batch_idxs[qi];
        int s0 = batch_offsets[b], e0 = batch_offsets[b + 1];
        int cnt = 0, last = s0;
        for (int b0 = s0; b0 < e0 && cnt < SGB_MAX_NEIGHBORS; b0 += 32) {
          int t = b0 + lane;
          bool hit = false;
          if (t < e0) hit = bq_hit(qp.x, qp.y, qp.z, xyz[3 * (size_t)t], xyz[3 * (size_t)t + 1], xyz[3 * (size_t)t + 2], r2);
          cnt = min(cnt + __popc(__ballot_sync(0xffffffffu, hit)), SGB_MAX_NEIGHBORS);
          last = b0 + 32;
        }
        int base = 0;
        if (lane == 0) {
          base = atomicAdd(&w.scalars[3], cnt);
          start_len[2 * (size_t)qi] = base;
          start_len[2 * (size_t)qi + 1] = cnt;
        }
        base = __shfl_sync(0xffffffffu, base, 0);
        if (lane == 0) bq_check_cursor(base, cnt, w);
        long long room = capacity - (long long)base;
        int cw = (base < 0 || room <= 0) ? 0 : (((long long)base + cnt >= capacity) ? (int)room : cnt);
        int done = 0;
        for (int b0 = s0; b0 < last && done < cw; b0 += 32) {
          int t = b0 + lane;
          bool hit = false;
          if (t < e0) hit = bq_hit(qp.x, qp.y, qp.z, xyz[3 * (size_t)t], xyz[3 * (size_t)t + 1], xyz[3 * (size_t)t + 2], r2);
          unsigned m = __ballot_sync(0xffffffffu, hit);
          int pos = done + __popc(m & ((1u << lane) - 1));
          if (hit && pos < cw) idx[(size_t)base + pos] = t;
          done += __popc(m);
        }
      }
    }
  }
}

static DeviceOnce g_bq_once;  // the query kernels' shared-memory attributes are set

static int bq_launch(int n, long long capacity, float radius, const float *xyz, const int32_t *batch_idxs,
                     const int32_t *batch_offsets, int B, int32_t *idx, int32_t *start_len, void *ws, size_t ws_bytes,
                     cudaStream_t st, BqWs &w) {
  SGB_REQUIRE(n >= 0 && B >= 1 && B <= kMaxSeg && radius > 0.f, SGB_ERR_ARG, "ballquery arguments");
  SGB_REQUIRE(xyz && batch_idxs && batch_offsets && start_len && ws, SGB_ERR_ARG, "null pointer");
  SGB_REQUIRE(bq_carve(ws, ws_bytes, n, w), SGB_ERR_WORKSPACE, "ballquery workspace too small");
  constexpr size_t smem0 = sizeof(float4) * BqCfg<0>::kSMax + 6 * BqCfg<0>::kBmWords;
  constexpr size_t smem1 = sizeof(float4) * BqCfg<1>::kSMax + 6 * BqCfg<1>::kBmWords;
  SGB_CURRENT_DEVICE(d);
  int rc = once_per_device(g_bq_once, d->ordinal, [] {
    SGB_CUDA_CHECK(cudaFuncSetAttribute(bq_query_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem0));
    SGB_CUDA_CHECK(cudaFuncSetAttribute(bq_query_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
    return SGB_OK;
  });
  if (rc) return rc;
  SGB_CUDA_CHECK(cudaMemsetAsync(w.keys, 0xFF, (size_t)w.cap * 8, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.slot_cnt, 0, (size_t)w.cap * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.slot_fill, 0, (size_t)w.cap * 4, st));
  SGB_CUDA_CHECK(cudaMemsetAsync(w.slot_lo, 0x7f, (size_t)w.cap * 4, st));  // 0x7f7f7f7f: above every point index
  SGB_CUDA_CHECK(cudaMemsetAsync(w.slot_hi, 0xFF, (size_t)w.cap * 4, st));  // -1
  SGB_CUDA_CHECK(cudaMemsetAsync(w.scalars, 0, 64 * 4, st));
  double h = (double)radius * (1.0 + 1e-4);
  int nb = div_up(n, 256);
  bq_insert_kernel<<<nb, 256, 0, st>>>(xyz, batch_idxs, n, 1.0 / h, start_len, w);
  SGB_LAUNCH_CHECK();
  bq_cellcnt_kernel<<<nb, 256, 0, st>>>(n, w);
  SGB_LAUNCH_CHECK();
  rc = exclusive_scan_i32(w.cell_cnt, w.cell_cnt, (size_t)n, nullptr, w.scan_tmp, st);
  if (rc) return rc;
  bq_cellstart_kernel<<<nb, 256, 0, st>>>(n, w);
  SGB_LAUNCH_CHECK();
  bq_scatter_kernel<<<nb, 256, 0, st>>>(xyz, n, w);
  SGB_LAUNCH_CHECK();
  bq_query_kernel<0><<<std::min(std::max(n, 1), BqCfg<0>::kPerSM * d->sms), BqCfg<0>::kThreads, smem0, st>>>(
      xyz, batch_idxs, batch_offsets, n, radius, capacity, idx, start_len, w);
  SGB_LAUNCH_CHECK();
  // the items pass 0 noted (stencils of up to 10240 candidates stay on the staged path; beyond that the exact scan)
  bq_query_kernel<1><<<std::min(std::max(n, 1), d->sms), BqCfg<1>::kThreads, smem1, st>>>(xyz, batch_idxs, batch_offsets, n, radius,
                                                                                        capacity, idx, start_len, w);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_ballquery_workspace_bytes(int n) {
  if (n < 0) n = 0;
  size_t cap = bq_cap(n);
  size_t b = align_up(64 * 4) + align_up(cap * 8) + 5 * align_up(cap * 4) + 3 * align_up(((size_t)n + 1) * 4) +
             3 * align_up((2 * (size_t)n + 2) * 4) +
             align_up(((size_t)n + 1) * 16) + align_up(scan_temp_elems((size_t)n + 1) * 4);
  return b + 1024;
}

int sgb_ballquery_batch_p_async(int n, long long capacity, float radius, const float *d_xyz,
                                const int32_t *d_batch_idxs, const int32_t *d_batch_offsets, int B, int32_t *d_idx,
                                int32_t *d_start_len, int32_t *d_total, void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    if (d_total) SGB_CUDA_CHECK(cudaMemsetAsync(d_total, 0, 8, st));
    return SGB_OK;
  }
  SGB_REQUIRE(capacity == 0 || d_idx, SGB_ERR_ARG, "null idx");
  SGB_REQUIRE(capacity < (1ll << 31), SGB_ERR_RANGE, "ballquery: capacity must stay below 2^31 entries (int32 cursor and start_len)");
  BqWs w;
  int rc = bq_launch(n, capacity, radius, d_xyz, d_batch_idxs, d_batch_offsets, B, d_idx, d_start_len, d_ws, ws_bytes,
                     st, w);
  if (rc) return rc;
  // d_total[0] = sum of list lengths, d_total[1] = range-error flag (hand d_total + 1 to sgb_bfs_cluster_count, which
  // reports it at its own synchronisation: this entry point never waits for the device)
  if (d_total) {
    SGB_CUDA_CHECK(cudaMemcpyAsync(d_total, &w.scalars[3], 4, cudaMemcpyDeviceToDevice, st));
    SGB_CUDA_CHECK(cudaMemcpyAsync(d_total + 1, &w.scalars[2], 4, cudaMemcpyDeviceToDevice, st));
  }
  return SGB_OK;
}

long long sgb_ballquery_batch_p(int n, int meanActive, float radius, const float *d_xyz, const int32_t *d_batch_idxs,
                                const int32_t *d_batch_offsets, int B, int32_t *d_idx, int32_t *d_start_len,
                                void *d_ws, size_t ws_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  SGB_REQUIRE(meanActive >= 0, SGB_ERR_ARG, "meanActive");
  BqWs w;
  int rc = bq_launch(n, (long long)n * meanActive, radius, d_xyz, d_batch_idxs, d_batch_offsets, B, d_idx,
                     d_start_len, d_ws, ws_bytes, st, w);
  if (rc) return rc;
  int h[4];
  SGB_CUDA_CHECK(cudaMemcpyAsync(h, w.scalars, sizeof(h), cudaMemcpyDeviceToHost, st));
  SGB_CUDA_CHECK(cudaStreamSynchronize(st));
  SGB_REQUIRE((h[2] & 1) == 0, SGB_ERR_RANGE, "ballquery: |xyz/radius| >= 131070 or batch index outside [0,1023]");
  SGB_REQUIRE(h[2] == 0, SGB_ERR_RANGE, "ballquery: neighbour total beyond 2^31 - 1 (int32 list cursor)");
  return (long long)h[3];
}
}
