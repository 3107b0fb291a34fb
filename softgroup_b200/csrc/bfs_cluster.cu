// bfs_cluster.cu -- soft-grouping clustering on the GPU, bit-exact with the reference's sequential BFS
// (softgroup/ops/src/bfs_cluster/bfs_cluster.cpp:33-126).
//
// The reference visits i = 0..N-1, starts a std::queue BFS from every unvisited i over the DIRECTED list graph
// and keeps components with (int)size >= thr; cluster_idxs is in BFS visitation order, clusters in seed order.
// Parallel restatement (SURVEY.md H1; validated against the compiled reference in tests/):
//   (1) label[v] = min index among all nodes that can reach v (v included). That node is exactly the seed whose
//       BFS claims v: it has no smaller ancestor, so it is unvisited when the outer loop reaches it, and no node on
//       its path to v can have been claimed earlier. Computed by min-propagation along directed edges with pointer
//       jumping (label[label[v]] is again an ancestor) until a pass changes nothing.
//   (2) sizes per label (warp-aggregated atomics) -> threshold -> one packed int64 exclusive scan gives every kept
//       seed its cluster id (rank among kept seeds = ascending seed order) and its output offset.
//   (3) one CTA per kept cluster replays the BFS level-synchronously. Queue order is reproduced with a 64-bit
//       atomicMin key per node: key[v] = min over parents u listing v of (queue position of u, slot of v in u's
//       list). The winning parent is the first discoverer; children of one parent keep list order; parents keep
//       queue order -> next level = concatenation over parents (in queue order) of their won children (in list
//       order), placed with a block scan of per-parent win counts. No sort is needed.
#include <algorithm>

#include "common.cuh"

namespace sgb {

struct BfsWs {
  int32_t *label;      // [N]
  int32_t *size;       // [N] component size at the seed
  long long *packed;   // [N] keep ? (1<<32 | size) : 0  -> exclusive scan
  unsigned long long *key;  // [N]
  int32_t *root_of;    // [N] cluster id -> seed
  int32_t *wins;       // [N] per queue position
  int32_t *cid_of;     // [N] seed -> cluster id (kept) or -1
  int32_t *members;    // [N] nodes of kept clusters, grouped by cluster (unordered inside)
  int32_t *cursor;     // [N] per-cluster fill cursor / per-cluster level totals
  int32_t *scalars;    // [64] 0: changed flag, 1: max list length, 8..19: pass flags, 32..43: frontier queue lengths
  long long *totals;   // [1] packed total
  long long *scan_tmp;
};

static bool bfs_carve(void *ws, size_t bytes, int N, BfsWs &w) {
  Arena a(ws, bytes);
  size_t n1 = (size_t)N + 1;
  w.scalars = a.take<int32_t>(64);
  w.totals = a.take<long long>(8);
  w.label = a.take<int32_t>(n1);
  w.size = a.take<int32_t>(n1);
  w.packed = a.take<long long>(n1);
  w.key = a.take<unsigned long long>(n1);
  w.root_of = a.take<int32_t>(n1);
  w.wins = a.take<int32_t>(n1);
  w.cid_of = a.take<int32_t>(n1);
  w.members = a.take<int32_t>(n1);
  w.cursor = a.take<int32_t>(n1);
  w.scan_tmp = a.take<long long>(scan_temp_elems(n1));
  return w.scan_tmp != nullptr;
}

__global__ void bfs_init_kernel(int N, BfsWs w) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  w.label[v] = v;
  w.size[v] = 0;
}

// L1-cached read of a word that other CTAs lower with atomics during the same kernel (ld.global.ca): the value may be
// STALE, i.e. higher than the current one (labels and claim keys only ever decrease) -- the caller then merely issues an
// atomicMin that the memory system resolves. Neighbour lists stay inside one object (a few thousand nodes, tens of KB),
// so these reads hit L1 instead of paying an L2 round trip per edge.
__device__ __forceinline__ int32_t ld_ca_i32(const int32_t *p) {
  int32_t v;
  asm volatile("ld.global.ca.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ unsigned long long ld_ca_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.global.ca.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}

// Label propagation (frontier iteration), two kernels per pass.
//   select: one THREAD per node chases its label (pointer jumping: an ancestor's label is an ancestor too) and decides
//           whether the node has something new to tell its out-neighbours -- its chased label is lower than the one it
//           pushed last time (`w.wins`, idle until the emit phase, keeps the last pushed label). Such nodes go into a
//           queue (node, label to push).
//   push:   one WARP per queue entry pushes the label to every listed node (4 bytes per edge are read once per CHANGE of the
//           source label instead of once per pass).
// Both steps once ran in one kernel with a static node -> warp mapping; passes 2-3 of a 150k-point scan, where 40 %
// resp. 2 % of the nodes are active, then took longer than the pass that reads EVERY list (a few warps with seven
// 1000-entry lists each while the others idle). Queue entries cost the same
// (~1000 edges each), so a strided walk over the queue is balanced.
// The pass in which nobody is selected ends the iteration: then label[v] <= pushed[u] <= label[u] for every edge u->v,
// the fixed point of the full iteration. Passes are enqueued in batches without a host round trip: pass `it` raises
// flags[it] when it selected anything and returns at once when pass it-1 did not. The queue lives in arrays the emit
// phase owns later (members = node, cid_of = label); the entry count of pass `it` in scalars[32 + it].
__global__ void bfs_frontier_select_kernel(int N, BfsWs w, int it, int cont, int32_t *__restrict__ flags) {
  if (it > 0 && *(volatile int32_t *)&flags[it - 1] == 0) return;
  const int first_pass = it == 0 && !cont;  // cont: a later batch continues the iteration (w.wins is valid)
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  volatile int32_t *label = w.label;
  bool active = false;
  int lu = 0;
  if (u < N) {
    const int l0 = label[u];
    lu = l0;
    while (true) {
      const int l2 = label[lu];
      if (l2 >= lu) break;
      lu = l2;
    }
    if (lu < l0) atomicMin(&w.label[u], lu);
    const int prev = first_pass ? 0x7fffffff : *(volatile int32_t *)&w.wins[u];
    active = lu < prev;
  }
  const unsigned m = __ballot_sync(0xffffffffu, active);
  if (!m) return;
  int base = 0;
  if (lane == 0) base = atomicAdd(&w.scalars[32 + it], __popc(m));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (active) {
    const int pos = base + __popc(m & ((1u << lane) - 1u));
    w.members[pos] = u;
    w.cid_of[pos] = lu;
    w.wins[u] = lu;  // what the push kernel of this pass tells the neighbours
  }
  if (lane == 0) flags[it] = 1;
}

__global__ void bfs_frontier_push_kernel(const int32_t *__restrict__ idxs, const int32_t *__restrict__ start_len, BfsWs w, int it,
                                         const int32_t *__restrict__ flags) {
  if (*(volatile const int32_t *)&flags[it] == 0) return;  // nothing selected in this pass (or the iteration ended earlier)
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int count = *(volatile int32_t *)&w.scalars[32 + it];
  for (int e = warp; e < count; e += nwarps) {
    const int u = w.members[e], lu = w.cid_of[e];
    const int s = __ldg(&start_len[2 * (size_t)u]), l = __ldg(&start_len[2 * (size_t)u + 1]);
    // four independent (index, label) load pairs in flight per lane: the loop is latency bound (a list entry, then the
    // label it points to), not bandwidth bound
    for (int j0 = 0; j0 < l; j0 += 128) {
      int v[4], lv[4];
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const int j = j0 + t * 32 + lane;
        v[t] = (j < l) ? __ldg(&idxs[(size_t)s + j]) : -1;
      }
#pragma unroll
      for (int t = 0; t < 4; t++) lv[t] = (v[t] >= 0) ? ld_ca_i32(&w.label[v[t]]) : 0;
#pragma unroll
      for (int t = 0; t < 4; t++)
        if (v[t] >= 0 && lv[t] > lu) atomicMin(&w.label[v[t]], lu);  // a stale (higher) value only costs a redundant atomic
    }
  }
}

__global__ void bfs_size_kernel(int N, const int32_t *__restrict__ start_len, BfsWs w) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  bool active = v < N;
  int len = active ? __ldg(&start_len[2 * (size_t)v + 1]) : 0;
  len = __reduce_max_sync(0xffffffffu, len);
  if ((threadIdx.x & 31) == 0 && len > *(volatile int32_t *)&w.scalars[1]) atomicMax(&w.scalars[1], len);
  int l = active ? w.label[v] : -1;
  unsigned am = __ballot_sync(0xffffffffu, active);
  if (!active) return;
  unsigned peers = __match_any_sync(am, l);
  int leader = __ffs(peers) - 1;
  if ((threadIdx.x & 31) == leader) atomicAdd(&w.size[l], __popc(peers));
}

__global__ void bfs_pack_kernel(int N, float thr, const int32_t *__restrict__ node_seg,
                                const float *__restrict__ seg_thr, BfsWs w) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  long long p = 0;
  if (w.label[v] == v) {
    float t = node_seg ? seg_thr[node_seg[v]] : thr;
    int sz = w.size[v];
    if ((float)sz >= t) p = (1ll << 32) | (long long)sz;  // `(int)CC.pt_idxs.size() >= thr` (bfs_cluster.cpp:78)
  }
  w.packed[v] = p;
}

__global__ void bfs_roots_kernel(int N, int nCluster, int sumNPoint, int32_t *__restrict__ cluster_offsets, BfsWs w) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v == 0) cluster_offsets[nCluster] = sumNPoint;
  if (v >= N) return;
  int cid = -1;
  if (w.label[v] == v) {
    long long p = w.packed[v];
    // a seed is kept iff the exclusive prefix grows by one cluster after it
    long long nxt = (v + 1 < N) ? w.packed[v + 1] : w.totals[0];
    if ((nxt - p) >> 32) {
      int c = (int)(p >> 32);
      w.root_of[c] = v;
      cluster_offsets[c] = (int)(p & 0xFFFFFFFFll);
      cid = c;
    }
  }
  w.cid_of[v] = cid;
}

// members of kept clusters grouped by cluster (order inside a group is irrelevant); key = "unvisited, label"
__global__ void bfs_members_kernel(int N, const int32_t *__restrict__ cluster_offsets, BfsWs w) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  int c = -1;
  if (v < N) {
    int l = w.label[v];
    w.key[v] = (0xFFFFFFFFull << 32) | (unsigned long long)(unsigned)l;
    c = w.cid_of[l];
  }
  // one atomic per (warp, cluster): consecutive nodes mostly belong to the same few components, and 131k single adds on
  // 40 cursor words serialised in L2
  const int lane = threadIdx.x & 31;
  const unsigned peers = __match_any_sync(0xffffffffu, c);
  if (c < 0) return;
  const int leader = __ffs(peers) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(&w.cursor[c], __popc(peers));
  base = __shfl_sync(peers, base, leader);
  w.members[cluster_offsets[c] + base + __popc(peers & ((1u << lane) - 1u))] = v;
}

constexpr int kEmitThreads = 256;

__global__ void __launch_bounds__(kEmitThreads) bfs_emit_kernel(const int32_t *__restrict__ idxs,
                                                                const int32_t *__restrict__ start_len,
                                                                const int32_t *__restrict__ cluster_offsets,
                                                                int32_t *__restrict__ cluster_idxs, BfsWs w) {
  const int c = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int nwarps = kEmitThreads / 32;
  const int seed = w.root_of[c];
  const int base = cluster_offsets[c];
  int32_t *order = cluster_idxs + 2 * (size_t)base;  // order[2*p+1] = p-th visited node
  int32_t *wins = w.wins + base;
  __shared__ int s_warp[nwarps];
  __shared__ int s_carry, s_total;

  if (tid == 0) {
    w.key[seed] = 0ull;
    order[0] = c;
    order[1] = seed;
  }
  __syncthreads();
  int a = 0, b = 1;
  while (true) {
    // ---- A: claim ------------------------------------------------------------------------------
    for (int p = a + warp; p < b; p += nwarps) {
      int u = __ldcg(&order[2 * (size_t)p + 1]);
      int s = __ldg(&start_len[2 * (size_t)u]), l = __ldg(&start_len[2 * (size_t)u + 1]);
      unsigned long long hi = (unsigned long long)(p + 1) << 32;
      for (int j = lane; j < l; j += 32) {
        int v = __ldg(&idxs[(size_t)s + j]);
        if (__ldg(&w.label[v]) == seed) atomicMin(&w.key[v], hi | (unsigned)j);
      }
    }
    __syncthreads();
    // ---- B: count wins per parent --------------------------------------------------------------
    for (int p = a + warp; p < b; p += nwarps) {
      int u = __ldcg(&order[2 * (size_t)p + 1]);
      int s = __ldg(&start_len[2 * (size_t)u]), l = __ldg(&start_len[2 * (size_t)u + 1]);
      unsigned long long hi = (unsigned long long)(p + 1) << 32;
      int cnt = 0;
      for (int j0 = 0; j0 < l; j0 += 32) {
        int j = j0 + lane;
        bool win = false;
        if (j < l) {
          int v = __ldg(&idxs[(size_t)s + j]);
          win = (__ldcg(&w.key[v]) == (hi | (unsigned)j));
        }
        cnt += __popc(__ballot_sync(0xffffffffu, win));
      }
      if (lane == 0) wins[p] = cnt;
    }
    if (tid == 0) s_carry = 0;
    __syncthreads();
    // ---- exclusive scan of wins[a..b) ----------------------------------------------------------
    for (int p0 = a; p0 < b; p0 += kEmitThreads) {
      int p = p0 + tid;
      int x = (p < b) ? __ldcg(&wins[p]) : 0;
      int inc = x;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      if (lane == 31) s_warp[warp] = inc;
      __syncthreads();
      int woff = 0;
      for (int k = 0; k < warp; k++) woff += s_warp[k];
      int carry = s_carry;
      if (p < b) wins[p] = carry + woff + inc - x;
      __syncthreads();
      if (tid == kEmitThreads - 1) s_carry = carry + woff + inc;
      __syncthreads();
    }
    if (tid == 0) s_total = s_carry;
    __syncthreads();
    const int total = s_total;
    if (total == 0) break;
    // ---- C: write won children in (parent queue order, list order) ------------------------------
    for (int p = a + warp; p < b; p += nwarps) {
      int u = __ldcg(&order[2 * (size_t)p + 1]);
      int s = __ldg(&start_len[2 * (size_t)u]), l = __ldg(&start_len[2 * (size_t)u + 1]);
      unsigned long long hi = (unsigned long long)(p + 1) << 32;
      int run = b + __ldcg(&wins[p]);
      for (int j0 = 0; j0 < l; j0 += 32) {
        int j = j0 + lane;
        bool win = false;
        int v = 0;
        if (j < l) {
          v = __ldg(&idxs[(size_t)s + j]);
          win = (__ldcg(&w.key[v]) == (hi | (unsigned)j));
        }
        unsigned m = __ballot_sync(0xffffffffu, win);
        if (win) {
          int pos = run + __popc(m & ((1u << lane) - 1));
          order[2 * (size_t)pos] = c;
          order[2 * (size_t)pos + 1] = v;
        }
        run += __popc(m);
      }
    }
    __syncthreads();
    a = b;
    b += total;
  }
}


// ---------------------------------------------------------------------------------------------------------
// emit v2: one THREAD-BLOCK CLUSTER (8 CTAs, hardware barrier.cluster) per component, one pass over the edges
// per BFS level.
//   A  (edges of the frontier, all warps of the cluster): one 8-byte L2 read of key[v] per edge; key[v] holds
//      either "unvisited | label" or the best (parent position, list slot) claim so far; claim with atomicMin
//      only when it improves. Nodes of other components are told apart by the label half of the unvisited key.
//   B' (members of the component, not edges): nodes claimed in this level set bit `slot` in their parent's bitmap
//      row (rows are indexed by queue position; every position is a parent exactly once, so the bitmap is cleared
//      once per call).
//   counts = popcount per row -> exclusive scan over the frontier (CTA 0) -> C': every claimed node is written at
//      b + offset(parent) + #set bits below its slot: queue order = (parent position, list slot), no sort.
// ---------------------------------------------------------------------------------------------------------
constexpr int kCl = 8;          // CTAs per cluster (portable maximum)
constexpr int kClThreads = 512;

__device__ __forceinline__ void cluster_sync_all() {
  __threadfence();
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(kClThreads)
    bfs_emit2_kernel(const int32_t *__restrict__ idxs, const int32_t *__restrict__ start_len,
                     const int32_t *__restrict__ cluster_offsets, int32_t *__restrict__ cluster_idxs, int nCluster, int W,
                     uint32_t *__restrict__ bitmap, BfsWs w) {
  const int tid = threadIdx.x, lane = tid & 31;
  const int crank = (int)cluster_ctarank();
  const int cl_id = blockIdx.x / kCl, n_cl = gridDim.x / kCl;
  const int gtid = crank * kClThreads + tid, gthreads = kCl * kClThreads;
  const int gwarp = gtid >> 5, gwarps = gthreads >> 5;
  __shared__ int s_warp[kClThreads / 32];
  __shared__ int s_carry;

  for (int c = cl_id; c < nCluster; c += n_cl) {
    const int seed = w.root_of[c];
    const int base = cluster_offsets[c];
    const int size = cluster_offsets[c + 1] - base;
    int32_t *order = cluster_idxs + 2 * (size_t)base;
    int32_t *wins = w.wins + base;
    const int32_t *members = w.members + base;
    uint32_t *bm = bitmap + (size_t)base * W;
    if (gtid == 0) {
      w.key[seed] = 0ull;
      order[0] = c;
      order[1] = seed;
    }
    int a = 0, b = 1;
    while (true) {
      cluster_sync_all();
      // ---- A: claim over the edges of frontier [a,b) ---------------------------------------------------
      for (int p = a + gwarp; p < b; p += gwarps) {
        const int u = __ldcg(&order[2 * (size_t)p + 1]);
        const int s = __ldg(&start_len[2 * (size_t)u]), l = __ldg(&start_len[2 * (size_t)u + 1]);
        const unsigned long long hi = (unsigned long long)(p + 1) << 32;
        for (int j0 = 0; j0 < l; j0 += 128) {
          int v[4];
          unsigned long long k[4];
#pragma unroll
          for (int t = 0; t < 4; t++) {
            int j = j0 + t * 32 + lane;
            v[t] = (j < l) ? __ldg(&idxs[(size_t)s + j]) : -1;
          }
#pragma unroll
          for (int t = 0; t < 4; t++) k[t] = (v[t] >= 0) ? ld_ca_u64(&w.key[v[t]]) : 0ull;  // stale = higher: see ld_ca_*
#pragma unroll
          for (int t = 0; t < 4; t++) {
            if (v[t] < 0) continue;
            const unsigned long long mine = hi | (unsigned)(j0 + t * 32 + lane);
            if (k[t] > mine) {
              // Is v a node of THIS component? An unvisited key carries the label; a visited key does not -- and v may be a
              // node of ANOTHER component (a directed edge into a component with a smaller seed: lists cut by the 1000 cap)
              // that a different cluster is emitting right now, whose claim keys must not be lowered from here (round-2
              // fix: found on the 1.5M-point STPLS3D-shape tile, where components touch). The label array is final.
              const bool same = ((uint32_t)(k[t] >> 32) == 0xFFFFFFFFu) ? ((uint32_t)k[t] == (uint32_t)seed)
                                                                        : (ld_ca_i32(&w.label[v[t]]) == seed);
              if (same) atomicMin(&w.key[v[t]], mine);
            }
          }
        }
      }
      cluster_sync_all();
      // ---- B': members claimed in this level mark (parent row, slot) ------------------------------------
      for (int m = gtid; m < size; m += gthreads) {
        const int v = members[m];
        const unsigned long long k = __ldcg(&w.key[v]);
        const uint32_t pp = (uint32_t)(k >> 32);
        if (pp >= (uint32_t)(a + 1) && pp <= (uint32_t)b) {
          const uint32_t j = (uint32_t)k;
          atomicOr(&bm[(size_t)(pp - 1) * W + (j >> 5)], 1u << (j & 31));
        }
      }
      cluster_sync_all();
      // ---- counts per parent ------------------------------------------------------------------------------
      for (int p = a + gtid; p < b; p += gthreads) {
        int cnt = 0;
        for (int x = 0; x < W; x++) cnt += __popc(__ldcg(&bm[(size_t)p * W + x]));
        wins[p] = cnt;
      }
      cluster_sync_all();
      // ---- exclusive scan of wins[a..b) by CTA 0 ------------------------------------------------------------
      if (crank == 0) {
        if (tid == 0) s_carry = 0;
        __syncthreads();
        const int warp = tid >> 5;
        for (int p0 = a; p0 < b; p0 += kClThreads) {
          int p = p0 + tid;
          int x = (p < b) ? __ldcg(&wins[p]) : 0;
          int inc = x;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
          }
          if (lane == 31) s_warp[warp] = inc;
          __syncthreads();
          int woff = 0;
          for (int q = 0; q < warp; q++) woff += s_warp[q];
          int carry = s_carry;
          if (p < b) wins[p] = carry + woff + inc - x;
          __syncthreads();
          if (tid == kClThreads - 1) s_carry = carry + woff + inc;
          __syncthreads();
        }
        if (tid == 0) w.cursor[c] = s_carry;  // level total (cursor[] is free again after bfs_members_kernel)
      }
      cluster_sync_all();
      const int total = __ldcg(&w.cursor[c]);
      if (total == 0) break;
      // ---- C': place the claimed members --------------------------------------------------------------------
      for (int m = gtid; m < size; m += gthreads) {
        const int v = members[m];
        const unsigned long long k = __ldcg(&w.key[v]);
        const uint32_t pp = (uint32_t)(k >> 32);
        if (pp >= (uint32_t)(a + 1) && pp <= (uint32_t)b) {
          const uint32_t j = (uint32_t)k;
          const uint32_t *row = bm + (size_t)(pp - 1) * W;
          int rank = 0;
          for (uint32_t x = 0; x < (j >> 5); x++) rank += __popc(__ldcg(&row[x]));
          rank += __popc(__ldcg(&row[j >> 5]) & ((1u << (j & 31)) - 1u));
          const int pos = b + __ldcg(&wins[pp - 1]) + rank;
          order[2 * (size_t)pos] = c;
          order[2 * (size_t)pos + 1] = v;
        }
      }
      a = b;
      b += total;
    }
  }
}

// as many 8-CTA emit2 clusters as a device keeps resident at once (several CTAs per SM: the kernel is latency bound on
// its per-level cluster barriers, so components in flight -- not threads per component -- is what fills the machine)
static DeviceOnce g_emit2_once;
static int g_emit2_clusters[kMaxDevices];

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_bfs_cluster_workspace_bytes(int N) {
  if (N < 0) N = 0;
  size_t n1 = (size_t)N + 1;
  size_t b = align_up(64 * 4) + align_up(64) + 7 * align_up(n1 * 4) + 2 * align_up(n1 * 8) +
             align_up(scan_temp_elems(n1) * 8);
  return b + 1024;
}

int sgb_bfs_cluster_count(const int32_t *d_ball_query_idxs, const int32_t *d_start_len, int N, float thr,
                          const int32_t *d_node_seg, const float *d_seg_thr, const int32_t *d_upstream_err, void *d_ws,
                          size_t ws_bytes, int *h_sumNPoint, int *h_maxLen, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(N >= 0 && h_sumNPoint, SGB_ERR_ARG, "bfs_cluster arguments");
  if (h_maxLen) *h_maxLen = 0;
  if (N == 0) { *h_sumNPoint = 0; return 0; }
  SGB_REQUIRE(d_start_len && d_ws, SGB_ERR_ARG, "null pointer");
  SGB_REQUIRE((d_node_seg == nullptr) == (d_seg_thr == nullptr), SGB_ERR_ARG, "node_seg / seg_thr must come together");
  BfsWs w;
  SGB_REQUIRE(bfs_carve(d_ws, ws_bytes, N, w), SGB_ERR_WORKSPACE, "bfs_cluster workspace too small");
  SGB_CURRENT_DEVICE(d);
  int nb = div_up(N, 256);
  SGB_CUDA_CHECK(cudaMemsetAsync(w.scalars, 0, 64 * 4, st));
  bfs_init_kernel<<<nb, 256, 0, st>>>(N, w);
  SGB_LAUNCH_CHECK();
  int grid = std::min(div_up((long long)N * 32, 256), d->sms * 16);
  // passes in batches of kBatch launches, ONE host synchronisation per batch (the one that reads the cluster totals):
  // sizes / threshold / scan are enqueued optimistically behind the batch and redone in the rare case that the last
  // pass of the batch still pushed labels (flags live in scalars[8..8+kBatch)).
  constexpr int kBatch = 12;
  int32_t *flags = w.scalars + 8;
  long long tot = 0;
  int sc[8 + kBatch], up_err = 0;
  for (int batch = 0; batch < 100000; batch++) {
    if (batch > 0) {
      SGB_CUDA_CHECK(cudaMemsetAsync(flags, 0, kBatch * 4, st));
      SGB_CUDA_CHECK(cudaMemsetAsync(w.scalars + 32, 0, kBatch * 4, st));
      SGB_CUDA_CHECK(cudaMemsetAsync(w.size, 0, (size_t)N * 4, st));
    }
    for (int it = 0; it < kBatch; it++) {
      bfs_frontier_select_kernel<<<nb, 256, 0, st>>>(N, w, it, batch > 0, flags);
      SGB_LAUNCH_CHECK();
      bfs_frontier_push_kernel<<<grid, 256, 0, st>>>(d_ball_query_idxs, d_start_len, w, it, flags);
      SGB_LAUNCH_CHECK();
    }
    bfs_size_kernel<<<nb, 256, 0, st>>>(N, d_start_len, w);
    SGB_LAUNCH_CHECK();
    bfs_pack_kernel<<<nb, 256, 0, st>>>(N, thr, d_node_seg, d_seg_thr, w);
    SGB_LAUNCH_CHECK();
    int rc = exclusive_scan_i64(w.packed, w.packed, (size_t)N, w.totals, w.scan_tmp, st);
    if (rc) return rc;
    SGB_CUDA_CHECK(cudaMemcpyAsync(&tot, w.totals, 8, cudaMemcpyDeviceToHost, st));
    SGB_CUDA_CHECK(cudaMemcpyAsync(sc, w.scalars, sizeof(sc), cudaMemcpyDeviceToHost, st));
    if (d_upstream_err && batch == 0) SGB_CUDA_CHECK(cudaMemcpyAsync(&up_err, d_upstream_err, 4, cudaMemcpyDeviceToHost, st));
    SGB_CUDA_CHECK(cudaStreamSynchronize(st));
    SGB_REQUIRE((up_err & 1) == 0, SGB_ERR_RANGE, "ball query upstream of bfs_cluster: |xyz/radius| >= 131070 or segment id outside [0,1023]");
    SGB_REQUIRE(up_err == 0, SGB_ERR_RANGE, "ball query upstream of bfs_cluster: neighbour total beyond 2^31 - 1 (int32 list cursor)");
    if (sc[8 + kBatch - 1] == 0) break;  // the last pass of the batch pushed nothing: fixed point
  }
  if (h_maxLen) *h_maxLen = sc[1];
  *h_sumNPoint = (int)(tot & 0xFFFFFFFFll);
  return (int)(tot >> 32);
}

size_t sgb_bfs_cluster_scratch_bytes(int sumNPoint, int maxLen) {
  int W = (std::max(maxLen, 1) + 31) / 32;
  if (W > 64) return 0;  // long-list fallback path needs no bitmap
  return (size_t)std::max(sumNPoint, 1) * W * 4 + 256;
}

int sgb_bfs_cluster_fill(const int32_t *d_ball_query_idxs, const int32_t *d_start_len, int N, int nCluster,
                         int sumNPoint, int maxLen, int32_t *d_cluster_idxs, int32_t *d_cluster_offsets, void *d_ws,
                         size_t ws_bytes, void *d_scratch, size_t scratch_bytes, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SGB_REQUIRE(N >= 0 && nCluster >= 0 && sumNPoint >= 0 && d_cluster_offsets, SGB_ERR_ARG, "bfs_cluster_fill arguments");
  if (N == 0 || nCluster == 0) {
    SGB_CUDA_CHECK(cudaMemsetAsync(d_cluster_offsets, 0, 4, st));
    return SGB_OK;
  }
  SGB_REQUIRE(d_start_len && d_cluster_idxs && d_ws, SGB_ERR_ARG, "null pointer");
  BfsWs w;
  SGB_REQUIRE(bfs_carve(d_ws, ws_bytes, N, w), SGB_ERR_WORKSPACE, "bfs_cluster workspace too small");
  int nb = div_up(N, 256);
  bfs_roots_kernel<<<nb, 256, 0, st>>>(N, nCluster, sumNPoint, d_cluster_offsets, w);
  SGB_LAUNCH_CHECK();
  int W = (std::max(maxLen, 1) + 31) / 32;
  if (W <= 64) {
    size_t need = (size_t)sumNPoint * W * 4;
    SGB_REQUIRE(d_scratch && scratch_bytes >= need, SGB_ERR_WORKSPACE, "bfs_cluster_fill scratch too small");
    SGB_CUDA_CHECK(cudaMemsetAsync(d_scratch, 0, need, st));
    SGB_CUDA_CHECK(cudaMemsetAsync(w.cursor, 0, (size_t)nCluster * 4, st));
    bfs_members_kernel<<<nb, 256, 0, st>>>(N, d_cluster_offsets, w);
    SGB_LAUNCH_CHECK();
    SGB_CURRENT_DEVICE(d);
    once_per_device(g_emit2_once, d->ordinal, [d] {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(d->sms * 4 / kCl * kCl);
      cfg.blockDim = dim3(kClThreads);
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = kCl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr; cfg.numAttrs = 1;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, bfs_emit2_kernel, &cfg) != cudaSuccess || n < 1) { cudaGetLastError(); n = d->sms / kCl; }
      g_emit2_clusters[d->ordinal] = n;
      return SGB_OK;
    });
    int n_cl = std::min(nCluster, g_emit2_clusters[d->ordinal]);
    bfs_emit2_kernel<<<n_cl * kCl, kClThreads, 0, st>>>(d_ball_query_idxs, d_start_len, d_cluster_offsets, d_cluster_idxs,
                                                       nCluster, W, (uint32_t *)d_scratch, w);
    SGB_LAUNCH_CHECK();
  } else {
    // lists longer than 2048 entries (never produced by the ball queries): per-CTA rescan kernel
    SGB_CUDA_CHECK(cudaMemsetAsync(w.key, 0xFF, (size_t)N * 8, st));
    bfs_emit_kernel<<<nCluster, kEmitThreads, 0, st>>>(d_ball_query_idxs, d_start_len, d_cluster_offsets,
                                                       d_cluster_idxs, w);
    SGB_LAUNCH_CHECK();
  }
  return SGB_OK;
}
}
