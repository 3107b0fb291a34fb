/*
 * oracle/sg_oracle.c -- TEST INFRASTRUCTURE ONLY (never on the product path).
 *
 * Plain-C, single-threaded CPU restatement of the reference's softgroup.ops algorithms
 * (thangvubk/SoftGroup, /root/reference/softgroup/ops/src). Each function cites the
 * reference file:line it follows. Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this library.
 *
 * Pinning: voxelize_idx / bfs_cluster / octree build are checked against the compiled,
 * unmodified reference (oracle/_ref, built by oracle/build_ref.py) and against the
 * fixtures under tests/golden/ generated from it (tests/golden/make_golden.py).
 * The GPU-only reference ops (ballquery_batch_p, voxelize_fp, sec_*, global_avg_pool,
 * get_mask_*) have no CPU implementation in the reference; their restatements here are
 * pinned on the GPU box against the reference's own CUDA kernels from oracle/_ref
 * (tests/test_gpu_vs_reference.py).
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared (see oracle/Makefile). -ffp-contract=off
 * matters: every fused multiply-add below is explicit (fmaf) and mirrors the contraction
 * nvcc 12.9 -O2 applies to the reference kernels (checked in the SASS of oracle/_ref).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_MAX_NEIGH 1000 /* bfs_cluster.cu:24 `int idx_temp[1000]`, octree_ball_query.cu:11 */

/* ------------------------------------------------------------------------------------------
 * voxelize_idx  (voxelize.cpp:11-39 voxelize_idx, :68-165 voxelize_inputmap, :41-57 outputmap)
 *
 * Voxel id = first-occurrence rank in point order (nActive++ on first sight, :90/:110).
 * Keys are the int64 coords narrowed to int32 (Point<3>, datatype.h:11; voxelize.cpp:101-102),
 * one map per batch index (:104-108).  Rows of output_map: [count, p0, p1, ... , 0-pad] with
 * ascending point index (:152-162).  Mode quirks kept: mode 1 -> front(), mode 2 -> back()
 * (:139-149).  Two-phase C interface: phase 1 computes input_map, M and maxActive and keeps a
 * handle; phase 2 fills the caller-allocated output arrays (the reference resize_()s them,
 * :29-33).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int N, ncol, M, maxActive, mode;
  int32_t *first;  /* [M] first point of each voxel */
  int32_t *count;  /* [M] */
  int32_t *last;   /* [M] last point of each voxel */
  int32_t *imap;   /* [N] */
} orc_vox_t;

static inline uint64_t orc_mix(uint64_t h) {
  h ^= h >> 33; h *= 0xff51afd7ed558ccdULL; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL; h ^= h >> 33;
  return h;
}

void *orc_voxelize_idx_begin(const int64_t *coords, int N, int ncol, int mode, int32_t *input_map,
                             int *M_out, int *maxActive_out) {
  orc_vox_t *h = (orc_vox_t *)calloc(1, sizeof(orc_vox_t));
  h->N = N; h->ncol = ncol; h->mode = mode;
  size_t cap = 16; while (cap < (size_t)N * 2 + 16) cap <<= 1;
  int32_t *slot_vox = (int32_t *)malloc(cap * sizeof(int32_t));
  int32_t *slot_key = (int32_t *)malloc(cap * 4 * sizeof(int32_t));
  memset(slot_vox, 0xff, cap * sizeof(int32_t));
  h->first = (int32_t *)malloc((size_t)(N + 1) * sizeof(int32_t));
  h->count = (int32_t *)calloc((size_t)N + 1, sizeof(int32_t));
  h->last = (int32_t *)malloc((size_t)(N + 1) * sizeof(int32_t));
  h->imap = (int32_t *)malloc((size_t)(N + 1) * sizeof(int32_t));
  int M = 0;
  for (int i = 0; i < N; i++) {
    int32_t k[4];
    if (ncol == 4) { k[0] = (int32_t)coords[4 * (size_t)i]; k[1] = (int32_t)coords[4 * (size_t)i + 1];
                     k[2] = (int32_t)coords[4 * (size_t)i + 2]; k[3] = (int32_t)coords[4 * (size_t)i + 3]; }
    else { k[0] = 0; k[1] = (int32_t)coords[3 * (size_t)i]; k[2] = (int32_t)coords[3 * (size_t)i + 1];
           k[3] = (int32_t)coords[3 * (size_t)i + 2]; }
    uint64_t hv = orc_mix(((uint64_t)(uint32_t)k[0] << 32 | (uint32_t)k[1]) * 0x9E3779B97F4A7C15ULL ^
                          orc_mix((uint64_t)(uint32_t)k[2] << 32 | (uint32_t)k[3]));
    size_t s = (size_t)hv & (cap - 1);
    int v;
    for (;;) {
      v = slot_vox[s];
      if (v < 0) { slot_vox[s] = v = M; memcpy(slot_key + 4 * s, k, sizeof(k)); h->first[M] = i; M++; break; }
      if (memcmp(slot_key + 4 * s, k, sizeof(k)) == 0) break;
      s = (s + 1) & (cap - 1);
    }
    h->count[v]++; h->last[v] = i; h->imap[i] = v; input_map[i] = v;
  }
  int maxActive = 1; /* voxelize.cpp:150 */
  if (mode == 3 || mode == 4)
    for (int v = 0; v < M; v++) if (h->count[v] > maxActive) maxActive = h->count[v];
  h->M = M; h->maxActive = maxActive;
  free(slot_vox); free(slot_key);
  *M_out = M; *maxActive_out = maxActive;
  return h;
}

void orc_voxelize_idx_finish(void *handle, const int64_t *coords, int64_t *output_coords, int32_t *output_map) {
  orc_vox_t *h = (orc_vox_t *)handle;
  const int W = h->maxActive + 1;
  memset(output_map, 0, (size_t)h->M * W * sizeof(int32_t));
  if (h->mode == 3 || h->mode == 4) {
    int32_t *fill = (int32_t *)calloc((size_t)h->M + 1, sizeof(int32_t));
    for (int i = 0; i < h->N; i++) { int v = h->imap[i]; output_map[(size_t)v * W + 1 + fill[v]++] = i; }
    for (int v = 0; v < h->M; v++) output_map[(size_t)v * W] = h->count[v];
    free(fill);
  } else {
    for (int v = 0; v < h->M; v++) {
      output_map[(size_t)v * W] = 1;
      /* mode 0: unique; mode 1: front(); mode 2: back()  (voxelize.cpp:131-149) */
      output_map[(size_t)v * W + 1] = (h->mode == 2) ? h->last[v] : h->first[v];
    }
  }
  /* voxelize_outputmap (:41-57): coords of rule[1] (the first listed point) */
  for (int v = 0; v < h->M; v++) {
    int p = output_map[(size_t)v * W + 1];
    for (int j = 0; j < h->ncol; j++) output_coords[(size_t)v * h->ncol + j] = coords[(size_t)p * h->ncol + j];
  }
  free(h->first); free(h->count); free(h->last); free(h->imap); free(h);
}

/* ------------------------------------------------------------------------------------------
 * voxelize_fp / voxelize_bp  (voxelize.cu:9-36, :38-62)
 * out[row][c] = ((0 + m*x0) + m*x1) + ...  with m = 1/n (mode 4) or 1; product and sum are
 * separate roundings in the reference because the sum is an atomicAdd.
 * ------------------------------------------------------------------------------------------ */
void orc_voxelize_fp(const float *feats, float *out, const int32_t *rules, int M, int maxActive, int C, int average) {
  for (int row = 0; row < M; row++) {
    const int32_t *r = rules + (size_t)row * (maxActive + 1);
    int n = r[0];
    float m = (average && n > 0) ? 1.0f / (float)n : 1.0f;
    for (int c = 0; c < C; c++) {
      float acc = 0.0f;
      for (int i = 1; i <= n; i++) { float t = m * feats[(size_t)r[i] * C + c]; acc = acc + t; }
      out[(size_t)row * C + c] = acc;
    }
  }
}

void orc_voxelize_bp(const float *d_out, float *d_feats, const int32_t *rules, int M, int maxActive, int C, int average) {
  for (int row = 0; row < M; row++) {
    const int32_t *r = rules + (size_t)row * (maxActive + 1);
    int n = r[0];
    float m = (average && n > 0) ? 1.0f / (float)n : 1.0f;
    for (int i = 1; i <= n; i++)
      for (int c = 0; c < C; c++) { float t = m * d_out[(size_t)row * C + c]; d_feats[(size_t)r[i] * C + c] += t; }
  }
}

/* ------------------------------------------------------------------------------------------
 * ballquery_batch_p  (bfs_cluster.cu:15-66)
 * Per query: scan k = start..end-1 of the query's batch segment in ascending index, strict
 * d2 < r*r, keep the first 1000 hits (:36-50).  d2 in the compiled contraction order
 * fmaf(dz,dz, fmaf(dx,dx, dy*dy)) (SASS of oracle/_ref: FMUL dy*dy; FFMA dx; FFMA dz).
 * Layout here: list start = exclusive prefix of counts in point order (the reference's
 * atomicAdd layout is nondeterministic, :52; compare per point).  Returns sum of counts.
 * If idx == NULL only start_len is produced.  Entries past `idx_capacity` are dropped (:55-61).
 * ------------------------------------------------------------------------------------------ */
static inline int orc_is_nb(const float *o, const float *p, float r2) {
  float dx = o[0] - p[0], dy = o[1] - p[1], dz = o[2] - p[2];
  float d2 = fmaf(dz, dz, fmaf(dx, dx, dy * dy));
  return d2 < r2;
}

long long orc_ballquery_batch_p(const float *xyz, const int32_t *batch_idxs, const int32_t *batch_offsets, int n,
                                float radius, int32_t *idx, long long idx_capacity, int32_t *start_len) {
  float r2 = radius * radius;
  long long cum = 0;
  for (int i = 0; i < n; i++) {
    int b = batch_idxs[i];
    int s = batch_offsets[b], e = batch_offsets[b + 1];
    int cnt = 0;
    for (int k = s; k < e; k++) {
      if (orc_is_nb(xyz + 3 * (size_t)i, xyz + 3 * (size_t)k, r2)) {
        if (cnt < ORC_MAX_NEIGH) { if (idx && cum + cnt < idx_capacity) idx[cum + cnt] = k; }
        else break;
        ++cnt;
      }
    }
    start_len[2 * (size_t)i] = (int32_t)cum; start_len[2 * (size_t)i + 1] = cnt;
    cum += cnt;
  }
  return cum;
}

/* ------------------------------------------------------------------------------------------
 * ballquery_batch_p on a uniform grid: the lists of orc_ballquery_batch_p (same test, same
 * ascending candidate order, same first 1000) without its O(n^2) scan.
 *
 * Why the 27 cells hold every neighbour: all three terms of d2 are >= 0, so d2 >= fl(dx*dx)
 * and d2 < r2 = fl(r*r) needs |fl(dx)| < |r|; rounding is monotone, so the exact |x_i - x_k|
 * < |r| as well (likewise y, z).  The cell edge c is |r| (1 + 2^-20), or extent / 2^20 when
 * that is larger (cell ids then fit 21 bits whatever the coordinates); the double-precision
 * cell coordinates (x - min) / c are <= 2^20 with an error below 2^-30, so two neighbours'
 * cells differ by at most one per axis.  A point with a NaN or Inf coordinate fails every
 * test (d2 is NaN or Inf): it is in no cell and has no neighbour, as in the scan.
 * Per segment b (batch_offsets[b] .. [b+1]) its finite points are sorted by (cell, index);
 * a query merges the index-sorted runs of its 27 cells and tests candidates in ascending
 * index until the 1000th hit.
 * ------------------------------------------------------------------------------------------ */
typedef struct { int64_t key; int32_t idx; } orc_cellpt_t;

static int orc_cellpt_cmp(const void *a, const void *b) {
  const orc_cellpt_t *p = (const orc_cellpt_t *)a, *q = (const orc_cellpt_t *)b;
  if (p->key != q->key) return p->key < q->key ? -1 : 1;
  return (p->idx > q->idx) - (p->idx < q->idx);
}

typedef struct { orc_cellpt_t *pts; int n; double mn[3], c; } orc_grid_t;

#define ORC_GRID_BITS 21
static inline int64_t orc_cell_key(const int64_t cc[3]) {
  return (cc[0] << (2 * ORC_GRID_BITS)) | (cc[1] << ORC_GRID_BITS) | cc[2];
}

static void orc_grid_build(orc_grid_t *g, const float *xyz, int s, int e, float radius) {
  double mx[3] = {0, 0, 0};
  int first = 1;
  g->pts = (orc_cellpt_t *)malloc(sizeof(orc_cellpt_t) * (size_t)(e > s ? e - s : 1));
  g->n = 0;
  g->mn[0] = g->mn[1] = g->mn[2] = 0;
  for (int k = s; k < e; k++) {
    const float *p = xyz + 3 * (size_t)k;
    if (!isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2])) continue;
    for (int a = 0; a < 3; a++) {
      if (first || p[a] < g->mn[a]) g->mn[a] = p[a];
      if (first || p[a] > mx[a]) mx[a] = p[a];
    }
    first = 0;
  }
  double ext = 0;
  for (int a = 0; a < 3; a++) ext = fmax(ext, mx[a] - g->mn[a]);
  g->c = fmax(fabs((double)radius) * (1.0 + ldexp(1.0, -20)), ext * ldexp(1.0, -20));
  for (int k = s; k < e; k++) {
    const float *p = xyz + 3 * (size_t)k;
    if (!isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2])) continue;
    int64_t cc[3];
    for (int a = 0; a < 3; a++) cc[a] = (int64_t)floor((p[a] - g->mn[a]) / g->c);
    g->pts[g->n].key = orc_cell_key(cc);
    g->pts[g->n].idx = k;
    g->n++;
  }
  qsort(g->pts, (size_t)g->n, sizeof(orc_cellpt_t), orc_cellpt_cmp);
}

static int orc_grid_lower(const orc_grid_t *g, int64_t key) {
  int lo = 0, hi = g->n;
  while (lo < hi) {
    int mid = lo + (hi - lo) / 2;
    if (g->pts[mid].key < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

/* neighbours of xyz[i] in grid g, ascending index, first 1000; written to out (if non-NULL) */
static int orc_grid_query(const orc_grid_t *g, const float *xyz, int i, float r2, int32_t *out) {
  const float *o = xyz + 3 * (size_t)i;
  if (!isfinite(o[0]) || !isfinite(o[1]) || !isfinite(o[2]) || g->n == 0) return 0;
  const int64_t lim = (int64_t)1 << ORC_GRID_BITS;
  double qc[3];
  for (int a = 0; a < 3; a++) {
    qc[a] = floor((o[a] - g->mn[a]) / g->c);
    if (qc[a] < -1 || qc[a] > (double)lim) return 0; /* no cell of the segment within one step */
  }
  int lo[27], hi[27], nr = 0;
  for (int d0 = -1; d0 <= 1; d0++)
    for (int d1 = -1; d1 <= 1; d1++)
      for (int d2 = -1; d2 <= 1; d2++) {
        int64_t cc[3] = {(int64_t)qc[0] + d0, (int64_t)qc[1] + d1, (int64_t)qc[2] + d2};
        if (cc[0] < 0 || cc[1] < 0 || cc[2] < 0 || cc[0] >= lim || cc[1] >= lim || cc[2] >= lim) continue;
        int64_t key = orc_cell_key(cc);
        int a = orc_grid_lower(g, key), b = orc_grid_lower(g, key + 1);
        if (a < b) { lo[nr] = a; hi[nr] = b; nr++; }
      }
  /* k-way merge of the runs: a binary min-heap of runs keyed by their next index */
  int heap[27], nh = 0;
#define ORC_HEAD(j) (g->pts[lo[j]].idx)
  for (int j = 0; j < nr; j++) {
    int c = nh++;
    while (c > 0 && ORC_HEAD(heap[(c - 1) / 2]) > ORC_HEAD(j)) { heap[c] = heap[(c - 1) / 2]; c = (c - 1) / 2; }
    heap[c] = j;
  }
  int cnt = 0;
  while (cnt < ORC_MAX_NEIGH && nh > 0) {
    int j = heap[0];
    int k = g->pts[lo[j]++].idx;
    if (lo[j] == hi[j]) j = heap[--nh]; /* run exhausted: sift the last run down from the root */
    if (nh > 0) {
      int c = 0, v = ORC_HEAD(j);
      for (;;) {
        int l = 2 * c + 1, m = c, vm = v;
        if (l < nh && ORC_HEAD(heap[l]) < vm) { m = l; vm = ORC_HEAD(heap[l]); }
        if (l + 1 < nh && ORC_HEAD(heap[l + 1]) < vm) m = l + 1;
        if (m == c) break;
        heap[c] = heap[m];
        c = m;
      }
      heap[c] = j;
    }
    if (orc_is_nb(o, xyz + 3 * (size_t)k, r2)) {
      if (out) out[cnt] = k;
      ++cnt;
    }
  }
#undef ORC_HEAD
  return cnt;
}

long long orc_ballquery_batch_p_grid(const float *xyz, const int32_t *batch_idxs, const int32_t *batch_offsets,
                                     int nbatch, int n, float radius, int32_t *idx, long long idx_capacity,
                                     int32_t *start_len) {
  float r2 = radius * radius;
  orc_grid_t *grids = (orc_grid_t *)calloc((size_t)(nbatch > 0 ? nbatch : 1), sizeof(orc_grid_t));
  for (int b = 0; b < nbatch; b++) orc_grid_build(&grids[b], xyz, batch_offsets[b], batch_offsets[b + 1], radius);
  int32_t tmp[ORC_MAX_NEIGH];
  long long cum = 0;
  for (int i = 0; i < n; i++) {
    int cnt = (r2 > 0) ? orc_grid_query(&grids[batch_idxs[i]], xyz, i, r2, idx ? tmp : NULL) : 0;
    if (idx)
      for (int j = 0; j < cnt && cum + j < idx_capacity; j++) idx[cum + j] = tmp[j];
    start_len[2 * (size_t)i] = (int32_t)cum; start_len[2 * (size_t)i + 1] = cnt;
    cum += cnt;
  }
  for (int b = 0; b < nbatch; b++) free(grids[b].pts);
  free(grids);
  return cum;
}

/* ------------------------------------------------------------------------------------------
 * bfs_cluster  (bfs_cluster.cpp:33-126): find_cc :33-58, get_clusters :60-86,
 * fill_cluster_idxs_ :89-99.  Two-phase: begin() returns sumNPoint / nCluster, finish() fills.
 * ------------------------------------------------------------------------------------------ */
typedef struct { int nCluster, sumNPoint; int32_t *pts; int32_t *sizes; } orc_bfs_t;

void *orc_bfs_cluster_begin(const float *class_numpoint_mean, const int32_t *ball_query_idxs, const int32_t *start_len,
                            int N, float threshold, int class_id, int *sumNPoint_out, int *nCluster_out) {
  orc_bfs_t *h = (orc_bfs_t *)calloc(1, sizeof(orc_bfs_t));
  uint8_t *visited = (uint8_t *)calloc((size_t)N + 1, 1);
  int32_t *queue = (int32_t *)malloc(((size_t)N + 1) * sizeof(int32_t));
  h->pts = (int32_t *)malloc(((size_t)N + 1) * sizeof(int32_t));
  h->sizes = (int32_t *)malloc(((size_t)N + 1) * sizeof(int32_t));
  float mean = class_numpoint_mean[class_id];
  float thr = (mean == -1.0f) ? threshold : threshold * mean; /* :70-77 */
  int sum = 0, nc = 0;
  for (int i = 0; i < N; i++) {
    if (visited[i]) continue;
    int head = 0, tail = 0;
    queue[tail++] = i; visited[i] = 1;
    while (head < tail) {
      int cur = queue[head++];
      int s = start_len[2 * (size_t)cur], l = start_len[2 * (size_t)cur + 1];
      for (int k = s; k < s + l; k++) {
        int v = ball_query_idxs[k];
        if (visited[v]) continue;
        visited[v] = 1; queue[tail++] = v;
      }
    }
    if ((float)(int)tail >= thr) { /* `(int)size >= thr`, int promoted to float (:78) */
      memcpy(h->pts + sum, queue, (size_t)tail * sizeof(int32_t));
      h->sizes[nc++] = tail; sum += tail;
    }
  }
  free(visited); free(queue);
  h->nCluster = nc; h->sumNPoint = sum;
  *sumNPoint_out = sum; *nCluster_out = nc;
  return h;
}

void orc_bfs_cluster_finish(void *handle, int32_t *cluster_idxs, int32_t *cluster_offsets) {
  orc_bfs_t *h = (orc_bfs_t *)handle;
  int pos = 0;
  cluster_offsets[0] = 0;
  for (int c = 0; c < h->nCluster; c++) {
    for (int j = 0; j < h->sizes[c]; j++, pos++) { cluster_idxs[2 * (size_t)pos] = c; cluster_idxs[2 * (size_t)pos + 1] = h->pts[pos]; }
    cluster_offsets[c + 1] = pos;
  }
  free(h->pts); free(h->sizes); free(h);
}

/* ------------------------------------------------------------------------------------------
 * sec_mean / sec_min / sec_max  (sec_mean.cu:13-37, :41-65, :69-93)
 * ------------------------------------------------------------------------------------------ */
void orc_sec_mean(const float *inp, const int32_t *offsets, float *out, int nProposal, int C) {
  for (int p = 0; p < nProposal; p++) {
    int s = offsets[p], e = offsets[p + 1];
    float count = (float)(e - s);
    for (int c = 0; c < C; c++) {
      float mean = 0;
      for (int i = s; i < e; i++) { float q = inp[(size_t)i * C + c] / count; mean = mean + q; }
      out[(size_t)p * C + c] = mean;
    }
  }
}
void orc_sec_min(const float *inp, const int32_t *offsets, float *out, int nProposal, int C) {
  for (int p = 0; p < nProposal; p++)
    for (int c = 0; c < C; c++) {
      float v = (float)1e50; /* +inf after narrowing (:48) */
      for (int i = offsets[p]; i < offsets[p + 1]; i++) if (inp[(size_t)i * C + c] < v) v = inp[(size_t)i * C + c];
      out[(size_t)p * C + c] = v;
    }
}
void orc_sec_max(const float *inp, const int32_t *offsets, float *out, int nProposal, int C) {
  for (int p = 0; p < nProposal; p++)
    for (int c = 0; c < C; c++) {
      float v = (float)-1e50;
      for (int i = offsets[p]; i < offsets[p + 1]; i++) if (inp[(size_t)i * C + c] > v) v = inp[(size_t)i * C + c];
      out[(size_t)p * C + c] = v;
    }
}

/* ------------------------------------------------------------------------------------------
 * global_avg_pool fp / bp  (roipool.cu:12-31, :47-60): (sum x) / n, divide after the sum.
 * ------------------------------------------------------------------------------------------ */
void orc_global_avg_pool_fp(const float *feats, const int32_t *offsets, float *out, int nProposal, int C) {
  for (int p = 0; p < nProposal; p++) {
    int s = offsets[p], e = offsets[p + 1];
    for (int c = 0; c < C; c++) {
      float v = 0;
      for (int i = s; i < e; i++) v = v + feats[(size_t)i * C + c];
      out[(size_t)p * C + c] = v / (float)(e - s);
    }
  }
}
void orc_global_avg_pool_bp(float *d_feats, const int32_t *offsets, const float *d_out, int nProposal, int C) {
  for (int p = 0; p < nProposal; p++) {
    int s = offsets[p], e = offsets[p + 1];
    for (int c = 0; c < C; c++)
      for (int i = s; i < e; i++) d_feats[(size_t)i * C + c] += d_out[(size_t)p * C + c] / (float)(e - s);
  }
}

/* ------------------------------------------------------------------------------------------
 * get_mask_iou_on_cluster / on_pred / get_mask_label  (cal_iou_and_masklabel.cu:9-33, :35-66,
 * :68-102).  The `+ 1e-5` literal is a double, so the division happens in fp64 (:29-31).
 * ------------------------------------------------------------------------------------------ */
void orc_get_mask_iou_on_cluster(const int32_t *proposals_idx, const int32_t *proposals_offset,
                                 const int64_t *instance_labels, const int32_t *instance_pointnum,
                                 float *proposals_iou, int nInstance, int nProposal) {
  for (int p = 0; p < nProposal; p++) {
    int s = proposals_offset[p], e = proposals_offset[p + 1];
    int total = e - s;
    for (int q = 0; q < nInstance; q++) {
      int inter = 0;
      for (int i = s; i < e; i++) if ((int)instance_labels[proposals_idx[i]] == q) inter++;
      proposals_iou[(size_t)p * nInstance + q] =
          (float)((double)(float)inter / ((double)(float)(total + instance_pointnum[q] - inter) + 1e-5));
    }
  }
}
void orc_get_mask_iou_on_pred(const int32_t *proposals_idx, const int32_t *proposals_offset,
                              const int64_t *instance_labels, const int32_t *instance_pointnum,
                              float *proposals_iou, int nInstance, int nProposal, const float *mask_scores_sigmoid) {
  for (int p = 0; p < nProposal; p++) {
    int s = proposals_offset[p], e = proposals_offset[p + 1];
    int total = 0;
    for (int i = s; i < e; i++) if (mask_scores_sigmoid[i] > 0.5) total++;
    for (int q = 0; q < nInstance; q++) {
      int inter = 0;
      for (int i = s; i < e; i++)
        if (mask_scores_sigmoid[i] > 0.5 && (int)instance_labels[proposals_idx[i]] == q) inter++;
      proposals_iou[(size_t)p * nInstance + q] =
          (float)((double)(float)inter / ((double)(float)(total + instance_pointnum[q] - inter) + 1e-5));
    }
  }
}
void orc_get_mask_label(const int32_t *proposals_idx, const int32_t *proposals_offset, const int64_t *instance_labels,
                        const int64_t *instance_cls, const float *proposals_iou, int nInstance, int nProposal,
                        float iou_thr, float *mask_label) {
  for (int p = 0; p < nProposal; p++) {
    int s = proposals_offset[p], e = proposals_offset[p + 1];
    float max_iou = 0.f; int max_ind = 0;
    for (int q = 0; q < nInstance; q++)
      if (proposals_iou[(size_t)p * nInstance + q] > max_iou && instance_cls[q] != -100) {
        max_iou = proposals_iou[(size_t)p * nInstance + q]; max_ind = q;
      }
    if (max_iou >= iou_thr)
      for (int i = s; i < e; i++) mask_label[i] = ((int)instance_labels[proposals_idx[i]] == max_ind) ? 1.f : 0.f;
  }
}

/* ------------------------------------------------------------------------------------------
 * Octree (SoftGroup++):  build_and_export_octree (octree_ball_query.cpp:19-165) and
 * octree_ball_query (octree_ball_query.cu:14-126).
 * Fixed 3 levels, 585 nodes in BFS order, 512 leaves; `<` goes low (:52-57); octant boxes by
 * halving (:60-84); leaf point lists keep ascending point index (stable split, :101-108).
 * ------------------------------------------------------------------------------------------ */
#define ORC_NODES 585
#define ORC_LEAVES 512
#define ORC_MIDS 73

void orc_build_octree(const float *points, const float *xyzwhl, int n, float *boxes /*[585,6]*/,
                      int32_t *pt_inds /*[n]*/, int32_t *pt_start_len /*[512,2]*/) {
  /* BFS numbering: node k's children are 8k+1 .. 8k+8 (export order, :115-148) */
  for (int j = 0; j < 6; j++) boxes[j] = xyzwhl[j];
  for (int k = 0; k < ORC_MIDS; k++) {
    const float *pb = boxes + 6 * k;
    for (int o = 0; o < 8; o++) {
      float *b = boxes + 6 * (8 * k + o + 1);
      float w = pb[3] / 2, h = pb[4] / 2, l = pb[5] / 2;
      b[0] = (o & 1) ? pb[0] + w / 2 : pb[0] - w / 2;
      b[1] = (o & 2) ? pb[1] + h / 2 : pb[1] - h / 2;
      b[2] = (o & 4) ? pb[2] + l / 2 : pb[2] - l / 2;
      b[3] = w; b[4] = h; b[5] = l;
    }
  }
  int32_t *leaf_of = (int32_t *)malloc(((size_t)n + 1) * sizeof(int32_t));
  int32_t cnt[ORC_LEAVES]; memset(cnt, 0, sizeof(cnt));
  for (int i = 0; i < n; i++) {
    int node = 0;
    for (int lvl = 0; lvl < 3; lvl++) {
      const float *b = boxes + 6 * node;
      int ox = points[3 * (size_t)i] < b[0] ? 0 : 1;
      int oy = points[3 * (size_t)i + 1] < b[1] ? 0 : 1;
      int oz = points[3 * (size_t)i + 2] < b[2] ? 0 : 1;
      node = 8 * node + ((oz << 2) + (oy << 1) + ox) + 1;
    }
    leaf_of[i] = node - ORC_MIDS; cnt[leaf_of[i]]++;
  }
  int32_t start[ORC_LEAVES]; int acc = 0;
  for (int l = 0; l < ORC_LEAVES; l++) { start[l] = acc; pt_start_len[2 * l] = acc; pt_start_len[2 * l + 1] = cnt[l]; acc += cnt[l]; }
  for (int i = 0; i < n; i++) pt_inds[start[leaf_of[i]]++] = i;
  free(leaf_of);
}

static inline int orc_box_hit(const float *box, const float *p, float r) { /* is_interection, .cu:14-44 */
  float dx = fabsf(box[0] - p[0]), dy = fabsf(box[1] - p[1]), dz = fabsf(box[2] - p[2]);
  float hw = box[3] / 2, hh = box[4] / 2, hl = box[5] / 2;
  if (dx > hw + r) return 0;
  if (dy > hh + r) return 0;
  if (dz > hl + r) return 0;
  if (dx <= hw) return 1;
  if (dy <= hh) return 1;
  if (dz <= hl) return 1;
  float ex = dx - hw, ey = dy - hh, ez = dz - hl;
  /* compiled contraction order of ex*ex + ey*ey + ez*ez (see tests: pinned on the GPU box) */
  float d = fmaf(ez, ez, fmaf(ex, ex, ey * ey));
  return d <= r * r;
}

long long orc_octree_ball_query(const float *points, const float *boxes, const int32_t *pt_inds,
                                const int32_t *pt_start_len, int n, float radius, int32_t *out_inds,
                                long long capacity, int32_t *out_start_len) {
  float r2 = radius * radius;
  long long cum = 0;
  uint8_t *act = (uint8_t *)malloc(ORC_NODES);
  int32_t *tmp = (int32_t *)malloc(ORC_MAX_NEIGH * sizeof(int32_t));
  for (int q = 0; q < n; q++) {
    const float *cp = points + 3 * (size_t)q;
    memset(act, 1, ORC_NODES);
    int count = 0;
    for (int node = 0; node < ORC_MIDS; node++) {
      int a = act[node];
      for (int o = 0; o < 8; o++) {
        int oc = node * 8 + o + 1;
        if (!a) { act[oc] = 0; continue; }
        int hit = orc_box_hit(boxes + 6 * oc, cp, radius);
        act[oc] = (uint8_t)hit;
        if (hit && oc >= ORC_MIDS) {
          int leaf = oc - ORC_MIDS;
          int s = pt_start_len[2 * leaf], e = s + pt_start_len[2 * leaf + 1];
          for (int i = s; i < e; i++) {
            int pi = pt_inds[i];
            if (orc_is_nb(cp, points + 3 * (size_t)pi, r2)) {
              if (count < ORC_MAX_NEIGH) tmp[count++] = pi;
              else break; /* leaves only the leaf loop (.cu:95-106) */
            }
          }
        }
      }
    }
    out_start_len[2 * (size_t)q] = (int32_t)cum; out_start_len[2 * (size_t)q + 1] = count;
    if (out_inds) for (int i = 0; i < count && cum + i < capacity; i++) out_inds[cum + i] = tmp[i];
    cum += count;
  }
  free(act); free(tmp);
  return cum;
}
