/*
 * sgb200.h -- C ABI of libsgb200.so, the H100 (sm_90a) implementation of SoftGroup's per-scan
 * inference hot path (reference: thangvubk/SoftGroup, paths below are relative to its root).
 *
 * Boundary rules
 *   - extern "C", plain pointers and sizes, no torch / ATen types.
 *   - Every pointer named d_* is DEVICE memory; h_* is HOST memory. `stream` is a cudaStream_t
 *     passed as void*. All work is enqueued on `stream`; functions documented as "blocking"
 *     synchronise that stream before returning (they return a count the caller needs to size
 *     the next allocation, exactly where the reference blocks on cudaMemcpy D2H).
 *   - The library owns no memory between calls. Scratch is caller-provided: ask
 *     sgb_*_workspace_bytes() and pass a device buffer of at least that size.
 *   - Return value: >= 0 on success (a count where documented), < 0 = SGB_ERR_*; the message is
 *     available from sgb_last_error(). Nothing falls back to the CPU.
 *   - Out-parameter convention follows the reference extension (softgroup/ops/src/softgroup_api.cpp:6-29):
 *     the caller pre-allocates outputs. Where the reference resize_()s an empty tensor inside the
 *     callee (voxelize.cpp:29-33, bfs_cluster.cpp:119-122) the C ABI is two-phase:
 *     *_count (returns sizes) then *_fill.
 */
#ifndef SGB200_H
#define SGB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGB_OK 0
#define SGB_ERR_CUDA (-1)      /* a CUDA call failed; see sgb_last_error() */
#define SGB_ERR_ARG (-2)       /* bad argument (null pointer, negative size, unsupported mode) */
#define SGB_ERR_WORKSPACE (-3) /* workspace too small */
#define SGB_ERR_RANGE (-4)     /* input outside the packed-key range (see each function) */
#define SGB_ERR_OVERFLOW (-5)  /* fixed-capacity structure overflowed */

#define SGB_MAX_NEIGHBORS 1000 /* softgroup/ops/src/bfs_cluster/bfs_cluster.cu:24, octree_ball_query.cu:11 */

const char *sgb_last_error(void);
/* ABI version of this header (bumped on any signature change). */
int sgb_abi_version(void);
/* Number of CUDA kernels this library has launched in this process (bench.py's gpu_launches evidence). */
long long sgb_launch_count(void);
/* 1 if a CUDA device is usable, 0 otherwise (never initialises a context when none exists). */
int sgb_device_available(void);

/* ---------------------------------------------------------------------------------------------
 * voxelize_idx -- replaces voxelize_idx_3d (softgroup/ops/src/softgroup_ops.cpp:13-19) =
 * voxelize_idx<3> / voxelize_inputmap / voxelize_outputmap (voxelize/voxelize.cpp:11-165).
 * coords: int64 [N, ncol], ncol = 4 (batch,x,y,z) or 3 (x,y,z). Voxel id = first-occurrence rank
 * in point order; output_map rows are [count, p0, p1, ..., 0-pad] with ascending point index.
 * mode: 0 unique, 1 first, 2 last, 3 sum, 4 mean (only the map differs; 4 is what the model uses).
 *
 * GPU path: keys are packed into 64 bits: batch in [0, 65535], x,y,z in [-32768, 32767]
 * (all reference configs fit, the corners included); anything outside returns SGB_ERR_RANGE.
 *   count (blocking): fills d_input_map [N]; returns M and maxActive through h_M / h_maxActive.
 *   fill: d_output_coords int64 [M, ncol], d_output_map int32 [M, maxActive+1]. Must be called with
 *         the SAME workspace contents left by count.
 * CPU path (host pointers, for DataLoader workers -- softgroup/data/custom.py:239; never touches
 * CUDA): sgb_voxelize_idx_cpu_begin / _finish with the same semantics and no key-range limit.
 * ------------------------------------------------------------------------------------------- */
size_t sgb_voxelize_idx_workspace_bytes(int N);
int sgb_voxelize_idx_count(const int64_t *d_coords, int N, int ncol, int mode, int32_t *d_input_map, void *d_ws,
                           size_t ws_bytes, int *h_M, int *h_maxActive, void *stream);
int sgb_voxelize_idx_fill(const int64_t *d_coords, int N, int ncol, int mode, int M, int maxActive,
                          int64_t *d_output_coords, int32_t *d_output_map, void *d_ws, size_t ws_bytes, void *stream);
void *sgb_voxelize_idx_cpu_begin(const int64_t *h_coords, int N, int ncol, int mode, int32_t *h_input_map, int *h_M,
                                 int *h_maxActive);
int sgb_voxelize_idx_cpu_finish(void *handle, const int64_t *h_coords, int64_t *h_output_coords,
                                int32_t *h_output_map);

/* voxelize_fp / voxelize_bp -- replace voxelize_fp_feat / voxelize_bp_feat (softgroup_ops.cpp:21-38,
 * voxelize/voxelize.cu:9-62). feats f32 [N,C], rules int32 [M, maxActive+1], out f32 [M,C].
 * fp overwrites d_out (no pre-zeroing needed); bp ACCUMULATES into d_d_feats like the reference. */
int sgb_voxelize_fp(const float *d_feats, float *d_out, const int32_t *d_rules, int mode, int M, int maxActive, int C,
                    void *stream);
int sgb_voxelize_bp(const float *d_d_out, float *d_d_feats, const int32_t *d_rules, int mode, int M, int maxActive,
                    int C, void *stream);

/* ---------------------------------------------------------------------------------------------
 * ballquery_batch_p -- replaces ballquery_batch_p_cuda (bfs_cluster/bfs_cluster.cu:68-101, kernel :15-66).
 * xyz f32 [n,3]; batch_idxs int32 [n]; batch_offsets int32 [B+1] (non-decreasing; query i scans the index
 * range of its batch). Per point: neighbours with d2 < radius^2 (strict, fp32, d2 evaluated as
 * fma(dz,dz,fma(dx,dx,dy*dy)) like the compiled reference), ascending point index, self included, first
 * 1000 kept. d_idx has capacity n*meanActive entries; lists that would cross the capacity are truncated
 * exactly like the reference (:55-61) and the caller relaunches with a larger meanActive
 * (softgroup/ops/functions.py:258-266). d_start_len int32 [n,2] = (start, count).
 * Returns (blocking) the total neighbour count, like the reference's `return cumsum`.
 * The *_async form never synchronises: it leaves d_total[0] = total, d_total[1] = error flags (int32 [2], device).
 * Points with a NaN / Inf coordinate get the empty list and are nobody's neighbour -- the reference's result, every
 * comparison with them being false (:38-44). B must be <= 1023 and finite |xyz/radius| < 131070: SGB_ERR_RANGE
 * otherwise (blocking form), or bit 1 of d_total[1] (async form; sgb_bfs_cluster_count reports it).
 * capacity must stay below 2^31 entries (int32 cursor). A neighbour total beyond 2^31 - 1 does not fit the int32 cursor
 * either: nothing is written past the wrap, and it is SGB_ERR_RANGE (blocking form) or bit 2 of d_total[1].
 * ------------------------------------------------------------------------------------------- */
size_t sgb_ballquery_workspace_bytes(int n);
long long sgb_ballquery_batch_p(int n, int meanActive, float radius, const float *d_xyz, const int32_t *d_batch_idxs,
                                const int32_t *d_batch_offsets, int B, int32_t *d_idx, int32_t *d_start_len,
                                void *d_ws, size_t ws_bytes, void *stream);
int sgb_ballquery_batch_p_async(int n, long long capacity, float radius, const float *d_xyz,
                                const int32_t *d_batch_idxs, const int32_t *d_batch_offsets, int B, int32_t *d_idx,
                                int32_t *d_start_len, int32_t *d_total, void *d_ws, size_t ws_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Octree ball query (SoftGroup++) -- replaces build_and_export_octree (octree_ball_query/octree_ball_query.cpp:150-165,
 * CPU pointer tree) and octree_ball_query (octree_ball_query.cu:128-147). Fixed 3 levels: boxes f32 [585,6] in BFS
 * order from xyzwhl = (centre, extent) f32 [6]; pt_inds int32 [n] (leaf-major, ascending inside a leaf);
 * pt_start_len int32 [512,2]. Query: neighbours in LEAF-MAJOR order, first 1000 kept; d_out_inds has capacity
 * n*mean_active with the reference's truncation; returns (blocking) the total count, like the reference.
 * The tree ignores batch indices (batch size 1 only), like the reference.
 * ------------------------------------------------------------------------------------------- */
size_t sgb_octree_workspace_bytes(int n);
int sgb_octree_build(const float *d_points, int n, const float *d_xyzwhl, float *d_boxes, int32_t *d_pt_inds,
                     int32_t *d_pt_start_len, void *d_ws, size_t ws_bytes, void *stream);
long long sgb_octree_ball_query(const float *d_points, const float *d_boxes, const int32_t *d_pt_inds,
                                const int32_t *d_pt_start_len, int n, int mean_active, float radius, int32_t *d_out_inds,
                                int32_t *d_out_start_len, int32_t *d_total, void *stream);

/* ---------------------------------------------------------------------------------------------
 * bfs_cluster -- replaces bfs_cluster / get_clusters / find_cc / fill_cluster_idxs_
 * (bfs_cluster/bfs_cluster.cpp:33-126), on the GPU, bit-exact including BFS visitation order.
 * d_ball_query_idxs int32 [nActive], d_start_len int32 [N,2] (DEVICE memory; the reference takes CPU
 * tensors). threshold semantics (:70-82): a component is kept when (float)size >= thr, where the caller
 * passes thr = threshold if class_numpoint_mean[class_id] == -1 else threshold * mean.
 *   count (blocking): returns nCluster, writes sumNPoint to *h_sumNPoint and the longest list length to *h_maxLen.
 *   fill: d_cluster_idxs int32 [sumNPoint,2] (cluster id, point idx), d_cluster_offsets int32 [nCluster+1].
 * Optional per-node segments (d_node_seg int32 [N], d_seg_thr f32 [nSeg]) give every node the threshold of
 * its segment (used to cluster all classes of a scan in one call); pass NULL for a single threshold.
 * The labelling is the exact directed one (lists cut by the 1000 cap make the graph asymmetric); label passes are
 * enqueued in batches and the host waits ONCE, for the totals. d_upstream_err (nullable): device int32 error flag of
 * the asynchronous ball query that produced the lists (d_total + 1 of sgb_ballquery_batch_p_async); it is read at that
 * same wait and reported as SGB_ERR_RANGE when non-zero.
 * ------------------------------------------------------------------------------------------- */
size_t sgb_bfs_cluster_workspace_bytes(int N);
int sgb_bfs_cluster_count(const int32_t *d_ball_query_idxs, const int32_t *d_start_len, int N, float thr,
                          const int32_t *d_node_seg, const float *d_seg_thr, const int32_t *d_upstream_err, void *d_ws,
                          size_t ws_bytes, int *h_sumNPoint, int *h_maxLen, void *stream);
/* scratch for fill: one bitmap row of ceil(maxLen/32) words per emitted point (0 when maxLen > 2048: fallback path) */
size_t sgb_bfs_cluster_scratch_bytes(int sumNPoint, int maxLen);
int sgb_bfs_cluster_fill(const int32_t *d_ball_query_idxs, const int32_t *d_start_len, int N, int nCluster,
                         int sumNPoint, int maxLen, int32_t *d_cluster_idxs, int32_t *d_cluster_offsets, void *d_ws,
                         size_t ws_bytes, void *d_scratch, size_t scratch_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Segment reductions -- replace sec_mean / sec_min / sec_max (sec_mean/sec_mean.cu:13-93) and
 * global_avg_pool_fp / _bp (roipool/roipool.cu:12-72). inp f32 [S,C]; offsets int32 [nP+1]; out f32 [nP,C].
 * Proposal p covers rows [offsets[p], offsets[p+1]); rows outside every proposal are never read.
 * min/max are exact: every value equals the reference's (`<` / `>` scans: NaN never wins, an empty proposal gives
 * +inf / -inf); only the sign of a zero result is not guaranteed, because the tree reduction cannot reproduce the
 * reference's first-occurrence choice between +0.0 and -0.0. mean / avg-pool sum len/rows_par terms per thread, then a
 * log2(rows_par) tree (rows_par = 256 / min(pow2 >= C, 32)), so per element
 * |out - mean64| <= (ceil(len/rows_par) + log2(rows_par) + 2) * 2^-24 * sum|x| / len; an empty proposal gives 0 (mean) /
 * NaN (avg-pool, 0/0).
 * ------------------------------------------------------------------------------------------- */
int sgb_sec_mean(const float *d_inp, const int32_t *d_offsets, float *d_out, int nProposal, int C, void *stream);
int sgb_sec_min(const float *d_inp, const int32_t *d_offsets, float *d_out, int nProposal, int C, void *stream);
int sgb_sec_max(const float *d_inp, const int32_t *d_offsets, float *d_out, int nProposal, int C, void *stream);
int sgb_global_avg_pool_fp(const float *d_feats, const int32_t *d_offsets, float *d_out, int nProposal, int C,
                           void *stream);
int sgb_global_avg_pool_bp(float *d_d_feats, const int32_t *d_offsets, const float *d_d_out, int nProposal, int C,
                           void *stream);

/* ---------------------------------------------------------------------------------------------
 * Mask IoU / labels -- replace get_mask_iou_on_cluster / get_mask_iou_on_pred / get_mask_label
 * (cal_iou_and_masklabel/cal_iou_and_masklabel.cu:9-164). Training-side ops of the binding surface.
 * proposals_idx here is the POINT-INDEX column (int32 [sumNPoint]); instance_labels int64 [N];
 * d_mask_scores_sigmoid may be NULL (on_cluster). iou f32 [nProposal, nInstance].
 * ------------------------------------------------------------------------------------------- */
int sgb_get_mask_iou(const int32_t *d_proposals_idx, const int32_t *d_proposals_offset,
                     const int64_t *d_instance_labels, const int32_t *d_instance_pointnum,
                     const float *d_mask_scores_sigmoid, float *d_proposals_iou, int nInstance, int nProposal,
                     void *stream);
int sgb_get_mask_label(const int32_t *d_proposals_idx, const int32_t *d_proposals_offset,
                       const int64_t *d_instance_labels, const int64_t *d_instance_cls,
                       const float *d_proposals_iou, int nInstance, int nProposal, float iou_thr,
                       float *d_mask_label, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Sparse convolution -- replaces what the reference delegates to spconv 2.x (call sites
 * softgroup/model/blocks.py:31-41,50-70,96-129; softgroup/model/softgroup.py:60-65,73-74).
 * indices int32 [M,4] (b,x,y,z), b in [0,65535], x,y,z in [0,32766].
 *
 * Rulebooks ("maps"): int32 [K, Mout]; map[k][j] = input row feeding output row j through kernel offset k,
 * or -1. Kernel offset order = row-major (k0,k1,k2) like the weight layout [out,k0,k1,k2,in]
 * (tools/convert_checkpoint.py:17-19).
 *   subm3:   K=27, Mout=M, map[k][j] = row of indices[j] + (k0-1,k1-1,k2-1)           (SubMConv3d k3 p1)
 *            subm3 does not report rows outside the range above: its callers pass indices that voxelize_idx or
 *            down2 have already checked, and reporting would cost a host wait per level. Such a row is nobody's
 *            neighbour, and its own map column holds only its centre entry (map[13][j] = j), -1 elsewhere.
 *   down2:   K=8; output voxels = distinct (b, x>>1, y>>1, z>>1) with every coordinate < out_shape
 *            = floor(shape/2) (inputs on the max plane of an odd dim are dropped), numbered by first
 *            occurrence in input order. count (blocking) returns Mout; fill writes d_out_indices [Mout,4],
 *            d_map [8,Mout] (children) and d_inv_map [8,M] (inv_map[k][i] = parent row if input i is child k
 *            of it, else -1) -- the inverse conv is the same kernel run with inv_map. With Mout = 0 (an axis of
 *            extent 1) d_out_indices and d_map may be NULL.                          (SparseConv3d k2 s2,
 *            SparseInverseConv3d k2)
 * ------------------------------------------------------------------------------------------- */
size_t sgb_rulebook_workspace_bytes(int M);
int sgb_rulebook_subm3(const int32_t *d_indices, int M, int32_t *d_map, void *d_ws, size_t ws_bytes, void *stream);
int sgb_rulebook_down2_count(const int32_t *d_indices, int M, const int32_t *h_spatial_shape /*[3]*/, void *d_ws,
                             size_t ws_bytes, void *stream);
int sgb_rulebook_down2_fill(const int32_t *d_indices, int M, int Mout, int32_t *d_out_indices, int32_t *d_map,
                            int32_t *d_inv_map, void *d_ws, size_t ws_bytes, void *stream);

/* out[j, out_off + n] = sum_k sum_c act(in[map[k][j], in_off + c]) * W[k][c][n]  (+ residual[j, res_off + n]) (+ bias[n])
 * act(x) = x                       if d_in_scale == NULL
 *        = max(x*scale[c]+shift[c], 0)   otherwise (eval-mode BatchNorm1d folded to scale/shift, then ReLU --
 *          the pre-activation of blocks.py:55-70); absent neighbours contribute exactly 0.
 * W is f32 [K, Cin, Cout] (the wrapper permutes the reference layout once). d_map == NULL means K == 1 and the
 * identity map (Custom1x1Subm3d, blocks.py:31-41, and nn.Linear). Row strides are in floats.
 * fp32 accumulate on CUDA cores (fp32-exact products; see DESIGN.md on why not plain TF32). */
int sgb_spconv_forward(const float *d_in, int in_stride, int in_off, const int32_t *d_map, int K, int Mout,
                       const float *d_W, int Cin, int Cout, const float *d_in_scale, const float *d_in_shift,
                       const float *d_residual, int res_stride, int res_off, const float *d_bias, float *d_out,
                       int out_stride, int out_off, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Tensor-core sparse convolution (spconv_tc.cu; wgmma.mma_async f16, fp32 accumulators in registers) -- the production path
 * for Cin <= 512, Cout <= 256. Every operand value x is carried as two fp16 numbers hi = fp16(x),
 * lo = fp16((x - hi) * 2^shift), shift = sgb_spconv_lo_shift(), and the product is hi*hi + hi*lo + lo*hi: fp32-grade
 * (DESIGN.md 3.2). Activations travel PACKED between convolutions: per row and 32-channel chunk 16 words of fp16 hi pairs
 * then 16 words of fp16 lo pairs (one 128-byte line), float32-typed buffers [rows][ceil(C/32)*32 words].
 *   Weights, pre-split and pre-packed by the host (softgroup_b200/spconv/core.py:pack_weight_tc) with the same shift:
 *     N = Cout rounded up to 16, nkc = ceil(Cin/32);
 *     Wp fp16 [K][nkc][4][2][N][8]: element (k, kc, q, part, n, e) = part(W[k][32*kc + 8*q + e][n]) (0 outside Cin/Cout),
 *     part 0 = hi, part 1 = lo -- per (k, kc) the K-major / no-swizzle wgmma B operands B_hi, B_lo of 16-byte chunks;
 *     passed as float* (two halves per word); sgb_spconv_tc_packed_floats = its length in words.
 *   sgb_spconv_forward_tc: d_in_pk packed input [Min][in_stride words] ALREADY activated (the consumer's
 *     BatchNorm(eval)+ReLU was applied by whoever packed it); d_map int32 [K][Mout] (-1 = no neighbour) or NULL for the
 *     identity (K == 1: 1x1 conv / nn.Linear). Outputs, either or both: d_out fp32 rows (strided: concat buffers);
 *     d_pk_out packed rows at channel offset pk_coff (multiple of 8) after y = relu?(x * pk_scale[c] + pk_shift[c]) per
 *     OUTPUT channel c -- the NEXT layer's BatchNorm(eval)+ReLU folded into this producer (an intermediate with a single
 *     consumer never exists in fp32); pk_fill != 0 also zeroes channels [pk_coff + N, round_up32(pk_coff + N)), the rest
 *     of the 32-channel chunk the written channels end in (N = Cout rounded up to 16; padding channels [pk_coff + Cout,
 *     pk_coff + N) are always written as zero), for any pk_coff; channels below pk_coff are never written.
 *   sgb_act_pack: the same packing for tensors without a producing convolution (C real channels, zeros up to Cfill).
 *   sgb_spconv_overflow: a packed value beyond the fp16 range (|y| > 65504, or NaN) raises a per-device flag instead of
 *     saturating silently; this call reads and clears it (blocking 4-byte read on `stream`).
 *   sgb_spconv_tc_plan: the tile configuration the launch uses for a problem size (pure function; sms <= 0: 132):
 *     out[0] = NT (columns per CTA), [1] = column parts, [2] = split-K cluster size, [3] = shared memory per CTA (bytes),
 *     [4] = pipeline stages, [5] = row tiles.
 * ------------------------------------------------------------------------------------------- */
long long sgb_spconv_tc_packed_floats(int K, int Cin, int Cout);
int sgb_spconv_lo_shift(void);
int sgb_spconv_overflow(int *h_flag, void *stream);
int sgb_spconv_tc_plan(int K, int Mout, int Cin, int Cout, int has_map, int sms, int *out);
int sgb_act_pack(const float *d_x, int x_stride, int x_off, const float *d_scale, const float *d_shift, int relu,
                 float *d_pk, int pk_stride, int pk_coff, int M, int C, int Cfill, void *stream);
int sgb_spconv_forward_tc(const float *d_in_pk, int in_stride, int Min, const int32_t *d_map, int K, int Mout,
                          const float *d_Wp, int Cin, int Cout, const float *d_residual, int res_stride, int res_off,
                          const float *d_bias, float *d_out, int out_stride, int out_off, float *d_pk_out, int pk_stride,
                          int pk_coff, const float *d_pk_scale, const float *d_pk_shift, int pk_relu, int pk_fill,
                          void *stream);
/* Two launch forms of one kernel implement sgb_spconv_forward_tc with bit-identical results (same products, same
 * accumulation order; split-K sums partial tiles in rank order):
 *   0 = one CTA per work item (128 rows x NT columns), column split and split-K thread-block clusters for the deep
 *       U-Net levels, 1 = persistent (as many CTAs as fit on the GPU walk the work items).
 * sgb_spconv_kernel_choice: which form sgb_spconv_forward_tc runs for a problem size (sms <= 0: 132).
 * sgb_spconv_forward_tc_ex: the same call with the form named explicitly (-1 = choose) -- parity tests and A/B tools. */
int sgb_spconv_kernel_choice(int K, int Mout, int Cin, int Cout, int sms);
int sgb_spconv_forward_tc_ex(const float *d_in_pk, int in_stride, int Min, const int32_t *d_map, int K, int Mout,
                             const float *d_Wp, int Cin, int Cout, const float *d_residual, int res_stride, int res_off,
                             const float *d_bias, float *d_out, int out_stride, int out_off, float *d_pk_out, int pk_stride,
                             int pk_coff, const float *d_pk_scale, const float *d_pk_shift, int pk_relu, int pk_fill, int kernel,
                             void *stream);

/* ---------------------------------------------------------------------------------------------
 * Per-class point selection in front of the ball query, all classes in one pass (grouping.cu) -- replaces the loop body
 * softgroup/model/softgroup.py:430-446 (`(scores[:, class_id] > score_thr).nonzero()`, the `min_npoint` skip, the gathers
 * of batch_idxs / coords_float / pt_offsets) for the classes h_classes[0..nc) (host array, any nc >= 1, ids in [0, C);
 * N * nc and nc * B below 2^31):
 *   entries in class-major, ascending point order: d_pts[e] = point, d_seg[e] = rank(class) * B + batch_idxs[point],
 *   d_shifted[e] = coords[point] + offsets[point] (fp32), all with capacity N * nc; d_seg_offsets int32 [nc*B + 1] =
 *   first entry of every (class, batch item) segment; d_total int32 [1 + nc] = number of entries, then entries per class
 *   (0 for a class below min_npoint). d_scores = softmax scores [N][C]. No host synchronisation and no host-to-device
 *   copy: the class ids travel in the kernel parameters, 256 per launch (4 launches up to 256 classes, one more per
 *   further 256). The segments feed sgb_ballquery_batch_p_async, which takes at most 1023 of them: nc * B <= 1023 there.
 * ------------------------------------------------------------------------------------------- */
size_t sgb_group_entries_workspace_bytes(int N, int nc, int B);
int sgb_group_entries(const float *d_scores, int N, int C, const int *h_classes, int nc, float score_thr, int min_npoint,
                      const int32_t *d_batch_idxs, int B, const float *d_coords, const float *d_offsets, int32_t *d_pts,
                      int32_t *d_seg, float *d_shifted, int32_t *d_seg_offsets, int32_t *d_total, void *d_ws, size_t ws_bytes,
                      void *stream);

/* y[i, c] = max(x[i, c]*scale[c] + shift[c], 0) (relu != 0) -- BatchNorm1d(eval)+ReLU over rows. */
int sgb_bn_relu(const float *d_x, int x_stride, const float *d_scale, const float *d_shift, int relu, float *d_y,
                int y_stride, int M, int C, void *stream);

/* out[i, :] = in[index[i], :]  (the "devoxelize" gather of softgroup.py:374); index int32 [N]. */
int sgb_gather_rows(const float *d_in, const int32_t *d_index, float *d_out, int N, int C, void *stream);

/* Host-side serialisation of instance masks into the reference's RLE wire format (softgroup/util/rle.py:5-19:
 * dict(length, counts='start len start len ...'), 1-based starts). h_ids: ascending point ids of all masks back to
 * back (int32), h_offs int64 [n_masks+1]. Writes the `counts` strings back to back into h_out and their byte ranges
 * into h_out_offs [n_masks+1]. Returns bytes written, or SGB_ERR_OVERFLOW if out_cap is too small
 * (12 bytes per run + 2 always suffices). No CUDA involved. */
long long sgb_rle_format_ids(const int32_t *h_ids, const long long *h_offs, int n_masks, char *h_out,
                             long long out_cap, long long *h_out_offs);

/* ---------------------------------------------------------------------------------------------
 * Instance masks, RLE, panoptic paste and evaluation intersections on the GPU (instances.cu) -- replace the dense
 * [nProposal, N] masks + numpy RLE of get_instances (softgroup/model/softgroup.py:537-604, softgroup/util/rle.py:5-19),
 * the numpy paste loop of panoptic_fusion (softgroup.py:606-639) and the per-pair np.count_nonzero of
 * ScanNetEval.assign_instances_for_scan (softgroup/evaluation/instance_eval.py:262-293).
 * Masks are bitmaps [rows][W], W = sgb_bitmap_words(N) = ceil((N+1)/32) 32-bit words (bit N always 0).
 *   sgb_inst_count:   npoint[p*nI+i] = #entries of proposal p with mask_scores[e,i] > thr (zeroed here).
 *   sgb_inst_scatter: bitmaps (zeroed here) of the kept instances; slot int32 [nI*nP], class-major (i*nP+p): bitmap row or -1.
 *   sgb_bitmap_set:   generic (row, point) -> bit; clear != 0 zeroes the bitmaps first.
 *   sgb_rle_count (blocking) / sgb_rle_fill: 1-based transition positions of every mask, ascending = `runs` of rle.py:15
 *     before `runs[1::2] -= runs[::2]`; inst_off int32 [n_inst+1]. sgb_rle_format_runs (host): the `counts` strings.
 *   sgb_bitmap_intersections: inter[r*nG+g], vert[r], void[r] from gslot int32 [N] (>= 0: gt column, -2: void, -1: other).
 *   sgb_panoptic_paste: instances visited in d_order; skipped when intersect/(size+1e-5) > skip_iou (float64), else
 *     pasted where nothing was pasted before: pan_cls[pt] = d_cls[row], pan_ids[pt] = 1, 2, ... in paste order.
 *   sgb_bitmap_ids_count / sgb_bitmap_ids_fill: rows -> ascending point-id lists (bits >= N ignored). count: offsets
 *     int64 [n_rows+1] (offsets[n_rows] = total), no host wait; fill, same workspace and stream: ids int32 [total].
 *   sgb_class_bitmaps: bitmaps (zeroed here) with bit pt of row row_of_label[labels[pt]] (labels int64 [N], rows < 0 and
 *     labels outside [0, n_labels) set nothing); counts int64 [n_rows] (may be null) = set bits per row.
 * ------------------------------------------------------------------------------------------- */
int sgb_inst_count(const int32_t *d_proposals_idx, const float *d_mask_scores, int ms_stride, int S, int nI, float thr,
                   int32_t *d_npoint, int nP, void *stream);
size_t sgb_bitmap_words(int N);
int sgb_inst_scatter(const int32_t *d_proposals_idx, const float *d_mask_scores, int ms_stride, int S, int nI, int nP, float thr,
                     const int32_t *d_slot, uint32_t *d_bitmaps, int n_inst, int N, void *stream);
int sgb_bitmap_set(const int32_t *d_row, const int32_t *d_pt, long long n, uint32_t *d_bitmaps, int n_rows, int N, int clear,
                   void *stream);
size_t sgb_rle_workspace_bytes(int n_inst, int N);
long long sgb_rle_count(const uint32_t *d_bitmaps, int n_inst, int N, void *d_ws, size_t ws_bytes, void *stream);
int sgb_rle_fill(const uint32_t *d_bitmaps, int n_inst, int N, int total_trans, int32_t *d_trans, int32_t *d_inst_off, void *d_ws,
                 size_t ws_bytes, void *stream);
long long sgb_rle_format_runs(const int32_t *h_trans, const int32_t *h_offs, int n_masks, char *h_out, long long out_cap,
                              long long *h_out_offs);
int sgb_bitmap_intersections(const uint32_t *d_bitmaps, int n_rows, int N, const int32_t *d_gslot, int nG, int32_t *d_inter,
                             int32_t *d_vert, int32_t *d_void, void *stream);
int sgb_panoptic_paste(const uint32_t *d_bitmaps, int N, const int32_t *d_order, const int32_t *d_cls, int n_inst, double skip_iou,
                       uint32_t *d_prev, uint32_t *d_pan_cls, uint32_t *d_pan_ids, void *stream);
size_t sgb_bitmap_ids_workspace_bytes(int n_rows, int N);
int sgb_bitmap_ids_count(const uint32_t *d_bitmaps, int n_rows, int N, long long *d_offsets, void *d_ws, size_t ws_bytes,
                         void *stream);
int sgb_bitmap_ids_fill(const uint32_t *d_bitmaps, int n_rows, int N, int32_t *d_ids, void *d_ws, size_t ws_bytes, void *stream);
int sgb_class_bitmaps(const int64_t *d_labels, int N, const int32_t *d_row_of_label, int n_labels, uint32_t *d_bitmaps, int n_rows,
                      long long *d_counts, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Point-id lists (the instances of forward_test(device_results=True)): list k is d_ids[d_offsets[k] .. d_offsets[k+1]),
 * d_offsets int64 [n+1] non-decreasing with d_offsets[0] = 0 and d_offsets[n] = total, d_ids int32 [total], ids in [0, N).
 * n may be any int, total any int64 (beyond 2^31 included). Ids outside [0, N) are never dereferenced: they count for no
 * op and in no count. Both calls enqueue on `stream` and never wait for the host; the id space is cut into fixed
 * 256-id chunks, so one long list or many short ones spread over the whole GPU alike.
 *   sgb_id_lists_reduce: per list and channel, over the rows d_values[id * ld + c] (f32 [N, C], row stride ld >= C, any
 *     C >= 1) of its ids, the ops in `ops` (SGB_REDUCE_* mask): d_min / d_max / d_mean f32 [n, C] (NULL when not asked
 *     for), and d_counts int64 [n] (always) = ids in [0, N) per list.
 *     min / max are exact, with the semantics of sgb_sec_min / sgb_sec_max: NaN never wins, an empty list gives +inf /
 *     -inf, only the sign of a zero result is unspecified.
 *     mean: float64 partial sums over each 256-id chunk, combined in chunk order (no float atomics), so the same bits on
 *     every run; an empty list gives NaN. Not order-exact: per element, with len the count and mean64 the float64 mean,
 *     |out - mean64| <= 2^-24 * |mean64| + (len/256 + 300) * 2^-52 * sum|x| / len.
 *     Launches: 2 (1 when total = 0; none when n = 0). Workspace: sgb_id_lists_reduce_workspace_bytes(total, C).
 *   sgb_id_lists_point_map: d_map int32 [N]: map[p] = the k of the highest d_conf[k] (f32 [n]) among the lists holding p;
 *     ties go to the smaller k, -0.0 ties with +0.0, a NaN confidence ranks below every number (-inf included), and a
 *     point in no list gets -1. One pass does a 64-bit atomicMax of (ordered bits of conf, ~k) per id into a per-point
 *     key, a second decodes it: the result does not depend on execution order. Launches: 2 (1 when n or total is 0), after
 *     one memset. Workspace: sgb_id_lists_point_map_workspace_bytes(N).
 * ------------------------------------------------------------------------------------------- */
#define SGB_REDUCE_MIN 1
#define SGB_REDUCE_MAX 2
#define SGB_REDUCE_MEAN 4
size_t sgb_id_lists_reduce_workspace_bytes(long long total, int C);
int sgb_id_lists_reduce(const long long *d_offsets, const int32_t *d_ids, int n, long long total, int N, const float *d_values,
                        long long ld, int C, int ops, float *d_min, float *d_max, float *d_mean, long long *d_counts, void *d_ws,
                        size_t ws_bytes, void *stream);
size_t sgb_id_lists_point_map_workspace_bytes(int N);
int sgb_id_lists_point_map(const long long *d_offsets, const int32_t *d_ids, int n, long long total, int N, const float *d_conf,
                           int32_t *d_map, void *d_ws, size_t ws_bytes, void *stream);

/* sgb_id_lists_fps: farthest-point sampling of K >= 1 points per list (same lists as above), d_out int32 [n, K] (int64
 * indexing: n * K may exceed 2^31). Points are d_xyz f32 [N, 3] rows (x, y, z at d_xyz[id * ld + 0..2], ld >= 3).
 * For list k, positions i = 0 .. len-1 hold ids p_i; position i is valid when 0 <= p_i < N. Invalid ids are never
 * dereferenced and never chosen.
 *   1. No valid position: row k is all -1.
 *   2. s_0 = the smallest valid position; d_i = +inf for every valid i.
 *   3. For j = 1 .. K-1: for every valid i, d_i = minimum(d_i, dist(i, s_{j-1})), where a NaN operand gives NaN (as
 *      np.minimum); s_j = the valid position with the largest d_i, a NaN ranking below every number, ties going to the
 *      smaller position.
 *   4. out[k, j] = p_{s_j}.
 * dist is float32, every operation rounded to nearest, no contraction, in this order: dx = x_i - x_s, dy, dz, then
 * (dx*dx + dy*dy) + dz*dz; numpy's float32 dx*dx + dy*dy + dz*dz gives the same bits. The argmax is a max over the 64-bit
 * key (0 for NaN, else the bits of d + 1 : 0xFFFFFFFF - position), so the result does not depend on the reduction
 * order. When a list has fewer distinct points than K, the tail repeats one position's id (s_0's when the points are
 * finite), as the tie rule implies. A list of more than 2^31 - 1 positions is outside this contract: its row is -1.
 * Granularity, by list length (positions, valid or not): up to SGB_FPS_WARP_MAX one warp, up to SGB_FPS_CTA_MAX one
 * CTA, beyond that one 8-CTA thread-block cluster, which keeps up to SGB_FPS_CLUSTER_MAX positions on chip and streams
 * longer lists from global memory every step (their d in the workspace). A bin pass sorts the lists into one queue per
 * granularity; the three kernels have fixed grids and pull lists from their queue. Enqueued on `stream`, no host wait.
 * Launches: SGB_FPS_LAUNCHES whatever the data (none when n = 0), after one memset.
 * Workspace: sgb_id_lists_fps_workspace_bytes(n, total) = three int32 queues of n lists plus 4 bytes per id. */
#define SGB_FPS_WARP_MAX 512
#define SGB_FPS_CTA_MAX 8192
#define SGB_FPS_CLUSTER_MAX 65536
#define SGB_FPS_LAUNCHES 4
size_t sgb_id_lists_fps_workspace_bytes(int n, long long total);
int sgb_id_lists_fps(const long long *d_offsets, const int32_t *d_ids, int n, long long total, int N, const float *d_xyz,
                     long long ld, int K, int32_t *d_out, void *d_ws, size_t ws_bytes, void *stream);

/* Test-time transform of the reference dataloader, first step (softgroup/data/custom.py:87-107,162-164):
 * out[i, :] = xyz[i, :] @ m in float64 (xyz float32 [N,3] device, m float64 [3,3] row-major HOST, out float64 [N,3] device),
 * accumulated like the BLAS kernels numpy calls: fma(z, m2j, fma(y, m1j, x * m0j)). */
int sgb_affine3_f64(const float *d_xyz, const double *h_m9, double *d_out, int N, void *stream);


/* ---------------------------------------------------------------------------------------------
 * Sparse U-Net executor (unet.cu): runs n_ops records of a plan in one call. The plan (array of sgb_unet_op) is compiled
 * once per model by softgroup_b200/model/unet_plan.py from the module tree of softgroup/model/blocks.py:44-143, fused
 * across modules (consumer BatchNorm+ReLU in the producer's epilogue, packed activations, residual / concat writes in
 * epilogues); per scan the caller supplies row counts M[level], rulebooks per level (subm [27][M_l], down [8][M_{l+1}],
 * inverse [8][M_l]) and one pointer per plan buffer. Results do not depend on how the ops are split into calls.
 * ------------------------------------------------------------------------------------------- */
enum { SGB_UNET_CONV = 1, SGB_UNET_ACT_PACK = 2, SGB_UNET_BN_RELU = 4 };
typedef struct sgb_unet_op {
  int32_t kind;                     /* SGB_UNET_* */
  int32_t level_in, level_out;      /* rows of the input / output: M[level] */
  int32_t map_kind;                 /* CONV: 0 identity (K = 1), 1 subm of level_out, 2 down level_in -> level_in + 1, 3 inverse -> level_out */
  int32_t K, Cin, Cout;             /* ACT_PACK: Cin = real channels, Cout = fill width; BN_RELU: Cin = channels */
  int32_t in_buf, in_stride, in_off;          /* fp32 source (ACT_PACK, BN_RELU) */
  int32_t pk_in_buf, pk_in_stride;            /* CONV: packed input, row stride in words */
  int32_t out_buf, out_stride, out_off;       /* fp32 destination (-1: none) */
  int32_t pk_out_buf, pk_out_stride, pk_out_coff, pk_fill, relu;  /* packed destination (-1: none) */
  int32_t res_buf, res_stride, res_off;       /* CONV: residual rows (-1: none) */
  const float *Wp, *bias, *scale, *shift;     /* device pointers: packed weights, bias, BatchNorm scale / shift of the op */
} sgb_unet_op;
int sgb_unet_run(const sgb_unet_op *ops, int n_ops, float *const *bufs, const int32_t *const *subm_maps,
                 const int32_t *const *down_maps, const int32_t *const *inv_maps, const int *M, int n_levels, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SGB200_H */
