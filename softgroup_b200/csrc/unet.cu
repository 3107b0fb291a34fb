// unet.cu -- executor of a compiled sparse U-Net plan: the ~170 convolution / pack launches of one backbone pass issued
// from ONE C call instead of ~170 Python->ctypes round trips (the host side of the forward was the bottleneck once the
// kernels got faster: Python spent longer per convolution than the GPU).
// The plan is data: softgroup_b200/model/unet_plan.py walks the module tree of the reference-shaped model
// (softgroup/model/blocks.py:44-143 -- ResidualBlock / UBlock) once and emits one record per launch, fused across modules
// (BatchNorm+ReLU of the consumer folded into the producing conv's epilogue, packed activations between convs, residual
// adds and concat writes in the epilogues). Per scan only the row counts, the rulebook pointers and the buffer pointers
// change. The caller runs a segment of ops per call, or one op per call when it times each launch.
#include "common.cuh"

extern "C" int sgb_unet_run(const sgb_unet_op *ops, int n_ops, float *const *bufs, const int32_t *const *subm_maps,
                            const int32_t *const *down_maps, const int32_t *const *inv_maps, const int *M, int n_levels,
                            void *stream) {
  SGB_REQUIRE(ops && bufs && M && n_ops >= 0 && n_levels >= 1, SGB_ERR_ARG, "unet_run arguments");
  for (int i = 0; i < n_ops; i++) {
    const sgb_unet_op &o = ops[i];
    SGB_REQUIRE(o.level_in >= 0 && o.level_in < n_levels && o.level_out >= 0 && o.level_out < n_levels, SGB_ERR_ARG,
                "unet_run: level out of range");
    const int Min = M[o.level_in], Mout = M[o.level_out];
    int rc = SGB_OK;
    switch (o.kind) {
      case SGB_UNET_CONV: {
        const int32_t *map = nullptr;
        if (o.map_kind == 1) map = subm_maps[o.level_out];
        else if (o.map_kind == 2) map = down_maps[o.level_in];   // [8][M of level_in + 1]
        else if (o.map_kind == 3) map = inv_maps[o.level_out];   // [8][M of level_out]
        SGB_REQUIRE(o.map_kind == 0 || map, SGB_ERR_ARG, "unet_run: missing rulebook");
        if (Min == 0 || Mout == 0) break;
        rc = sgb_spconv_forward_tc(bufs[o.pk_in_buf], o.pk_in_stride, Min, map, o.K, Mout, o.Wp, o.Cin, o.Cout,
                                   o.res_buf >= 0 ? bufs[o.res_buf] : nullptr, o.res_stride, o.res_off, o.bias,
                                   o.out_buf >= 0 ? bufs[o.out_buf] : nullptr, o.out_stride, o.out_off,
                                   o.pk_out_buf >= 0 ? bufs[o.pk_out_buf] : nullptr, o.pk_out_stride, o.pk_out_coff, o.scale,
                                   o.shift, o.relu, o.pk_fill, stream);
        break;
      }
      case SGB_UNET_ACT_PACK:
        rc = sgb_act_pack(bufs[o.in_buf], o.in_stride, o.in_off, o.scale, o.shift, o.relu, bufs[o.pk_out_buf], o.pk_out_stride,
                          o.pk_out_coff, Min, o.Cin, o.Cout, stream);  // Cout = fill width
        break;
      case SGB_UNET_BN_RELU:
        rc = sgb_bn_relu(bufs[o.in_buf] + o.in_off, o.in_stride, o.scale, o.shift, o.relu, bufs[o.out_buf] + o.out_off, o.out_stride,
                         Min, o.Cin, stream);
        break;
      default:
        SGB_REQUIRE(false, SGB_ERR_ARG, "unet_run: unknown op kind");
    }
    if (rc) return rc;
  }
  return SGB_OK;
}
