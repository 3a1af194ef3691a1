// yb_conv_tc.cuh -- interface of the tensor-core (wgmma / TMA) implicit-GEMM convolutions
// (implemented in yb_conv_tc.cu).
#pragma once
#include <cuda_runtime.h>

#include "yb_kernels.cuh"
#include "yb_model.h"

namespace yb {

// non-zero if the bf16 tensor-core kernel takes this layer (input view `in`, bf16 or f32 output)
int tc_conv_supported(const Layer &l, const TV &in, const TV &out, bool out_bf16);
// builds the per-layer launch state (TMA tensor maps, tile schedule); throws yb::Error on failure.
// wide_rows: prefer wide pixel tiles (the plan will get tc_plan_fuse_yolo: NCHW plane stores in the epilogue)
// res: fused shortcut operand (bf16; needs a bf16 output)
void *tc_make_plan(const Layer &l, const TV &in, const TV &out, bool out_bf16, const TV &res, bool res_bf16,
                   int act2, const void *d_weights_bf16, int ldn, const float *d_bias, int wide_rows = 0);
// tf32 variant for the FP32 detection heads of the exact (INT8 / XNOR) networks: f32 in, f32 [ldn][K] weights, f32 out
int tc_tf32_supported(const Layer &l, const TV &in, const TV &out);
void *tc_make_plan_tf32(const Layer &l, const TV &in, const TV &out, const void *d_weights_f32, int ldn, const float *d_bias,
                        int wide_rows);
// INT8 (s8 wgmma) variant; want_pool_tile: 8 x 16 pixel tiles, so that tc_plan_fuse_pool can fuse the following max-pool
int tc_i8_supported(const Layer &l, const TV &q, const TV &out);
void *tc_make_plan_i8(const Layer &l, const TV &q, const TV &out, const void *d_weights_s8, int ldn, const float *d_bias,
                      float alpha1, int *acc_out, int want_pool_tile = 0);
// XNOR layer as +-1 s8 on the s8 wgmma (q: s8 activation with -1 borders)
void *tc_make_plan_xnor(const Layer &l, const TV &q, const TV &out, const void *d_weights_pm1, int ldn, const float *d_bias,
                        const float *d_mean, int *counts_out, int want_pool_tile = 0);
// non-zero if an integer plan of `l` made with want_pool_tile takes tc_plan_fuse_pool (qnext: the next integer layer's input)
int tc_pool_fuse_supported(const Layer &l, const TV &qnext);
// fuse the following 2x2/2 max-pool + the next integer layer's input conversion (1: s8 quantised, 2: +-1 bytes) into an integer
// plan; the plan then writes no output of its own (`out` may have no base)
void tc_plan_fuse_pool(void *plan, int mode, float mult, const TV &qnext);
// fuse the following [yolo] layer into the (f32-output) plan: logistic + NCHW store in the epilogue; the plan then writes no
// NHWC output (`out` may have no base)
void tc_plan_fuse_yolo(void *plan, float *d_yolo_nchw, int classes);
// tensor-core stem (3-channel 3x3 from the caller's NCHW f32 image, bf16 NHWC out)
int tc_stem_supported(const Layer &l, const TV &out);
void *tc_stem_make_plan(const Layer &l, const TV &out, const void *d_w_32x32_bf16, const float *d_bias);
// the tensor-core stem fused with layer 1, a 3x3 / stride-2 convolution 32 -> 64 filters (bf16 out1): the stem output never
// reaches HBM.  The plan takes the same launch / free calls as the stem's.
int tc_stem_s2_supported(const Layer &l0, const Layer &l1, const TV &out1);
void *tc_stem_s2_make_plan(const Layer &l0, const Layer &l1, const TV &out1, const void *d_w_32x32_bf16, const float *d_bias,
                           const void *d_w1_bf16, const float *d_bias1);
void tc_stem_launch(void *plan, const float *d_in_nchw, cudaStream_t s);
void tc_stem_launch_u8(void *plan, const unsigned char *d_in_hwc, cudaStream_t s);   // frames already of the network size
void tc_stem_free_plan(void *plan);
void tc_launch(void *plan, cudaStream_t s);
void tc_free_plan(void *plan);

}  // namespace yb
