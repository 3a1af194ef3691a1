// yb_conv_tc.cuh -- interface of the tensor-core (wgmma / TMA) implicit-GEMM convolutions
// (implemented in yb_conv_tc.cu).
#pragma once
#include <cuda_runtime.h>

#include <memory>

#include "yb_device.cuh"
#include "yb_model.h"

namespace yb {

// The diagnostic switches of the tensor-core plans (DESIGN, appendix), read with the engine's
struct TcSwitches {
    int bn = 0;              // YB_TC_BN: k_conv_tc_reg filter-tile width, rounded down to a power of two >= 32; 0 unset
    int grid = 0;            // YB_TC_GRID: at most this many CTAs per persistent grid; <= 0 no cap
    bool no_bstat = false;   // YB_TC_NO_BSTAT: the ring streams the filter tiles, none stays resident
    bool stats = false;      // YB_TC_STATS: run the role-counter instantiations, print their counters when the plan is freed
    int dbg = 0;             // YB_TC_DBG: bit mask of bottleneck experiments
};

// One tensor-core convolution: the layer, its operands and what its epilogue fuses.  tc_conv_supported also takes views rooted
// at any base with the activation arena's alignment, with the device pointers left null.
struct TcConv {
    TcKind kind = TC_BF16;
    const Layer *l = nullptr;
    TV in{};                       // padded NHWC activations (bf16 / f32); integer kinds: the s8 input, channels zero-padded to in.ldc
    TV out{};                      // padded NHWC output; no base where a fused [yolo] or max-pool takes its place
    bool out_bf16 = false;
    TV res{};                      // fused shortcut operand (bf16, as the output), or no base
    int act2 = ACT_LINEAR;         // activation after the shortcut add
    const void *w = nullptr;       // [ldn][K] filter matrix, K ordered (ky, kx, c); integer kinds: c padded to in.ldc
    int ldn = 0;
    const float *bias = nullptr;
    float alpha1 = 0.f;            // TC_S8: R_MULT / (input_mult * weights_mult); TC_S8_GPU: 1 / (input_mult * weights_mult)
    const float *mean = nullptr;   // TC_XNOR, TC_XNOR_GPU, TC_PM1Z_GPU: per-filter mean |w|
    int *acc_out = nullptr;        // integer kinds: raw s32 accumulators / popcounts, NCHW (tests), or null
    float *yolo_out = nullptr;     // fused [yolo] layer: its NCHW f32 output, or null
    int yolo_classes = 0;
    SideFmt pool_fmt = SIDE_NONE;  // fused 2x2/2 max-pool + the next integer layer's input conversion into this format; SIDE_NONE: none
    float pool_mult = 0.f;         // SIDE_S8, SIDE_S8_SAT: the next layer's input multiplier
    TV pool_next{};                // the next integer layer's input
    TcSwitches sw{};
};

// The launch state of a tensor-core convolution (TMA tensor maps, tile schedule) and of a tensor-core stem
struct TcPlan;
struct StemPlan;
struct TcPlanDelete {
    void operator()(TcPlan *plan) const;     // with YB_TC_STATS set, prints the plan's cycle counters first
    void operator()(StemPlan *plan) const;
};
using TcPlanPtr = std::unique_ptr<TcPlan, TcPlanDelete>;
using StemPlanPtr = std::unique_ptr<StemPlan, TcPlanDelete>;

// non-zero if the tensor-core kernels take this convolution, fusions included
int tc_conv_supported(const TcConv &c);
// builds the plan of a supported convolution; throws yb::Error on failure
TcPlanPtr tc_make_plan(const TcConv &c);
void tc_launch(const TcPlan &plan, cudaStream_t s);

// tensor-core stem (3-channel 3x3 from the caller's NCHW f32 image, bf16 NHWC out)
int tc_stem_supported(const Layer &l, const TV &out);
StemPlanPtr tc_stem_make_plan(const Layer &l, const TV &out, const void *d_w_32x32_bf16, const float *d_bias);
// the tensor-core stem fused with layer 1, a 3x3 / stride-2 convolution 32 -> 64 filters (bf16 out1): the stem output never
// reaches HBM.  The plan takes the same launch calls as the stem's.  max_grid > 0 caps its persistent grid (YB_TC_GRID).
int tc_stem_s2_supported(const Layer &l0, const Layer &l1, const TV &out1);
StemPlanPtr tc_stem_s2_make_plan(const Layer &l0, const Layer &l1, const TV &out1, const void *d_w_32x32_bf16,
                                 const float *d_bias, const void *d_w1_bf16, const float *d_bias1, int max_grid);
void tc_stem_launch(const StemPlan &plan, const float *d_in_nchw, cudaStream_t s);
void tc_stem_launch_u8(const StemPlan &plan, const unsigned char *d_in_hwc, cudaStream_t s);   // frames already of the network size

// What a plan decided, for tests (read-only): up to n of {kernel (TC_PLAN_*), kind (TcKind), TW, TH, BN, BK, nt, bstat,
// stages, sps, grid, num_work, tma_epi, jshift, out_ldc (the output's pixel stride in elements, 0 without an NHWC output)}
// into fields; returns how many were written.  The stem plans report kernel, kind, grid, num_work (tiles) and out_ldc, and
// k_stem_s2_tc its S2_TW x S2_TH tiles of layer-1 pixels and its 64 filters as TW, TH, BN; every other field is -1.
enum { TC_PLAN_CONV = 0, TC_PLAN_CONV_REG = 1, TC_PLAN_STEM = 2, TC_PLAN_STEM_S2 = 3, TC_PLAN_NFIELDS = 15 };
int tc_plan_fields(const TcPlan &plan, int *fields, int n);
int tc_stem_plan_fields(const StemPlan &plan, int *fields, int n);

}  // namespace yb
