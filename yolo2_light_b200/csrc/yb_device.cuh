// yb_device.cuh -- what the SIMT kernels (yb_kernels.cuh) and the tensor-core kernels (yb_conv_tc.cu) share: the tensor view,
// the activations, the operand kinds and, defined once, the integer layers' arithmetic -- the conversion of an f32 activation
// into an integer convolution's input and the reference's float epilogues of the XNOR and INT8 convolutions, chosen per
// arithmetic by IntEpi.  Every kernel that converts or finishes an integer layer calls these, so all of them stay
// bit-identical to the reference together.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace yb {

struct TV {            // tensor view (POD, passed by value to kernels)
    char *base;        // address of channel 0 of padded pixel (n=0, y=-P, x=-P)
    int N, H, W, C;
    int ldc;           // elements per pixel in the underlying buffer
    int P;             // border
    int Hp, Wp;        // H+2P, W+2P
};

template <typename T>
__device__ __forceinline__ T *tv_px(const TV &t, int n, int y, int x) {
    return reinterpret_cast<T *>(t.base) + ((size_t)(n * t.Hp + y + t.P) * t.Wp + (x + t.P)) * (size_t)t.ldc;
}

// a view of esz-byte elements whose every pixel starts 16-byte aligned: a 16-byte aligned base and pixel stride.  Every
// kernel that loads or stores 16 bytes of a pixel's channels at a time is placed only on such a view.
__host__ __device__ __forceinline__ bool vec16_view(const TV &t, int esz) {
    return (reinterpret_cast<uintptr_t>(t.base) & 15) == 0 && t.ldc * esz % 16 == 0;
}

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

enum { ACT_LOGISTIC = 0, ACT_RELU = 1, ACT_LINEAR = 3, ACT_LEAKY = 7 };

// activate(), reference additionally.h:126-157 (scalar build): leaky = x>0 ? x : (float)(.1 * (double)x),
// logistic = (float)(1./(1.+exp(-x))) in double.  Used by the "exact" paths.
__device__ __forceinline__ float act_exact(float x, int a) {
    if (a == ACT_LEAKY) return (x > 0.f) ? x : (float)(0.1 * (double)x);
    if (a == ACT_LINEAR) return x;
    if (a == ACT_LOGISTIC) return (float)(1.0 / (1.0 + exp(-(double)x)));
    if (a == ACT_RELU) return x * (x > 0.f);
    return x;
}

// The arithmetic of a convolution, decided once per convolution by the engine's layer plan (Builder::conv_arith).  The five
// integer ones are defined by IntEpi below.
enum Arith {
    AR_F32,            // float convolution
    AR_XNOR_PM1_F32,   // CPU XNOR rule, stride != 1 or pad != 1: the reference's float-GEMM fallback over +-1 floats
    AR_XNOR,           // CPU XNOR rule: popcounts, xnor_epilogue
    AR_XNOR_GPU,       // GPU XNOR rule, c % 32 == 0 (path A): the bit GEMM's count, xnor_gpu_epilogue
    AR_PM1Z_GPU,       // GPU XNOR rule, c < 32 (path B): zero-padded +-1 convolution, pm1z_gpu_epilogue
    AR_INT8,           // CPU INT8 rule: s8 quant_i8 inputs, int8_epilogue
    AR_INT8_GPU,       // GPU INT8 rule: s8 quant_i8_sat inputs, int8_gpu_epilogue
};

// Operand types of a tensor-core convolution
enum TcKind {
    TC_BF16 = 0,   // bf16 x bf16 -> f32; bf16 or f32 output
    TC_S8 = 1,     // INT8: s8 x s8 -> s32, the reference's exact requantising epilogue; f32 output
    TC_XNOR = 2,   // XNOR layer as +-1 s8 on the s8 wgmma (dot = 2*count - K exactly); f32 output
    TC_TF32 = 3,   // f32 operands read as tf32: the float detection heads of the exact (INT8 / XNOR) networks, and every float
                   // convolution of the GPU INT8 rule; f32 output
    TC_S8_GPU = 4, // INT8 of the GPU rule: s8 x s8 -> s32, the unscaled epilogue int8_gpu_epilogue; f32 output
    TC_XNOR_GPU = 5,  // XNOR layer of the GPU XNOR rule, c % 32 == 0: TC_XNOR's GEMM, the bit GEMM's epilogue xnor_gpu_epilogue
    TC_PM1Z_GPU = 6,  // XNOR layer of the GPU XNOR rule, c < 32: +-1 s8 (SIDE_PM1Z_S8) x +-1 s8 -> s32, pm1z_gpu_epilogue
};

// The converted ("side") input of an integer convolution, padded NHWC.  The four integer formats are what the kernels write;
// SIDE_NONE and SIDE_PM1_F32 occur only in the engine's layer plan.
enum SideFmt {
    SIDE_NONE = 0,   // no converted input (f32 convolutions); as a fusion: none
    SIDE_PM1_F32,    // +-1 floats (k_binarize_pm1): the XNOR layers that take the reference's float-GEMM fallback
    SIDE_S8,         // s8 quant_i8(x, the layer's input multiplier): INT8 convolutions
    SIDE_PM1_S8,     // +-1 bytes, +1 where x > 0: XNOR layers on the s8 wgmma
    SIDE_BITS,       // sign bits, bit = (x > 0), 32 channels per 32-bit word: XNOR layers on the popcount kernels
    SIDE_S8_SAT,     // s8 quant_i8_sat(x, the layer's input multiplier): INT8 convolutions of the GPU rule
    SIDE_PM1Z_S8,    // +-1 bytes, +1 where x >= 0, zero border: XNOR layers below 32 channels under the GPU XNOR rule
};

// channels per 32-bit word of an integer side format
__host__ __device__ constexpr int side_per_word(SideFmt f) { return f == SIDE_BITS ? 32 : 4; }
// the formats the kernels write: everything but the plan-only SIDE_NONE and SIDE_PM1_F32
__host__ __device__ constexpr bool side_int(SideFmt f) {
    return f == SIDE_S8 || f == SIDE_PM1_S8 || f == SIDE_BITS || f == SIDE_S8_SAT || f == SIDE_PM1Z_S8;
}
// the s8 formats of the INT8 layers: the byte is the quantised activation under the layer's input multiplier
__host__ __device__ constexpr bool side_s8(SideFmt f) { return f == SIDE_S8 || f == SIDE_S8_SAT; }

// INT8 input quantisation (reference yolov2_forward_network_quantized.c:527-631): xq = clamp(+-127, (int16_t)(x * input_mult))
// with x86 float->int16 semantics (cvttss2si, low 16 bits, indefinite -> 0).  NaN and -inf give 0, and so does -FLT_MAX for
// every multiplier >= 2^-97.
__device__ __forceinline__ int quant_i8(float x, float mult) {
    const float v = __fmul_rn(x, mult);
    int i;
    if (!(v > -2147483648.0f && v < 2147483648.0f)) i = (int)0x80000000;
    else i = __float2int_rz(v);
    int s = (int)(short)(i & 0xffff);
    if (s > 127) s = 127;
    if (s < -127) s = -127;
    return s;
}

// INT8 input quantisation of the GPU rule (cuda_f32_to_int8 + max_abs, reference gpu.cu:730-739): v = x * input_mult rounded
// once, converted to int as CUDA does it (truncation, saturating at +-2^31, NaN -> 0), then clamped to +-127.  It agrees with
// quant_i8 for |v| < 32768; above that quant_i8 wraps through int16 and this saturates (v = 40000: -127 there, +127 here).
// v <= -2^31 (and -inf) gives -127 here: max_abs read without overflow.  The reference evaluates abs(INT_MIN) there, whose
// result its compiler decides; that case cannot be checked against the reference binary.
__device__ __forceinline__ int quant_i8_sat(float x, float mult) {
    const int i = __float2int_rz(__fmul_rn(x, mult));
    return i > 127 ? 127 : i < -127 ? -127 : i;
}

// One f32 value in side format F: the s8 byte (mult: the layer's input multiplier), the +-1 byte or the sign bit, in the low
// bits of the result.  The sign is x > 0 (binarize_cpu, float_to_bit): NaN, -inf and -FLT_MAX give -1 / 0 alike.  SIDE_PM1Z_S8
// takes x >= 0 instead (binarize_kernel of the GPU build, gpu.cu:813-818): +0 and -0 give +1, NaN gives -1.
template <SideFmt F>
__device__ __forceinline__ uint32_t side_code(float x, float mult) {
    static_assert(side_int(F), "integer side formats only");
    if constexpr (F == SIDE_S8) return (uint32_t)quant_i8(x, mult) & 0xffu;
    else if constexpr (F == SIDE_S8_SAT) return (uint32_t)quant_i8_sat(x, mult) & 0xffu;
    else if constexpr (F == SIDE_PM1_S8) return x > 0.f ? 0x01u : 0xFFu;
    else if constexpr (F == SIDE_PM1Z_S8) return x >= 0.f ? 0x01u : 0xFFu;
    else return x > 0.f ? 1u : 0u;
}

// code of channel j (0 <= j < side_per_word(F)) at its place in the word: byte j or bit j
template <SideFmt F>
__device__ __forceinline__ uint32_t side_place(uint32_t code, int j) { return code << (F == SIDE_BITS ? j : 8 * j); }

// the word of channels v[0 .. N) in side format F (N <= side_per_word(F))
template <SideFmt F, int N = side_per_word(F)>
__device__ __forceinline__ uint32_t side_word(const float *v, float mult) {
    uint32_t w = 0;
#pragma unroll
    for (int j = 0; j < N; ++j) w |= side_place<F>(side_code<F>(v[j], mult), j);
    return w;
}

// 16 channels v[0 .. 16) in an s8 side format: four words, one 16-byte store
template <SideFmt F>
__device__ __forceinline__ uint4 side_word4(const float *v, float mult) {
    return make_uint4(side_word<F>(v, mult), side_word<F>(v + 4, mult), side_word<F>(v + 8, mult), side_word<F>(v + 12, mult));
}

// the 32-bit words of pixel (n, y, x) of a side tensor (s8 formats: ldc in bytes, a multiple of 4; sign bits: ldc in words)
template <SideFmt F>
__device__ __forceinline__ uint32_t *side_px(const TV &q, int n, int y, int x) {
    if constexpr (F == SIDE_BITS) return tv_px<uint32_t>(q, n, y, x);
    else return reinterpret_cast<uint32_t *>(tv_px<int8_t>(q, n, y, x));
}

// XNOR epilogue, dot = 2*count - K: act((float)dot * mean + bias) in the reference's float operation order -- one multiply,
// one add, no FMA contraction (additionally.c:1531, yolov2_forward_network.c:243-261).
__device__ __forceinline__ float xnor_epilogue(int dot, float mean, float bias, int act) {
    return act_exact(__fadd_rn(__fmul_rn((float)dot, mean), bias), act);
}

// INT8 requantising epilogue (yolov2_forward_network_quantized.c:474-490, :598-627): q16 = clamp(+-32767, acc / 32) [C truncating
// division]; y = (float)q16 * alpha1; y += bias; leaky: y > 0 ? y : y / 10.
__device__ __forceinline__ float int8_epilogue(int acc, float alpha1, float bias, int act) {
    int q = acc / 32;
    if (q > 32767) q = 32767;
    if (q < -32767) q = -32767;
    float y = __fmul_rn((float)q, alpha1);
    y = __fadd_rn(y, bias);
    if (act == ACT_LEAKY) y = (y > 0.f) ? y : __fdiv_rn(y, 10.f);
    return y;
}

// INT8 epilogue of the GPU rule (forward_convolutional_layer_gpu_cudnn_quantized, yolov2_forward_network_gpu.cu:184-229, :314):
// y = act((float)acc * alpha1 + bias), alpha1 = 1 / (input_mult * weights_mult) -- no /32, no int16 clamp.  One rounded multiply,
// one rounded add, then act_exact, the operation order of int8_epilogue and the activation of every other f32 layer.  cuDNN's
// fused convolution-bias-activation may contract the multiply and the add (one rounding less); that cannot be checked here.
// Monotone non-decreasing in acc for alpha1 > 0, as the fused max-pool needs.
__device__ __forceinline__ float int8_gpu_epilogue(int acc, float alpha1, float bias, int act) {
    return act_exact(__fadd_rn(__fmul_rn((float)acc, alpha1), bias), act);
}

// The activations of the GPU XNOR rule.  Leaky is the bit GEMM's fused `v >= 0 ? v : 0.1f*v` (gpu.cu:1983), a float product;
// it equals the activation kernel's `(x > 0) ? x : .1f*x` on every input, -0 included.  The others are act_exact: relu is the
// same expression as the reference's; logistic there is `1.f/(1.f+expf(-x))` in float, which may differ from act_exact's
// double-precision logistic in the last bit.
__device__ __forceinline__ float act_gpu(float x, int act) {
    if (act == ACT_LEAKY) return x >= 0.f ? x : __fmul_rn(0.1f, x);
    return act_exact(x, act);
}

// Epilogue of an XNOR layer with c % 32 == 0 under the GPU XNOR rule (gemm_nn_custom_bin_mean_transposed_tensor_kernel,
// gpu.cu:1974-1990), dot = 2*count - K: `(float)dot * mean + bias`, which nvcc contracts to one FFMA -- one rounding -- then
// the activation.  Monotone non-decreasing in dot for mean > 0, as the fused max-pool needs.
__device__ __forceinline__ float xnor_gpu_epilogue(int dot, float mean, float bias, int act) {
    return act_gpu(__fmaf_rn((float)dot, mean, bias), act);
}

// Epilogue of an XNOR layer with c < 32 under the GPU XNOR rule (yolov2_forward_network_gpu.cu:94-138): s = sum of
// sign(w) * b(x) with b(x) = x >= 0 ? +1 : -1 and out-of-image taps 0, the convolution of the +-mean weights as the exact
// integer s times mean, rounded once; then add_bias_gpu (a second rounding) and the activation.  cuDNN's own summation order
// is not reproduced: this is the correctly rounded convolution.
__device__ __forceinline__ float pm1z_gpu_epilogue(int s, float mean, float bias, int act) {
    return act_gpu(__fadd_rn(__fmul_rn((float)s, mean), bias), act);
}

// whether arithmetic a's epilogue scales by the filter's mean |w| (the XNOR arithmetics) rather than the layer's ALPHA1 (INT8)
__host__ __device__ constexpr bool arith_mean(Arith a) { return a == AR_XNOR || a == AR_XNOR_GPU || a == AR_PM1Z_GPU; }

// Integer arithmetic A as every integer kernel finishes it, from its signed integer result r: the s32 accumulator (INT8), dot =
// 2*count - K (XNOR) or the zero-padded +-1 sum (PM1Z).  The s8 wgmma computes r directly; the popcount kernels form it from
// their count as 2*(count - padbits) - K.
template <Arith A>
struct IntEpi {
    static_assert(A == AR_XNOR || A == AR_XNOR_GPU || A == AR_PM1Z_GPU || A == AR_INT8 || A == AR_INT8_GPU, "integer arithmetics only");
    static constexpr bool MEAN = arith_mean(A);   // scale: the filter's mean |w|, else the layer's ALPHA1
    static __device__ __forceinline__ float finish(int r, float scale, float bias, int act) {
        if constexpr (A == AR_XNOR) return xnor_epilogue(r, scale, bias, act);
        else if constexpr (A == AR_XNOR_GPU) return xnor_gpu_epilogue(r, scale, bias, act);
        else if constexpr (A == AR_PM1Z_GPU) return pm1z_gpu_epilogue(r, scale, bias, act);
        else if constexpr (A == AR_INT8) return int8_epilogue(r, scale, bias, act);
        else return int8_gpu_epilogue(r, scale, bias, act);
    }
    // the raw result keep_counts stores, K = size*size*C: the reference's popcount (r + K) / 2 for the two XNOR arithmetics
    static __device__ __forceinline__ int raw(int r, int K) { return A == AR_XNOR || A == AR_XNOR_GPU ? (r + K) / 2 : r; }
};

}  // namespace yb
