// yb_conv_tc.cu -- FP32-variant convolution (reference yolov2_forward_network.c:204-261, SURVEY 8a row a2) as a
// persistent, warp-specialised implicit GEMM on the Hopper (sm_90a) tensor cores:
//
//     D[pixel, filter] = sum_{tap, c} A[pixel + tap, c] * W[filter, (tap, c)]
//
//   * A (activations, bf16, padded NHWC) is never materialised as an im2col matrix: for every (tap, 64-channel)
//     K-block the TMA engine loads a [TH x TW pixels] x [BK channels] box straight out of the activation tensor,
//     shifted by the tap, into swizzled shared memory.  Out-of-image taps read the tensor's zero border
//     (or TMA's out-of-bounds zero fill at the ends of the batch), so there is no bounds logic anywhere.
//     Tiles are rectangles of TW x TH = 128 output pixels over (x, merged batch*row) so that the 19*2^k-wide
//     YOLO grids tile exactly.  Stride-2 convolutions use a 5-D view that splits x and y into (half, parity).
//   * W ([filters][K] bf16, K ordered (ky, kx, c)) is the K-major B operand, loaded by TMA as well.
//   * Two consumer warpgroups issue wgmma.mma_async (bf16 x bf16 -> f32, M=64 each, N=BN, K=16) straight from
//     the shared-memory ring; each releases a ring stage through an mbarrier once the wgmmas reading it have retired.
//   * bf16-output layers, stride 1 and 2 (all but the detection heads), run k_conv_tc_reg: BN <= 256, the epilogue works
//     on the register fragments, adds the shortcut residual when fused (reference :443-449), and stores bf16 slabs by
//     TMA (see there).
//   * Everything else runs k_conv_tc (BN <= 128): at the end of a tile the register accumulators go to a padded
//     [128][BN+4] shared-memory tile, and the same 8 warps run the epilogue from it with one pixel row per thread: add
//     bias (folded batch-norm), apply leaky-ReLU and store f32 for detection heads -- optionally with the following
//     [yolo] layer applied (:453-472).  The producer warp keeps loading the next tile's stages meanwhile.
//   * The same kernel runs the INT8 variant (s8 x s8 -> s32 wgmma, exact requantising epilogue,
//     yolov2_forward_network_quantized.c:474-490, or the GPU rule's unscaled one, yolov2_forward_network_gpu.cu:184-229),
//     wide XNOR layers as +-1 bytes on the s8 wgmma, and the float heads of the exact networks on tf32 wgmma.
//
// Warp roles of k_conv_tc (288 threads): warps 0-7 = two consumer warpgroups (wgmma + epilogue), warp 8 = TMA producer.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "yb_conv_tc.cuh"
#include "yb_cuda.h"

namespace yb {

namespace {

constexpr int TC_BM = 128;
constexpr int TC_EPI_WARPS = 8;              // two warpgroups; in the epilogue, two warps per 32-row quarter, each takes half of the columns
constexpr int TC_THREADS = 32 * TC_EPI_WARPS + 32;
constexpr int TC_PRODUCER_WARP = TC_EPI_WARPS;
constexpr int TC_ACC_BAR = 3;                // named barrier of the 256 consumer threads (1, 2: the TMA-epilogue groups)

// Where the regions of a plan's dynamic shared memory lie: byte offsets from the kernel's 1024-byte aligned base, placed by
// tc_smem_layout.  The resident filter matrix (bstat_bytes) starts at offset 0.
struct TcSmem {
    uint32_t ring;                  // operand ring: stages x stage_bytes
    uint32_t full, empty;           // mbarriers per ring stage: its K-blocks have landed / the consumers are done with them
    uint32_t bstat_bar;             // mbarrier: the resident filter matrix has landed
    uint32_t stg_full, stg_ready;   // k_conv_tc_reg's mbarriers per consumer warpgroup g: stg_full[g][slab], stg_ready[g]
    uint32_t bias;                  // f32 bias of all nt * BN filters
    uint32_t ymask;                 // k_conv_tc: fused [yolo] mask, one bit per filter
    uint32_t stg;                   // epilogue staging or TMA-epilogue tiles (stg_bytes)
    uint32_t acc;                   // k_conv_tc: [128][acc_pitch] 32-bit accumulator tile
};

struct TcParams {
    int N;                    // images
    int TW, TWlog2, TH;       // tile = TW x TH output pixels (TW*TH == 128)
    int xt, jt, nt;           // #tiles along x, merged rows, filters
    int num_work;             // tiles = work items of the persistent loop (xt * jt * nt)
    int kind;                 // TcKind: TC_BF16 bf16 x bf16 -> f32;  TC_S8 s8 x s8 -> s32, exact requantising epilogue;
                              // TC_S8_GPU the same GEMM, the GPU rule's unscaled epilogue;
                              // TC_XNOR XNOR layer as +-1 s8 on the s8 wgmma (dot = 2*count - K exactly), reference float epilogue;
                              // TC_XNOR_GPU the same GEMM, the GPU XNOR rule's bit-GEMM epilogue; TC_PM1Z_GPU zero-padded +-1
                              // s8 GEMM, the GPU XNOR rule's epilogue of the layers below 32 channels;
                              // TC_TF32 f32 operands read as tf32 (K = 8 per MMA) -> f32: float heads of the exact nets
    int kk;                   // MMAs per K-block (BK bytes / 32)
    float alpha1;             // INT8: R_MULT / (input_mult * weights_mult); TC_S8_GPU: 1 / (input_mult * weights_mult)
    const float *mean;        // the XNOR kinds (2, 5, 6): per-filter mean |w|
    int xK;                   // kinds 2 and 5: true K (size*size*C) for the raw popcount dump: count = (dot + K) / 2
    int *acc_out;             // INT8: optional raw s32 accumulators, NCHW (tests)
    float *yolo_out;          // fused [yolo] layer (reference yolov2_forward_network.c:453-472): NCHW f32 destination, or null
    int yolo_per;             // 4 + classes + 1
    int PR, row_off;          // merged-row pitch per image; output row = (J % PR) - row_off
    int OH, OW, OHp, OWp;
    int size, cblocks, kblocks;
    int BK, BN;
    int stride2;
    int xoff, yoff;
    int stages;
    uint32_t stage_bytes, a_bytes, b_bytes;   // per stage (all sub-blocks); per K-block A tile; per K-block B tile
    int bstat;                                // 1: the whole filter matrix (nt == 1, <= 72 KB) is loaded once per CTA and stays in
                                              //    shared memory; the ring then streams activations only
    uint32_t bstat_bytes;
    // TMA epilogue: slab width in columns (0: off).  Each epilogue group writes its slab into a swizzled shared-memory tile and
    // one thread stores it with cp.async.bulk.tensor; the shortcut residual comes in the same way (TMA load + mbarrier).
    // Non-zero for every k_conv_tc_reg plan (bf16 slabs) and for the stride-1 integer kinds without the raw-accumulator dump
    // (f32 slabs of k_conv_tc); the other k_conv_tc plans store through the per-warp LSU staging tiles.
    int tma_epi;
    uint32_t stg_bytes;       // epilogue staging / TMA-epilogue tiles
    int acc_pitch;            // words per row of the shared-memory accumulator tile (BN + 4: conflict-free row reads)
    // Fused 2x2 / stride-2 max-pool + input conversion of the NEXT integer layer (integer kinds, tiles of 8 x 16 pixels):
    // the epilogue reduces every 2x2 window inside the warp (lane ^ 1 = x neighbour, lane ^ 8 = y neighbour), converts it into
    // the next layer's side format pool_fmt (SIDE_S8 or SIDE_S8_SAT with pool_mult, or SIDE_PM1_S8) and writes bytes straight into that layer's
    // input: the f32 activation and the pooled f32 tensor never reach HBM.  pool_fmt SIDE_NONE: no fused max-pool.  jshift = 1 moves every tile down one merged row so
    // that window rows (oy even, oy + 1) fall into the same tile (the padded layout puts oy = 0 on an odd merged row).
    int pool_fmt, jshift;     // SideFmt
    float pool_mult;
    signed char *pool_out; long pool_ldc; int pool_Hp, pool_Wp;   // next layer's s8 input: padded NHWC, bytes
    int sps;                                  // K-blocks per pipeline stage (amortises the per-stage barrier round trip)
    TcSmem sm;
    uint32_t desc_hi;         // high word of the wgmma shared-memory descriptors (SBO, swizzle mode)
    char *out; long out_ldc; int n;
    const char *res;          // fused shortcut operand (bf16, k_conv_tc_reg at stride 1 only), or null
    const float *bias; int act, act2;
    unsigned long long *stats; // YB_TC_STATS=1: per-CTA cycle counters [grid][TC_NSTATS] (diagnostic)
    int dbg;                  // YB_TC_DBG bit mask for bottleneck experiments: 1 no TMA, 4 no epilogue memory ops
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\telect.sync rx|px, %1;\n\t@px mov.s32 %0, 1;\n\t}"
        : "+r"(pred) : "r"(0xffffffffu));
    return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok;
}
// Bounded wait: a protocol bug must surface as a trap (CUDA error), never as a hung GPU.  No printf here: a function
// call anywhere in the kernel makes ptxas serialize every wgmma (C7510), and the consumers wait between wgmma issues.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > 4000000000LL) __trap();   // ~2 s at 2 GHz
}

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *tm, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// L2 eviction hint for data that is dead after this kernel (the C/2 tensor a 3x3 layer reads, the shortcut operand): evict-first
// leaves the L2 to the output this kernel writes, which the next layer reads right away
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void tma_load_3d_hint(uint32_t dst, const CUtensorMap *tm, uint32_t bar, int c0, int c1, int c2, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *tm, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap *tm, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}

__device__ __forceinline__ void tma_store_3d(const CUtensorMap *tm, uint32_t src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(tm), "r"(src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *tm) { asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// Programmatic dependent launch: the prologue before this (barrier init, tensor-map prefetch, bias -> smem: weights only)
// overlapped the tail of the previous kernel; from here on the kernel touches activations it wrote.
__device__ __forceinline__ void pdl_wait_and_launch() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// --- wgmma (sm_90a) ----------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor: start address >> 4 (bits 0-13), LBO = 1 (unused by the swizzled K-major layouts), high word
// = SBO >> 4 | swizzle mode << 30 (1: 128B, 2: 64B, 3: 32B).  K advances inside a swizzle row by adding to the start address.
__device__ __forceinline__ uint64_t wg_desc(uint32_t addr, uint32_t hi) {
    return ((uint64_t)hi << 32) | (uint64_t)(((addr & 0x3FFFFu) >> 4) | (1u << 16));
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins the accumulator registers around a batch of wgmmas, so that the compiler moves no instruction touching them into the
// batch (it would otherwise have to fence every wgmma on its own)
template <typename T, int N>
__device__ __forceinline__ void wg_fence_operand(T (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
        if constexpr (std::is_same<T, float>::value) asm volatile("" : "+f"(d[i])::"memory");
        else asm volatile("" : "+r"(d[i])::"memory");
    }
}

// One M=64 x N x (32 bytes of K) wgmma per call; d: this thread's accumulator fragment (N/2 values).  scale_d == 0 overwrites.
// TC_BF16: bf16 -> f32, TC_S8 (every integer kind): s8 -> s32, TC_TF32: tf32 -> f32.
template <TcKind KIND, int N> struct Wg;
template <> struct Wg<TC_BF16, 32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_BF16, 64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_BF16, 128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_BF16, 256> {
    static __device__ __forceinline__ void mma(float (&d)[128], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_S8, 32> {
    static __device__ __forceinline__ void mma(uint32_t (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_S8, 64> {
    static __device__ __forceinline__ void mma(uint32_t (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_S8, 128> {
    static __device__ __forceinline__ void mma(uint32_t (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_TF32, 32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_TF32, 64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};
template <> struct Wg<TC_TF32, 128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(a), "l"(b), "r"(scale_d) : "memory");
    }
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}

// The shared-memory accumulator tile: 32 consecutive columns of one row (the epilogue's view, one pixel row per thread)
__device__ __forceinline__ void acc_ld32(uint32_t addr, uint32_t (&v)[32]) {
#pragma unroll
    for (int c = 0; c < 8; ++c)
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[4 * c]), "=r"(v[4 * c + 1]), "=r"(v[4 * c + 2]), "=r"(v[4 * c + 3])
                     : "r"(addr + 16u * (uint32_t)c) : "memory");
}
// wgmma accumulator fragment of one warpgroup (rows row0 .. row0 + 63) -> accumulator tile.  Thread (warp w, lane l) holds rows
// row0 + 16 w + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1).
template <typename T, int NR>
__device__ __forceinline__ void acc_store_frag(uint32_t acc, int pitch, int row0, const T (&d)[NR]) {
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int r = row0 + 16 * w + (lane >> 2), c = 2 * (lane & 3);
    const uint32_t a0 = acc + 4u * (uint32_t)(r * pitch + c), a1 = a0 + 4u * 8u * (uint32_t)pitch;
#pragma unroll
    for (int j = 0; j < NR / 4; ++j) {
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a0 + 32u * (uint32_t)j), "r"(*reinterpret_cast<const uint32_t *>(&d[4 * j])),
                     "r"(*reinterpret_cast<const uint32_t *>(&d[4 * j + 1])) : "memory");
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a1 + 32u * (uint32_t)j), "r"(*reinterpret_cast<const uint32_t *>(&d[4 * j + 2])),
                     "r"(*reinterpret_cast<const uint32_t *>(&d[4 * j + 3])) : "memory");
    }
}

// The aligned base of the dynamic shared memory: 128B swizzle atoms are 1024-byte aligned.  Every region lies at an offset
// from it (TcParams::sm).
__device__ __forceinline__ uint32_t smem_base(const void *smem_raw) { return (smem_u32(smem_raw) + 1023u) & ~1023u; }
__device__ __forceinline__ void *smem_ptr(uint32_t addr) { return __cvta_shared_to_generic(addr); }
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// --- The pipeline both kernels share: work items, the operand ring, the role counters ------------------------------------
// Work item w: filter tile w % nt (first filter n0) of pixel tile w / nt, whose first pixel is column x0 of merged row J0.  The
// producer, the consumers and k_conv_tc_reg's store threads walk the same items, w = blockIdx.x, + gridDim.x, ...
// BN: p.BN, or the same width as a compile-time constant.
struct TcItem { int n0, x0, J0; };
__device__ __forceinline__ TcItem tc_item(const TcParams &p, int w, int BN) {
    const int m = w / p.nt;
    return {(w % p.nt) * BN, (m % p.xt) * p.TW, (m / p.xt) * p.TH + p.jshift};
}
// The output pixel of accumulator row r of item t's tile.  A row that falls on a border or padding row of the merged-row
// tiling, past the batch or past the output's width is no output pixel (valid() is false).
struct TcPixel {
    int img, oy, ox;
    __device__ __forceinline__ bool valid(const TcParams &p) const { return img < p.N && oy >= 0 && oy < p.OH && ox < p.OW; }
};
__device__ __forceinline__ TcPixel tc_pixel(const TcParams &p, const TcItem &t, int r) {
    const int J = t.J0 + (r >> p.TWlog2);
    const int img = J / p.PR;
    return {img, J - img * p.PR - p.row_off, t.x0 + (r & (p.TW - 1))};
}

// Position in the operand ring: the stage and the parity of its barriers' current phase.  The producer and every consumer
// warp step through the stages in the same order.
struct TcRing {
    int stage = 0;
    uint32_t phase = 0;
    __device__ __forceinline__ void advance(int stages) { if (++stage == stages) { stage = 0; phase ^= 1u; } }
};
// The ring's barriers and the resident filter matrix's, by one thread before the block's first barrier: full[s] and bstat_bar
// complete on the producer's arrive.expect_tx and the bytes of its loads; empty[s] on one arrival per consumer warp
// (tc_mma_loop's release).
__device__ __forceinline__ void tc_init_ring(const TcParams &p, uint32_t base) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(base + p.sm.full + 8u * s, 1); mbar_init(base + p.sm.empty + 8u * s, TC_EPI_WARPS); }
    mbar_init(base + p.sm.bstat_bar, 1);
}

// Runs f(BN, KK) with the plan's filter-tile width and wgmmas per K-block as std::integral_constants.  BN_MAX: the kernel's
// widest filter tile.
template <int BN_MAX, typename F>
__device__ __forceinline__ void tc_dispatch(const TcParams &p, F &&f) {
    auto by_kk = [&](auto bn_c) {
        if (p.kk == 4) f(bn_c, std::integral_constant<int, 4>{});
        else if (p.kk == 2) f(bn_c, std::integral_constant<int, 2>{});
        else f(bn_c, std::integral_constant<int, 1>{});
    };
    if constexpr (BN_MAX == 256) {
        if (p.BN == 256) { by_kk(std::integral_constant<int, 256>{}); return; }
    }
    if (p.BN == 128) by_kk(std::integral_constant<int, 128>{});
    else if (p.BN == 64) by_kk(std::integral_constant<int, 64>{});
    else by_kk(std::integral_constant<int, 32>{});
}

// Role counters of the ST instantiations (YB_TC_STATS=1): cycles of one CTA, p.stats[blockIdx.x * TC_NSTATS + slot].  The
// consumer slots are warp 0's, the store slots the store thread's of consumer warpgroup 0.
enum TcStat {
    STAT_PROD_WAIT_EMPTY,    // producer: waiting for free ring stages
    STAT_PROD_TMA_ISSUE,     // producer: issuing TMA loads
    STAT_PROD_TOTAL,         // producer: all of its work items
    STAT_CONS_WAIT_FULL,     // consumer: waiting for loaded ring stages
    STAT_CONS_WAIT_READY,    // k_conv_tc_reg consumer: waiting on stg_ready, the first work item apart
    STAT_CONS_FIRST_READY,   // k_conv_tc_reg consumer: waiting on stg_ready before the first work item's epilogue
    STAT_CONS_TOTAL,         // consumer: all of its work items
    STAT_STORE_WAIT_FULL,    // k_conv_tc_reg store thread: waiting on stg_full
    STAT_STORE_WAIT_READ,    // k_conv_tc_reg store thread: waiting for its bulk stores to read shared memory
    TC_NSTATS = 16           // slots per CTA, padded to a power of two: with a multiply in its index, k_conv_tc_reg<true> spills more
};
__device__ __forceinline__ unsigned long long &tc_stat(const TcParams &p, TcStat s) { return p.stats[blockIdx.x * TC_NSTATS + s]; }
// Runs f(); the ST instantiations add the cycles it took to cycles, the others read no clock
template <bool ST, typename F>
__device__ __forceinline__ void timed(long long &cycles, F &&f) {
    if constexpr (ST) { const long long c0 = clock64(); f(); cycles += clock64() - c0; }
    else f();
}

// TMA producer (one elected thread): walks the consumers' work items and keeps the ring full (base: the aligned shared memory)
template <bool ST>
__device__ __forceinline__ void tc_produce(const CUtensorMap *tmA, const CUtensorMap *tmB, const TcParams &p, uint32_t base,
                                           int w_first, int w_step) {
    TcRing ring;
    long long w_empty = 0, w_tma = 0; const long long t_begin = ST ? clock64() : 0;
    // loop-invariant parameters in registers; the (tap, channel-block) walk is incremental (no integer divisions per
    // K-block in this single thread)
    const int sps = p.sps, kblocks = p.kblocks, cblocks = p.cblocks, BK = p.BK, fsize = p.size, stages = p.stages;
    const int xoff = p.xoff, yoff = p.yoff, stride2 = p.stride2;
    const uint32_t a_bytes = p.a_bytes, b_bytes = p.b_bytes, stage_bytes = p.stage_bytes;
    const uint32_t b_off = (uint32_t)sps * a_bytes;
    const uint32_t smemB = base, smem0 = base + p.sm.ring, bstat_bar = base + p.sm.bstat_bar;
    const int bstat = p.bstat;
    if (bstat) {   // resident filter matrix: kblocks boxes of [BN filters][BK], once
        mbar_arrive_expect_tx(bstat_bar, p.bstat_bytes);
        for (int kb = 0; kb < kblocks; ++kb) tma_load_2d(smemB + (uint32_t)kb * b_bytes, tmB, bstat_bar, kb * BK, 0);
    }
    for (int w = w_first; w < p.num_work; w += w_step) {
        const TcItem it = tc_item(p, w, p.BN);
        // channel block, tap x/y, K column of the weight matrix
        int cb = 0, ky = 0, kx = 0, kcol = 0;
        for (int kb0 = 0; kb0 < kblocks; kb0 += sps) {
            const int nsub = min(sps, kblocks - kb0);
            timed<ST>(w_empty, [&] { mbar_wait(base + p.sm.empty + 8u * (uint32_t)ring.stage, ring.phase ^ 1u); });
            const uint32_t fb = base + p.sm.full + 8u * (uint32_t)ring.stage;
            const uint32_t a_dst = smem0 + (uint32_t)ring.stage * stage_bytes;
            const uint32_t b_dst = a_dst + b_off;
            if (p.dbg & 1) {
                mbar_arrive(fb);
                ring.advance(stages);
                continue;
            }
            mbar_arrive_expect_tx(fb, (uint32_t)nsub * (a_bytes + (bstat ? 0u : b_bytes)));
            timed<ST>(w_tma, [&] {
                for (int j = 0; j < nsub; ++j) {
                    const uint32_t ad = a_dst + (uint32_t)j * a_bytes, bd = b_dst + (uint32_t)j * b_bytes;
                    const int c0 = cb * BK;
                    if (stride2) tma_load_5d(ad, tmA, fb, c0, kx & 1, it.x0 + (kx >> 1), ky & 1, it.J0 + (ky >> 1));
                    else tma_load_3d(ad, tmA, fb, c0, it.x0 + kx + xoff, it.J0 + ky + yoff);
                    if (!bstat) tma_load_2d(bd, tmB, fb, kcol, it.n0);
                    kcol += BK;
                    if (++cb == cblocks) { cb = 0; if (++kx == fsize) { kx = 0; ++ky; } }
                }
            });
            ring.advance(stages);
        }
    }
    if (ST && p.stats) {
        tc_stat(p, STAT_PROD_WAIT_EMPTY) = w_empty; tc_stat(p, STAT_PROD_TMA_ISSUE) = w_tma;
        tc_stat(p, STAT_PROD_TOTAL) = clock64() - t_begin;
    }
}

// The K-blocks of the current work item into warpgroup wg's accumulator fragment d (rows 64 wg .. + 63
// of the tile; KK wgmmas of K = 32 bytes per K-block).  A ring stage is released once the wgmmas that read it have retired,
// one stage behind the issue (wgmma.wait_group 1) so that the tensor pipe never drains.  Nothing but wgmmas touches the
// accumulators while wgmmas are in flight, and every batch is the same KK wgmmas: ptxas then inserts no fences of its own
// and serializes nothing (the -Xptxas -v log has no C75xx notes).
template <TcKind KIND, int BN, int KK, bool ST, typename T>
__device__ __forceinline__ void tc_mma_loop(T (&d)[BN / 2], const TcParams &p, uint32_t base, int wg, int lane, TcRing &ring,
                                            long long &w_full) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] = T(0);
    wg_fence_operand(d);
    const int sps = p.sps, stages = p.stages, kblocks = p.kblocks;
    const uint32_t a_bytes = p.a_bytes, b_bytes = p.b_bytes, stage_bytes = p.stage_bytes, hi = p.desc_hi;
    const uint32_t b_off = (uint32_t)sps * a_bytes, a_wg = (uint32_t)wg * (a_bytes >> 1);
    const uint32_t smemB = base, smem0 = base + p.sm.ring;   // resident filter matrix, ring
    const uint32_t full = base + p.sm.full, empty = base + p.sm.empty;   // the ring's mbarriers, 8 bytes per stage
    // one arrival per consumer warp (tc_init_ring)
    auto release = [&](int s) { __syncwarp(); if (lane == 0) mbar_arrive(empty + 8u * (uint32_t)s); };
    // one commit group per K-block; a stage (sps K-blocks, fewer at the end of the work item) is released once the group of
    // its last K-block has retired, which wgmma.wait_group 1 shows one K-block later
    int pend = -1, jj = 0;
    for (int kb = 0; kb < kblocks; ++kb) {
        if (jj == 0) timed<ST>(w_full, [&] { mbar_wait(full + 8u * (uint32_t)ring.stage, ring.phase); });
        const uint32_t st_base = smem0 + (uint32_t)ring.stage * stage_bytes;
        const uint32_t a_kb = st_base + a_wg + (uint32_t)jj * a_bytes;
        const uint32_t b_kb = p.bstat ? smemB + (uint32_t)kb * b_bytes : st_base + b_off + (uint32_t)jj * b_bytes;
        wg_fence();
#pragma unroll
        for (int k = 0; k < KK; ++k)
            Wg<KIND, BN>::mma(d, wg_desc(a_kb + 32u * (uint32_t)k, hi), wg_desc(b_kb + 32u * (uint32_t)k, hi),
                              (kb > 0 || k > 0) ? 1u : 0u);
        wg_commit();
        wg_wait<1>();
        if (pend >= 0) { release(pend); pend = -1; }
        if (++jj == sps || kb + 1 == kblocks) {
            pend = ring.stage; jj = 0;
            ring.advance(stages);
        }
    }
    wg_wait<0>();
    wg_fence_operand(d);
    if (pend >= 0) release(pend);
}

// The reference's float epilogue of integer arithmetic A (bit-exact) on the s8 wgmma's accumulator, which is A's signed result
// (IntEpi).  f: filter index (the XNOR arithmetics read its mean |w|).
template <Arith A>
__device__ __forceinline__ float int_epilogue(const TcParams &p, int acc, int f, float bias) {
    return IntEpi<A>::finish(acc, IntEpi<A>::MEAN ? ((f < p.n) ? __ldg(p.mean + f) : 0.f) : p.alpha1, bias, p.act);
}

// One CTA per 128-pixel x BN-filter tile, persistent over the tiles (grid <= #SMs, one CTA per SM).
// ST: compiled with the per-role cycle counters of YB_TC_STATS=1 (diagnostic); the production instantiations (ST = false)
// contain no clock64() reads.
// EPI: which epilogue family is compiled in -- 0: LSU stores, float kinds (f32 heads / fused [yolo]); 2: the integer
// kinds (s8 requantising, s8 unscaled and XNOR-as-+-1 epilogues).  The bf16-output layers run k_conv_tc_reg.
// tmO1, tmR: unused (the parameter list of k_conv_tc_reg, so that a plan launches either kernel the same way).
template <bool ST, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv_tc(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
          const __grid_constant__ CUtensorMap tmO1, const __grid_constant__ CUtensorMap tmR, const TcParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = smem_base(smem_raw);

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int w_first = (int)blockIdx.x, w_step = (int)gridDim.x;

    if (warp == TC_PRODUCER_WARP && elect_one()) {
        prefetch_tmap(&tmA);
        prefetch_tmap(&tmB);
        tc_init_ring(p, base);
        if (p.tma_epi) prefetch_tmap(&tmO);
        fence_mbar_init();
    }
    // bias (folded batch-norm) for all filter tiles -> shared memory, once per CTA
    const float *bias_s = reinterpret_cast<const float *>(smem_ptr(base + p.sm.bias));
    // fused [yolo]: one bit per filter, set where the entry is a box width/height (no logistic)
    const uint32_t *ymask_s = reinterpret_cast<const uint32_t *>(smem_ptr(base + p.sm.ymask));
    // 4 KB of staging per epilogue warp (32 rows x 128 B, XOR-swizzled) for the coalescing transposes, or the TMA-epilogue tiles
    const uint32_t stg_base = base + p.sm.stg;
    const uint32_t acc_base = base + p.sm.acc;               // [128 rows][acc_pitch] 32-bit accumulators of the current tile
    // (filled through shared-window addresses: EPI 2 spills more when the generic pointers are live from here on)
    for (int i = threadIdx.x; i < p.nt * p.BN; i += TC_THREADS)
        st_shared_u32(base + p.sm.bias + 4u * (uint32_t)i, __float_as_uint((i < p.n) ? __ldg(p.bias + i) : 0.f));
    if (p.yolo_out) {
        for (int wd = threadIdx.x; wd < p.nt * p.BN / 32; wd += TC_THREADS) {
            uint32_t m = 0;
            for (int j = 0; j < 32; ++j) { const int e = (wd * 32 + j) % p.yolo_per; if (e == 2 || e == 3) m |= 1u << j; }
            st_shared_u32(base + p.sm.ymask + 4u * (uint32_t)wd, m);
        }
    }
    __syncthreads();
    pdl_wait_and_launch();

    if (warp == TC_PRODUCER_WARP) {
        // ======================= TMA producer =======================
        if (elect_one()) tc_produce<ST>(&tmA, &tmB, p, base, w_first, w_step);
    } else {
        // ======================= consumers (warps 0..7): wgmma main loop, then the epilogue of the same tile =======================
        const int ew = warp;                      // consumer warp; warpgroup ew >> 2 computes accumulator rows 64 * (ew >> 2) .. + 63
        const int wg = ew >> 2;
        TcRing ring;
        long long w_full = 0;
        if (p.bstat) mbar_wait(base + p.sm.bstat_bar, 0);
        // The K-blocks of the current work item into this warpgroup's registers, then both warpgroups' accumulators into the
        // shared-memory tile.
        auto mainloop = [&](auto kind_c) {
            tc_dispatch<128>(p, [&](auto bn_c, auto kk_c) {
                constexpr TcKind KIND = decltype(kind_c)::value;
                constexpr int BN = decltype(bn_c)::value;
                constexpr int KK = decltype(kk_c)::value;   // wgmmas per K-block
                using T = typename std::conditional<KIND == TC_S8, uint32_t, float>::type;
                T d[BN / 2];
                tc_mma_loop<KIND, BN, KK, ST>(d, p, base, wg, lane, ring, w_full);
                named_bar_sync(TC_ACC_BAR, 32 * TC_EPI_WARPS);   // every warp is done with the previous tile's accumulators
                acc_store_frag(acc_base, p.acc_pitch, wg * 64, d);
                named_bar_sync(TC_ACC_BAR, 32 * TC_EPI_WARPS);   // the whole 128 x BN tile is in place
            });
        };
        auto run_mainloop = [&]() {
            // EPI 2: TC_S8_GPU and the XNOR kinds run the same s8 wgmma as TC_S8
            if constexpr (EPI == 2) mainloop(std::integral_constant<TcKind, TC_S8>{});
            else if (p.kind == TC_BF16) mainloop(std::integral_constant<TcKind, TC_BF16>{});
            else mainloop(std::integral_constant<TcKind, TC_TF32>{});
        };

        // Epilogue.  Per slab: read the accumulator row(s) and the residual first, then the math and the stores.
        const int q = ew & 3;                     // 32-row quarter of the accumulator tile this warp reads
        const int half = ew >> 2;                 // which half of the columns this warp owns
        const int cbeg = (p.BN >= 64) ? half * (p.BN >> 1) : 0;
        const int cend = (p.BN >= 64) ? cbeg + (p.BN >> 1) : (half == 0 ? p.BN : 0);
        const int r = q * 32 + lane;              // accumulator row == pixel within the tile
        const bool leaky = p.act == ACT_LEAKY;
        const uint32_t taddr = acc_base + 4u * (uint32_t)(r * p.acc_pitch);
        const long long t_begin = ST ? clock64() : 0;
        for (int w = w_first; w < p.num_work; w += w_step) {
            run_mainloop();
            const TcItem it = tc_item(p, w, p.BN);
            const TcPixel px = tc_pixel(p, it, r);
            const int n0 = it.n0, img = px.img, oy = px.oy, ox = px.ox;
            const bool valid = px.valid(p) && !(p.dbg & 4);
            const long pix = ((long)(img * p.OHp + oy + 1) * p.OWp + ox + 1);
            char *orow = p.out + pix * p.out_ldc * 4;
            const float *bs = bias_s + n0;

            // ---- f32 output (detection heads) of one 32-column slab, one row per thread
            auto finish_f32 = [&](const uint32_t (&v)[32], int f0) {
                if (!valid || (n0 + f0) >= p.n) return;
                float x[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    float a = __uint_as_float(v[j]) + bs[f0 + j];
                    x[j] = leaky ? fmaxf(a, 0.1f * a) : a;   // == a > 0 ? a : 0.1a
                }
                if (p.yolo_out) {
                    // detection head with the [yolo] layer fused: logistic on x, y, objectness and class entries (w, h stay
                    // raw), written straight into the NCHW tensor the reference decoder reads -- the f32 NHWC copy of the
                    // head and the separate yolo kernel disappear
                    const int c0 = n0 + f0;
                    const int nvalid = p.n - c0;                       // columns >= n are padding
                    const uint32_t raw = ymask_s[c0 >> 5];             // bit j: entry (c0 + j) % (4+classes+1) is w or h -> stays raw
                    float *dst = p.yolo_out + (((size_t)img * p.n + c0) * p.OH + oy) * (size_t)p.OW + ox;
                    const size_t plane = (size_t)p.OH * p.OW;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const float sg = __fdividef(1.f, 1.f + __expf(-x[j]));
                        const float v = ((raw >> j) & 1u) ? x[j] : sg;
                        if (j < nvalid) dst[(size_t)j * plane] = v;
                    }
                } else {
                    float4 *op = reinterpret_cast<float4 *>(orow + (size_t)(n0 + f0) * 4);
#pragma unroll
                    for (int g = 0; g < 8; ++g) {
                        const int left = p.n - (n0 + f0 + g * 4);   // the output may be a channel slice: nothing past filter n
                        if (left <= 0) break;
                        if (left >= 4) op[g] = make_float4(x[g * 4 + 0], x[g * 4 + 1], x[g * 4 + 2], x[g * 4 + 3]);
                        else {   // bounded and unrolled: a runtime index into x would put it in local memory
#pragma unroll
                            for (int e = 0; e < 3; ++e)
                                if (e < left) reinterpret_cast<float *>(op + g)[e] = x[g * 4 + e];
                        }
                    }
                }
            };

            // ---- coalesced f32 store of one 32-column slab (integer kinds at stride 2 or with the raw-accumulator dump): a row
            // is 128 B; the warp's 32 rows go through its private XOR-swizzled 4 KB staging tile so that every global store
            // instruction writes 4 rows x 128 contiguous bytes instead of 32 rows x 16 B (32 different lines per instruction:
            // what kept the early INT8 layers at 0.8 TB/s in round 1)
            auto store_f32_slab = [&](const float (&y)[32], int f0) {
                const uint32_t stg = stg_base + (uint32_t)ew * 4096u;
                const int srow = lane >> 3, schunk = lane & 7;
                const unsigned long long obase = (unsigned long long)(uintptr_t)orow;
                const int vflag = valid ? 1 : 0;
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(stg + (uint32_t)lane * 128u + (uint32_t)((c ^ (lane & 7)) << 4)),
                                 "r"(__float_as_uint(y[c * 4 + 0])), "r"(__float_as_uint(y[c * 4 + 1])),
                                 "r"(__float_as_uint(y[c * 4 + 2])), "r"(__float_as_uint(y[c * 4 + 3])) : "memory");
                __syncwarp();
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int row = i * 4 + srow;
                    const unsigned long long op = __shfl_sync(0xffffffffu, obase, row);
                    const int ok = __shfl_sync(0xffffffffu, vflag, row);
                    uint32_t w0, w1, w2, w3;
                    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3)
                                 : "r"(stg + (uint32_t)row * 128u + (uint32_t)((schunk ^ (row & 7)) << 4)) : "memory");
                    const int left = p.n - (n0 + f0 + schunk * 4);   // the output may be a channel slice: nothing past filter n
                    uint4 *dst = reinterpret_cast<uint4 *>(op + (size_t)(n0 + f0) * 4) + schunk;
                    if (ok && left >= 4) *dst = make_uint4(w0, w1, w2, w3);
                    else if (ok && left > 0) {
                        uint32_t *d1 = reinterpret_cast<uint32_t *>(dst);
                        d1[0] = w0;
                        if (left > 1) d1[1] = w1;
                        if (left > 2) d1[2] = w2;
                    }
                }
                __syncwarp();
            };

            // ---- fused 2x2/2 max-pool + conversion to the next integer layer's input (TcParams::pool_fmt).  All three epilogue
            // functions are monotone non-decreasing in the s32 accumulator (truncating /32, clamp, x positive ALPHA1, + bias, leaky;
            // the GPU rule's (float)acc x positive ALPHA1, + bias, leaky; resp. x mean >= 0, + bias, leaky), each step rounding
            // monotonically, so max over the window commutes with them EXACTLY: the window maximum is taken on the raw
            // accumulators and the float epilogue runs once per pooled value.  Window = lanes {l, l^1, l^8, l^9} (tile rows are 8
            // pixels wide).  The reduction is a reduce-scatter: lane^1 halves the 32 columns, lane^8 halves them again, every lane
            // ends up with the maxima of 8 columns of its window and finishes those -- a quarter of the float work per lane.
            // Elements outside the image count as "skipped" (INT_MIN) like the reference's out-of-range taps (additionally.c:1448-1482).
            auto pool_store_raw = [&](auto arith_c, const uint32_t (&v)[32], int f0) {
                constexpr Arith A = decltype(arith_c)::value;
                const bool b0 = lane & 1, b3 = lane & 8;
                int h16[16], h8[8];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int lo_ = valid ? (int)v[j] : INT_MIN, hi_ = valid ? (int)v[j + 16] : INT_MIN;
                    const int keep = b0 ? hi_ : lo_, send = b0 ? lo_ : hi_;
                    const int got = __shfl_xor_sync(0xffffffffu, send, 1);
                    h16[j] = max(keep, got);
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int keep = b3 ? h16[j + 8] : h16[j], send = b3 ? h16[j] : h16[j + 8];
                    const int got = __shfl_xor_sync(0xffffffffu, send, 8);
                    h8[j] = max(keep, got);
                }
                const int cbase = f0 + (b0 ? 16 : 0) + (b3 ? 8 : 0);     // this lane's 8 columns of the slab
                uint32_t w0 = 0, w1 = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int f = n0 + cbase + j;
                    const float t = int_epilogue<A>(p, h8[j], f, bs[cbase + j]);
                    uint32_t b8 = (p.pool_fmt == SIDE_S8) ? side_code<SIDE_S8>(t, p.pool_mult)
                                : (p.pool_fmt == SIDE_S8_SAT) ? side_code<SIDE_S8_SAT>(t, p.pool_mult) : side_code<SIDE_PM1_S8>(t, 0.f);
                    if (f >= p.n) b8 = 0;
                    if (j < 4) w0 |= side_place<SIDE_S8>(b8, j); else w1 |= side_place<SIDE_S8>(b8, j - 4);
                }
                const TcPixel o{img, oy & ~1, ox & ~1};                 // the window's origin: the same pooled pixel in all four lanes
                if (o.valid(p) && !(p.dbg & 4)) {
                    signed char *dst = p.pool_out + ((size_t)(img * p.pool_Hp + (o.oy >> 1) + 1) * p.pool_Wp + (o.ox >> 1) + 1) * (size_t)p.pool_ldc + n0 + cbase;
                    *reinterpret_cast<uint2 *>(dst) = make_uint2(w0, w1);
                }
            };

            // ---- TMA store of one 32-column f32 slab (integer kinds): the group's [128 pixels][32 floats] tile, 128-byte rows with
            // the 128B swizzle, written by one thread per row and stored by one cp.async.bulk.tensor
            auto tma_store_f32_slab = [&](const float (&y)[32], int f0) {
                const int g = half;
                const uint32_t out_tile = stg_base + (uint32_t)g * 16384u;
                const bool boss = (q == 0) && (lane == 0);
                const uint32_t rsw = (uint32_t)(r & 7), row_off = (uint32_t)r * 128u;
                if (boss) tma_store_wait_read0();   // the store that last used this tile has finished reading it
                named_bar_sync(1 + g, 128);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    uint32_t o0 = __float_as_uint(y[c * 4 + 0]), o1 = __float_as_uint(y[c * 4 + 1]);
                    uint32_t o2 = __float_as_uint(y[c * 4 + 2]), o3 = __float_as_uint(y[c * 4 + 3]);
                    if (!valid) { o0 = o1 = o2 = o3 = 0u; }           // border / padding rows inside the tensor stay zero
                    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(out_tile + row_off + (((uint32_t)c ^ rsw) << 4)),
                                 "r"(o0), "r"(o1), "r"(o2), "r"(o3) : "memory");
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                named_bar_sync(1 + g, 128);
                if (boss) {
                    const TcItem t = tc_item(p, w, p.BN);   // decoded again here: EPI 2 spills when `it` stays live
                    tma_store_3d(&tmO, out_tile, n0 + f0, t.x0 + 1, t.J0);
                    tma_store_commit();
                }
            };

            if constexpr (EPI == 2) {
                // ---- integer kinds: the exact float epilogue of the kind's arithmetic per 32-column slab (or the fused max-pool),
                // f32 stores
                auto int_slabs = [&](auto arith_c) {
                    constexpr Arith A = decltype(arith_c)::value;
                    for (int f0 = cbeg; f0 < cend; f0 += 32) {
                        uint32_t v0[32];
                        acc_ld32(taddr + 4u * (uint32_t)f0, v0);
                        if (p.pool_fmt != SIDE_NONE) { pool_store_raw(arith_c, v0, f0); continue; }
                        float y[32];
#pragma unroll
                        for (int j = 0; j < 32; ++j) y[j] = int_epilogue<A>(p, (int)v0[j], n0 + f0 + j, bs[f0 + j]);
                        if (p.tma_epi) tma_store_f32_slab(y, f0);
                        else store_f32_slab(y, f0);
                        if (!valid || !p.acc_out) continue;
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int f = n0 + f0 + j;
                            if (f < p.n) p.acc_out[(((size_t)img * p.n + f) * p.OH + oy) * p.OW + ox] = IntEpi<A>::raw((int)v0[j], p.xK);
                        }
                    }
                };
                if (p.kind == TC_XNOR) int_slabs(std::integral_constant<Arith, AR_XNOR>{});
                else if (p.kind == TC_S8_GPU) int_slabs(std::integral_constant<Arith, AR_INT8_GPU>{});
                else if (p.kind == TC_XNOR_GPU) int_slabs(std::integral_constant<Arith, AR_XNOR_GPU>{});
                else if (p.kind == TC_PM1Z_GPU) int_slabs(std::integral_constant<Arith, AR_PM1Z_GPU>{});
                else int_slabs(std::integral_constant<Arith, AR_INT8>{});
            } else {
                for (int f0 = cbeg; f0 < cend; f0 += 64) {
                    if (cend - f0 >= 64) {
                        uint32_t v0[32], v1[32];
                        acc_ld32(taddr + 4u * (uint32_t)f0, v0);
                        acc_ld32(taddr + 4u * (uint32_t)f0 + 128u, v1);
                        finish_f32(v0, f0);
                        finish_f32(v1, f0 + 32);
                    } else {
                        uint32_t v0[32];
                        acc_ld32(taddr + 4u * (uint32_t)f0, v0);
                        finish_f32(v0, f0);
                    }
                }
            }
        }
        if (EPI == 2 && p.tma_epi && q == 0 && lane == 0) tma_store_wait_all();   // this group's bulk stores have completed
        if (ST && p.stats && ew == 0 && lane == 0) { tc_stat(p, STAT_CONS_WAIT_FULL) = w_full; tc_stat(p, STAT_CONS_TOTAL) = clock64() - t_begin; }
    }
}

// Register-accumulator kernel of the bf16-output layers, stride 1 and 2 (384 threads).  Warpgroups 0 and 1 are consumers with up to 216
// registers each: a consumer warpgroup keeps the f32 accumulators of its 64 rows x BN (<= 256) filters of the tile in registers
// and runs the epilogue straight on its wgmma fragment -- bias, leaky, the fused shortcut residual and the second leaky in fp32,
// then round to bf16.  Warpgroup 2 gives its registers away with setmaxnreg: warp 8 is the TMA producer, warps 9 and 10 are the
// store warps of consumer warpgroups 0 and 1 (one elected thread each).
//
// Each consumer warpgroup has one staging buffer: its half tile, 64 pixel rows x BN bf16, laid out as BN / SW slabs of SW columns
// (SW = 64, or 32 when BN == 32) with the tensor maps' swizzle.  The epilogue reads each residual word from it and writes the
// output word to the same address (the same thread owns both).  The store thread stores each slab with cp.async.bulk.tensor as
// soon as the consumers have written it, and once that store has read the slab it loads the next work item's residual slab into
// it (L2 evict-first).  So the epilogue's memory traffic runs while the consumers finish the epilogue, when the operand ring is
// full and the TMA engine would otherwise idle (issued under the next main loop instead, it held up the operand loads), and the
// residual has a whole main loop to land.  The mbarriers per consumer warpgroup g:
//   stg_full[g][s] -- 4 arrivals, one per consumer warp after fence.proxy.async: slab s is written;
//   stg_ready[g]   -- the store thread's arrival (expect_tx = the residual bytes): the buffer is free and holds the residual.
// A consumer goes from its epilogue straight into the next main loop: no named barrier and no TMA call in the consumers, and the
// two warpgroups never wait for each other.
//
// Stride 2: tile row J (a merged half row of the input, J = image * (OH + 1) + oy) goes to output merged padded row J + image + 1,
// which is affine only within one image.  A half tile inside one image is stored as one box; its rows with oy == OH (not an output
// row) land on that image's bottom border, and the epilogue writes them as zeros.  A half tile that straddles two images goes out
// one tile row at a time through tmO1 (box: SW channels x TW pixels x 1 row), skipping the rows with oy == OH and those past the
// batch: no store touches an image's top border or needs a negative row (bulk tensor stores fault on negative coordinates).
// Tile row t of a slab starts at byte t * TW * 2 SW.  Bulk tensor copies need 128-byte aligned shared memory (plan_tiles
// keeps TW * SW >= 64), and the TMA engine takes the swizzle phase from the shared-memory address (16-byte chunk c of the
// 128-byte row at address a is chunk c ^ ((a >> 7) & 7) at 128B, c ^ ((a >> 7) & 3) at 64B), the rule slab_off follows from
// the 1024-byte aligned buffer: a row box that starts off the swizzle's 1024 / 512-byte repeat reads its rows as written.
// Stride-2 plans have no fused residual.
constexpr int TCR_THREADS = 384;
constexpr int TCR_PRODUCER_REGS = 40, TCR_CONSUMER_REGS = 216;   // 128 * 40 + 256 * 216 <= 64 K registers
constexpr int TCR_STORE_WARP = 9;                                // store warps 9 (consumer warpgroup 0) and 10 (warpgroup 1)
constexpr int TCR_MAX_SLABS = 4;                                 // BN / SW <= 256 / 64

// Store thread of consumer warpgroup g: walks the consumers' work items (see k_conv_tc_reg).  buf: the warpgroup's staging buffer,
// stg_full: its first per-slab barrier.  ST: cycles spent waiting on stg_full and in cp.async.bulk.wait_group.read go to
// STAT_STORE_WAIT_FULL and STAT_STORE_WAIT_READ (warpgroup 0's thread).
template <bool ST>
__device__ __forceinline__ void tcr_store(const CUtensorMap *tmO, const CUtensorMap *tmO1, const CUtensorMap *tmR, const TcParams &p,
                                          uint32_t buf, uint32_t stg_full, uint32_t stg_ready, int g, int w_first, int w_step) {
    const int SW = p.tma_epi, BN = p.BN;
    const uint32_t tile = 64u * 2u * (uint32_t)SW;                  // one slab: 64 pixel rows x SW bf16
    // the half tile as a TMA box: 64 of the TW x TH pixels (TW == 128: one half row; else TH / 2 whole rows)
    const int hx = (p.TW == 128) ? 64 * g : 0, hy = (p.TW == 128) ? 0 : g * (p.TH >> 1);
    long long w_full = 0, w_read = 0;
    // box origin of work item w's half tile (first filter, padded x, merged padded output row); returns its slabs holding
    // filters < n.  Stride 1: tile rows are the output's padded rows.  Stride 2: y = J0 + image + 1 for a half tile inside one
    // image (rows past the batch fall outside the tensor), y = -1 - J0 for one that straddles two images (stored row by row;
    // J0: merged row of its first tile row).
    auto item = [&](int w, int &n0, int &x, int &y) {
        const TcItem it = tc_item(p, w, BN);
        n0 = it.n0; x = it.x0 + 1 + hx; y = it.J0 + hy;
        if (p.stride2) {
            const int i0 = y / p.PR, i1 = min((y + max(p.TH >> 1, 1) - 1) / p.PR, p.N - 1);
            y = i0 == i1 ? y + i0 + 1 : -1 - y;
        }
        return (min(BN, p.n - n0) + SW - 1) / SW;
    };
    auto store_slab = [&](uint32_t src, int c, int x, int y) {
        if (y >= 0) { tma_store_3d(tmO, src, c, x, y); return; }
        const int J0 = -1 - y;
        int img = J0 / p.PR, oy = J0 - img * p.PR;
        for (int t = 0; t < (p.TH >> 1); ++t) {   // TW <= 32 here: the half tile is TH / 2 rows of TW pixels
            if (img < p.N && oy < p.OH) tma_store_3d(tmO1, src, c, x, J0 + t + img + 1);
            if (++oy == p.PR) { oy = 0; ++img; }
            src += (uint32_t)(p.TW * 2 * SW);
        }
    };
    auto wait_read = [&]() { timed<ST>(w_read, tma_store_wait_read0); };   // the bulk stores issued so far have read shared memory
    auto load_res = [&](int s, int n0, int x, int y) {
        tma_load_3d_hint(buf + (uint32_t)s * tile, tmR, stg_ready, n0 + s * SW, x, y, l2_policy_evict_first());
    };
    if (w_first < p.num_work) {   // the first item's residual overlaps the first main loop
        if (p.res) {
            int n0, x, y;
            const int ns = item(w_first, n0, x, y);
            mbar_arrive_expect_tx(stg_ready, (uint32_t)ns * tile);
            for (int s = 0; s < ns; ++s) load_res(s, n0, x, y);
        } else mbar_arrive(stg_ready);
    }
    // Per item: store each slab as soon as the consumers have written it, and once that store has read the slab, load the
    // next item's residual slab into it -- all of it while the consumers are still in the epilogue, when the operand ring is
    // full and the TMA engine would otherwise idle.
    uint32_t phases = 0;   // bit s: phase parity of slab s's stg_full (masked filter tiles skip the slabs >= their ns)
    for (int w = w_first; w < p.num_work; w += w_step) {
        int n0, x, y, n0n = 0, xn = 0, yn = 0;
        const int ns = item(w, n0, x, y);
        const bool next = w + w_step < p.num_work, res_next = next && p.res;
        const int nsn = next ? item(w + w_step, n0n, xn, yn) : 0;
        for (int s = 0; s < ns; ++s) {
            const uint32_t fb = stg_full + 8u * (uint32_t)s;
            timed<ST>(w_full, [&] { mbar_wait(fb, (phases >> s) & 1u); });
            phases ^= 1u << s;
            // the consumers are past this item's stg_ready: its phase is complete and the next item's may begin
            if (s == 0 && res_next) mbar_arrive_expect_tx(stg_ready, (uint32_t)nsn * tile);
            store_slab(buf + (uint32_t)s * tile, n0 + s * SW, x, y);
            tma_store_commit();
            if (res_next && s < nsn) { wait_read(); load_res(s, n0n, xn, yn); }
        }
        if (res_next) {
            for (int s = ns; s < nsn; ++s) { wait_read(); load_res(s, n0n, xn, yn); }
        } else if (next) {
            wait_read();
            mbar_arrive(stg_ready);
        }
    }
    tma_store_wait_all();   // bulk groups are per thread: these are this warpgroup's stores only
    if (ST && p.stats && g == 0) { tc_stat(p, STAT_STORE_WAIT_FULL) = w_full; tc_stat(p, STAT_STORE_WAIT_READ) = w_read; }
}

template <bool ST>
__global__ void __launch_bounds__(TCR_THREADS, 1)
k_conv_tc_reg(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
              const __grid_constant__ CUtensorMap tmO1, const __grid_constant__ CUtensorMap tmR, const TcParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = smem_base(smem_raw);
    // per consumer warpgroup g: stg_full for each of up to TCR_MAX_SLABS slabs, and stg_ready
    auto stg_full = [&](int g, int s) { return base + p.sm.stg_full + 8u * (uint32_t)(g * TCR_MAX_SLABS + s); };
    auto stg_ready = [&](int g) { return base + p.sm.stg_ready + 8u * (uint32_t)g; };
    float *bias_s = reinterpret_cast<float *>(smem_ptr(base + p.sm.bias));
    // staging buffers of warpgroups 0 and 1, 64 * BN bf16 each
    const uint32_t stg_base = base + p.sm.stg;

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int w_first = (int)blockIdx.x, w_step = (int)gridDim.x;
    const bool epi_mem = !(p.dbg & 4);

    if (warp == TC_PRODUCER_WARP && elect_one()) {
        prefetch_tmap(&tmA);
        prefetch_tmap(&tmB);
        prefetch_tmap(&tmO);
        if (p.stride2) prefetch_tmap(&tmO1);
        if (p.res) prefetch_tmap(&tmR);
        tc_init_ring(p, base);
        for (int g = 0; g < 2; ++g) {
            for (int s = 0; s < TCR_MAX_SLABS; ++s) mbar_init(stg_full(g, s), 4);
            mbar_init(stg_ready(g), 1);
        }
        fence_mbar_init();
    }
    for (int i = threadIdx.x; i < p.nt * p.BN; i += TCR_THREADS) bias_s[i] = (i < p.n) ? __ldg(p.bias + i) : 0.f;
    __syncthreads();
    pdl_wait_and_launch();

    if (wg == 2) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TCR_PRODUCER_REGS));
        if (warp == TC_PRODUCER_WARP) {
            if (elect_one()) tc_produce<ST>(&tmA, &tmB, p, base, w_first, w_step);
        } else if (warp < TCR_STORE_WARP + 2 && epi_mem) {
            const int g = warp - TCR_STORE_WARP;
            if (elect_one()) tcr_store<ST>(&tmO, &tmO1, &tmR, p, stg_base + (uint32_t)g * 128u * (uint32_t)p.BN, stg_full(g, 0), stg_ready(g), g, w_first, w_step);
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TCR_CONSUMER_REGS));

    // ======================= consumers: warpgroup wg owns rows 64 wg .. + 63 of every tile =======================
    // wgmma fragment: this thread holds rows rl and rl + 8 (of the warpgroup's 64), columns 8 j + cq, 8 j + cq + 1
    const int rl = 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
    const bool leaky = p.act == ACT_LEAKY, leaky2 = p.act2 == ACT_LEAKY;
    const bool has_res = p.res != nullptr;
    TcRing ring;
    uint32_t stg_phase = 0;
    // w_ready: waits on stg_ready after the first work item (the first item's, whose residual fetch overlaps only one main loop,
    // goes to STAT_CONS_FIRST_READY right away)
    long long w_full = 0, w_ready = 0; const long long t_begin = ST ? clock64() : 0;
    if (p.bstat) mbar_wait(base + p.sm.bstat_bar, 0);

    tc_dispatch<256>(p, [&](auto bn_c, auto kk_c) {
        constexpr int BN = decltype(bn_c)::value;
        constexpr int KK = decltype(kk_c)::value;
        constexpr int SW = BN >= 64 ? 64 : 32;             // slab width (columns); rows of 128 B (128B swizzle) or 64 B (64B swizzle)
        constexpr uint32_t ROWB = SW * 2, TILE = 64u * ROWB;
        const uint32_t buf = stg_base + (uint32_t)wg * (uint32_t)(BN / SW) * TILE;
        // byte offset of (row, 16-byte chunk c) in a slab + this thread's column pair: conflict-free for the fragment layout
        auto slab_off = [&](int row, int c) -> uint32_t {
            const int sw = (SW == 64) ? (row & 7) : ((row >> 1) & 3);
            return (uint32_t)row * ROWB + ((uint32_t)(c ^ sw) << 4) + 2u * (uint32_t)cq;
        };
        for (int w = w_first; w < p.num_work; w += w_step) {
            float d[BN / 2];
            tc_mma_loop<TC_BF16, BN, KK, ST>(d, p, base, wg, lane, ring, w_full);
            if (!epi_mem) continue;
            const TcItem it = tc_item(p, w, BN);
            const int n0 = it.n0;
            bool valid[2];
#pragma unroll
            for (int h = 0; h < 2; ++h)                    // border / padding rows of the merged-row tiling are stored as zeros
                valid[h] = tc_pixel(p, it, 64 * wg + rl + 8 * h).valid(p);
            const int nslab = (min(BN, p.n - n0) + SW - 1) / SW;   // slabs holding filters < n
            // the buffer is back from the store thread: the previous item's bulk stores have read it, this item's residual is in it
            long long dt = 0;
            timed<ST>(dt, [&] { mbar_wait(stg_ready(wg), stg_phase); });
            if (w != w_first) w_ready += dt;
            else if (ST && p.stats && warp == 0 && lane == 0) tc_stat(p, STAT_CONS_FIRST_READY) = dt;
            stg_phase ^= 1u;
#pragma unroll
            for (int s = 0; s < BN / SW; ++s) {
                if (s >= nslab) break;
                const uint32_t slab = buf + (uint32_t)s * TILE;
#pragma unroll
                for (int jj = 0; jj < SW / 8; ++jj) {
                    const int j = s * (SW / 8) + jj;
                    const float2 b = *reinterpret_cast<const float2 *>(bias_s + n0 + 8 * j + cq);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float a = d[4 * j + e] + ((e & 1) ? b.y : b.x);
                        d[4 * j + e] = leaky ? fmaxf(a, 0.1f * a) : a;   // == a > 0 ? a : 0.1a
                    }
                }
                // (no "memory" clobbers on the slab accesses: only this thread touches these words between the barriers, and the
                // bias loads may then be scheduled freely around them)
                if (has_res) {
                    uint32_t u[SW / 8][2];
#pragma unroll
                    for (int jj = 0; jj < SW / 8; ++jj)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u[jj][h]) : "r"(slab + slab_off(rl + 8 * h, jj)));
#pragma unroll
                    for (int jj = 0; jj < SW / 8; ++jj) {
                        const int j = s * (SW / 8) + jj;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            float a = d[4 * j + 2 * h] + __uint_as_float(u[jj][h] << 16);
                            float c = d[4 * j + 2 * h + 1] + __uint_as_float(u[jj][h] & 0xffff0000u);
                            if (leaky2) { a = fmaxf(a, 0.1f * a); c = fmaxf(c, 0.1f * c); }
                            d[4 * j + 2 * h] = a; d[4 * j + 2 * h + 1] = c;
                        }
                    }
                }
#pragma unroll
                for (int jj = 0; jj < SW / 8; ++jj) {
                    const int j = s * (SW / 8) + jj;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t o = valid[h] ? pack_bf16x2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]) : 0u;
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(slab + slab_off(rl + 8 * h, jj)), "r"(o));
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the TMA engine
                __syncwarp();
                if (lane == 0) mbar_arrive(stg_full(wg, s));
            }
        }
    });
    if (ST && p.stats && warp == 0 && lane == 0) {
        tc_stat(p, STAT_CONS_WAIT_FULL) = w_full; tc_stat(p, STAT_CONS_WAIT_READY) = w_ready;
        tc_stat(p, STAT_CONS_TOTAL) = clock64() - t_begin;
    }
}

// ------------------------------------------------------------------------------------------------------
// Stem convolution (3 input channels, 3x3 / stride 1 / pad 1) on the tensor cores.
// K = 27 is padded to 32: every thread gathers the 3x3x3 window of ITS pixel straight from the caller's NCHW f32
// image (the layout conversion is fused away), converts to bf16 and writes one 64-byte row of a 64B-swizzled A tile;
// the warpgroup then issues four wgmmas (two M=64 row halves x two K=16 steps, N = 32) and every thread reads its
// pixel's row back through a shared-memory transpose, then bias + leaky-ReLU into bf16 NHWC.  No TMA (the gather is
// irregular), single-buffered, several CTAs per SM.
// ------------------------------------------------------------------------------------------------------
struct StemTcP {
    const float *in;          // NCHW f32, set per call
    const unsigned char *in8; // or: HWC 8-bit frames of exactly the network size (U8 instantiations), set per call
    char *out; int out_ldc;   // bf16 padded NHWC (k_stem_s2_tc: layer 1's output)
    const __nv_bfloat16 *w;   // [32 rows (filters, zero padded)][32 k] bf16, k = (ky,kx,c), k >= 27 zero
    const float *bias;
    int N, H, W, OHp, OWp, nf, act;
    long npix;
    int ntiles;
    // k_stem_s2_tc only: layer 1 (3x3 / stride 2 / pad 1, 32 -> 64 filters) and its tiling
    const __nv_bfloat16 *w1;  // [64 filters][9 * 32] bf16, K ordered (ky, kx, c)
    const float *bias1;
    int act1, OH, OW, xt, yt;
};

// U8: the input is the caller's 8-bit HWC frame (already of the network size): value = (float)((double)v / 255.0) exactly as
// load_image_stb computes it (additionally.c:3093-3103), through a 256-entry table (the correctly rounded f32 division v / 255.f
// gives the same 256 floats, but ~8 instructions per value made this issue-bound kernel 0.3 ms slower) -- the u8 -> planar float pass over the batch
// (71 MB written, 71 MB read back) disappears from the serving path.
template <bool U8>
__global__ void __launch_bounds__(128) k_stem_tc(StemTcP p) {
    __shared__ __align__(1024) uint8_t a_tile[128 * 64];
    __shared__ __align__(1024) uint8_t b_tile[32 * 64];
    __shared__ __align__(16) float acc_s[128 * 36];   // [pixel][filter] f32, rows padded to 36 words
    __shared__ float bias_s[32];
    __shared__ unsigned long long optr[128];   // global address of every pixel's output row of the current tile (0: none)
    __shared__ float lut[U8 ? 256 : 1];
    const int t = threadIdx.x;
    if constexpr (U8) { lut[t] = (float)((double)(float)t / 255.0); lut[t + 128] = (float)((double)(float)(t + 128) / 255.0); }
    const uint32_t a_addr = smem_u32(a_tile), b_addr = smem_u32(b_tile), acc_addr = smem_u32(acc_s);
    if (t < 32) bias_s[t] = (t < p.nf) ? p.bias[t] : 0.f;
    {   // weights -> swizzled B tile (row f, 16-byte chunk j at f*64 + ((j ^ ((f>>1)&3)) << 4))
        const int f = t >> 2, j = t & 3;
        const uint4 v = *reinterpret_cast<const uint4 *>(p.w + f * 32 + j * 8);
        *reinterpret_cast<uint4 *>(b_tile + f * 64 + ((j ^ ((f >> 1) & 3)) << 4)) = v;
    }
    __syncthreads();
    // descriptors: K-major, 64-byte rows (64B swizzle = 2), SBO = 8 rows * 64 B
    const uint32_t hi = ((8u * 64u) >> 4) | (2u << 30);
    const size_t plane = (size_t)p.H * p.W;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const unsigned pix = (unsigned)tile * 128u + (unsigned)t;     // npix < 2^31 (checked by the plan): 32-bit divisions
        const bool ok = pix < (unsigned)p.npix;
        int x = 0, y = 0, n = 0;
        if (ok) { const unsigned row = pix / (unsigned)p.W; x = (int)(pix - row * (unsigned)p.W); n = (int)(row / (unsigned)p.H); y = (int)(row - (unsigned)n * (unsigned)p.H); }
        // ---- gather 27 taps (k = (ky*3 + kx)*3 + c), pad to 32, as bf16
        uint32_t packed[16];
        {
            float v[32];
            if constexpr (U8) {
                const unsigned char *img8 = p.in8 + (size_t)n * 3 * plane;
                if (ok && x >= 1 && x + 1 < p.W && y >= 1 && y + 1 < p.H) {
                    const unsigned char *r1 = img8 + ((size_t)y * p.W + x) * 3, *r0 = r1 - (size_t)p.W * 3, *r2 = r1 + (size_t)p.W * 3;
#pragma unroll
                    for (int j = 0; j < 9; ++j) {          // j = kx * 3 + c: nine consecutive bytes per image row
                        v[0 * 9 + j] = lut[__ldg(r0 - 3 + j)];
                        v[1 * 9 + j] = lut[__ldg(r1 - 3 + j)];
                        v[2 * 9 + j] = lut[__ldg(r2 - 3 + j)];
                    }
                } else {
#pragma unroll
                    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                        for (int kx = 0; kx < 3; ++kx) {
                            const int iy = y + ky - 1, ix = x + kx - 1;
                            const bool in_img = ok && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
#pragma unroll
                            for (int c = 0; c < 3; ++c)
                                v[(ky * 3 + kx) * 3 + c] = in_img ? lut[__ldg(img8 + ((size_t)iy * p.W + ix) * 3 + c)] : 0.f;
                        }
                }
            } else {
            const float *img = p.in + (size_t)n * 3 * plane;
            if (ok && x >= 1 && x + 1 < p.W && y >= 1 && y + 1 < p.H) {
                // interior pixel (all but the image frame): nine row pointers, immediate offsets -1 / 0 / +1 -- the bounds-checked
                // form below costs ~10 integer instructions per tap and made this kernel issue-bound (ncu: 627 instructions per
                // warp and tile)
                const float *c0 = img + (size_t)y * p.W + x;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float *r1 = c0 + (size_t)c * plane, *r0 = r1 - p.W, *r2 = r1 + p.W;
                    v[(0 * 3 + 0) * 3 + c] = __ldg(r0 - 1); v[(0 * 3 + 1) * 3 + c] = __ldg(r0); v[(0 * 3 + 2) * 3 + c] = __ldg(r0 + 1);
                    v[(1 * 3 + 0) * 3 + c] = __ldg(r1 - 1); v[(1 * 3 + 1) * 3 + c] = __ldg(r1); v[(1 * 3 + 2) * 3 + c] = __ldg(r1 + 1);
                    v[(2 * 3 + 0) * 3 + c] = __ldg(r2 - 1); v[(2 * 3 + 1) * 3 + c] = __ldg(r2); v[(2 * 3 + 2) * 3 + c] = __ldg(r2 + 1);
                }
            } else {
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int iy = y + ky - 1, ix = x + kx - 1;
                    const bool in_img = ok && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                        v[(ky * 3 + kx) * 3 + c] = in_img ? __ldg(img + (size_t)c * plane + (size_t)iy * p.W + ix) : 0.f;
                }
            }
            }
#pragma unroll
            for (int k = 27; k < 32; ++k) v[k] = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) packed[k] = pack_bf16x2(v[2 * k], v[2 * k + 1]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
            *reinterpret_cast<uint4 *>(a_tile + t * 64 + ((j ^ ((t >> 1) & 3)) << 4)) =
                make_uint4(packed[4 * j], packed[4 * j + 1], packed[4 * j + 2], packed[4 * j + 3]);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
        __syncthreads();
        {
            float d0[16], d1[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
            wg_fence();
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const uint64_t bdesc = wg_desc(b_addr + 32u * k, hi);
                Wg<TC_BF16, 32>::mma(d0, wg_desc(a_addr + 32u * k, hi), bdesc, (uint32_t)k);            // pixels 0..63
                Wg<TC_BF16, 32>::mma(d1, wg_desc(a_addr + 64u * 64u + 32u * k, hi), bdesc, (uint32_t)k);  // pixels 64..127
            }
            wg_commit();
            wg_wait<0>();
            acc_store_frag(acc_addr, 36, 0, d0);
            acc_store_frag(acc_addr, 36, 64, d1);
        }
        __syncthreads();
        uint32_t acc[32];
        acc_ld32(acc_addr + 4u * 36u * (uint32_t)t, acc);
        char *orow = ok ? p.out + ((size_t)(n * p.OHp + y + 1) * p.OWp + x + 1) * (size_t)p.out_ldc * 2 : nullptr;
        if (p.nf == 32) {
            // 64-byte pixel rows: stage the tile in shared memory (the A tile is free once the MMA has retired) and write it out
            // 512 contiguous bytes per warp instruction.  One STG.128 per thread on its own row touched 16 lines per instruction:
            // the L1 store wavefronts, not HBM, bounded this kernel.
            uint4 o[4];
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                float r[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float a = __uint_as_float(acc[g * 8 + j]) + bias_s[g * 8 + j];
                    r[j] = (p.act == ACT_LEAKY) ? fmaxf(a, 0.1f * a) : a;
                }
                o[g] = make_uint4(pack_bf16x2(r[0], r[1]), pack_bf16x2(r[2], r[3]), pack_bf16x2(r[4], r[5]), pack_bf16x2(r[6], r[7]));
            }
#pragma unroll
            for (int g = 0; g < 4; ++g) *reinterpret_cast<uint4 *>(a_tile + t * 64 + ((g ^ ((t >> 1) & 3)) << 4)) = o[g];
            optr[t] = (unsigned long long)(uintptr_t)orow;
            __syncthreads();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int j = t + 128 * k, px = j >> 2, part = j & 3;
                const unsigned long long dst = optr[px];
                if (dst)
                    *reinterpret_cast<uint4 *>(dst + (unsigned long long)(part * 16)) =
                        *reinterpret_cast<const uint4 *>(a_tile + px * 64 + ((part ^ ((px >> 1) & 3)) << 4));
            }
        } else if (ok) {
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                if (g * 8 >= p.nf) break;
                float r[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float a = __uint_as_float(acc[g * 8 + j]) + bias_s[g * 8 + j];
                    r[j] = (p.act == ACT_LEAKY) ? fmaxf(a, 0.1f * a) : a;
                }
                reinterpret_cast<uint4 *>(orow)[g] = make_uint4(pack_bf16x2(r[0], r[1]), pack_bf16x2(r[2], r[3]),
                                                                pack_bf16x2(r[4], r[5]), pack_bf16x2(r[6], r[7]));
            }
        }
        __syncthreads();   // accumulator row drained and A tile consumed before the next tile overwrites them
    }
}

// ------------------------------------------------------------------------------------------------------
// The tensor-core stem fused with the 3x3 / stride-2 / pad-1 convolution that reads it (32 -> 64 filters): the stem output
// (378 MB in bf16 for yolov3 at 608^2, batch 16) stays in shared memory, HBM sees the image and layer 1's output only.
// Work item: a 16 x 8 tile of layer-1 output pixels of one image, all 64 filters.  Per tile:
//   1. The tile's image patch (3 x 19 x 35 values, f32 or 8-bit through the same table as k_stem_tc, zeros outside the image)
//      is loaded into registers while the previous tile's layer 1 runs and stored to shared memory; from it, the im2col rows of the 17 x 33 stem pixels the tile
//      reads (2 * 8 + 1 rows, 2 * 16 + 1 columns, pad 1 included), k_stem_tc's A operand with no bounds logic.  561 rows padded
//      to 640 = 10 M=64 chunks.
//   2. stem wgmmas: warpgroup g takes chunks 5 g .. 5 g + 4, two m64n32k16 each, as k_stem_tc does; then bias, leaky and
//      bf16, k_stem_tc's arithmetic: the stem values are bit-identical.  Stem pixels outside the image are layer 1's zero pad
//      and are written as zeros.
//   3. Layer 1 reads those values from "sets": 16 rows of 64 bytes (1 KB), row ox = stem pixel (sy, 2 ox + kx), one set per
//      stem row sy and column phase kx (odd region columns sit in two sets).  Per kx: the 9 even rows' sets, then the 8 odd
//      ones, so that tap (ky, kx) of the 128 tile pixels (oy, ox) -> stem (2 oy + ky, 2 ox + kx) is one canonical 128-row
//      K-major matrix (64B swizzle) starting at set ky / 2 of parity ky & 1; warpgroup g's 64 rows start 4 sets further.  Every
//      operand base is 1 KB aligned: plain descriptors, no gather, no bank conflicts.  Layer 1 then runs k_conv_tc_reg's
//      instruction sequence at BN = 64 (filter matrix resident in shared memory, taps in (ky, kx) order, two m64n64k16 per
//      tap) and its epilogue (bias, leaky, bf16): bit-identical to the unfused layer.
//   4. The accumulators go through a swizzled staging tile (8 KB per warpgroup) to 16-byte coalesced stores into layer 1's
//      padded NHWC output; pixels past OW / OH are not stored, the zero border is never written.
// Shared memory: the im2col rows, the sets and the staging tiles share one region (their lifetimes are separated by the
// block barriers), ~104 KB per CTA in all: two CTAs per SM, so that one CTA's patch loads and stores overlap the other's
// wgmmas.  Persistent grid of 2 CTAs per SM (YB_TC_GRID caps it).
// ------------------------------------------------------------------------------------------------------
constexpr int S2_TW = 16, S2_TH = 8;                           // layer-1 output pixels per tile
constexpr int S2_RW = 2 * S2_TW + 1, S2_RH = 2 * S2_TH + 1;    // stem region of a tile: 33 x 17
constexpr int S2_ROWS = 640;                                   // 561 stem pixels padded to 10 chunks of 64
constexpr uint32_t S2_B1 = 0;                                  // layer-1 filters: 9 taps x [64 filters][64 B]
constexpr uint32_t S2_BS = 9u * 4096u;                         // stem filters: [32][64 B]
constexpr uint32_t S2_U = S2_BS + 2048u;                       // im2col rows | sets | staging
constexpr uint32_t S2_SETS_KX = 17u * 1024u;                   // per kx: 9 even-row sets, then 8 odd-row sets
constexpr uint32_t S2_STG = (uint32_t)S2_ROWS * 64u;           // staging tiles (in U), past the im2col rows
constexpr uint32_t S2_MISC = S2_U + S2_STG + 2u * 8192u;       // biases (32 + 64 floats), u8 table (256 floats), image patch
constexpr int S2_PH = S2_RH + 2, S2_PW = S2_RW + 2, S2_PP = 36; // image patch of a tile: 3 x 19 x 35 f32, rows of 36
constexpr size_t S2_SMEM = 1024 + S2_MISC + 4 * (32 + 64 + 256) + 4 * 3 * S2_PH * S2_PP;
static_assert(S2_STG + 2u * 8192u >= 3u * S2_SETS_KX, "sets must fit the shared region");

template <bool U8>
__global__ void __launch_bounds__(256, 2) k_stem_s2_tc(StemTcP p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 64B swizzle atoms: 512-byte aligned
    const uint32_t base = smem_u32(sm), U = base + S2_U;
    float *bias0_s = reinterpret_cast<float *>(sm + S2_MISC), *bias1_s = bias0_s + 32, *lut = bias1_s + 64, *patch = lut + 256;
    const int t = threadIdx.x, lane = t & 31;
    const int warp = __shfl_sync(0xffffffffu, t >> 5, 0), wg = warp >> 2;
    if constexpr (U8) lut[t] = (float)((double)(float)t / 255.0);
    if (t < 32) bias0_s[t] = p.bias[t];
    if (t < 64) bias1_s[t] = p.bias1[t];
    if (t < 128) {   // stem filters, swizzled as in k_stem_tc
        const int f = t >> 2, j = t & 3;
        *reinterpret_cast<uint4 *>(sm + S2_BS + f * 64 + ((j ^ ((f >> 1) & 3)) << 4)) = *reinterpret_cast<const uint4 *>(p.w + f * 32 + j * 8);
    }
    for (int i = t; i < 9 * 64 * 4; i += 256) {   // layer-1 filters: tap r, filter f, 16-byte chunk j (the TMA box layout of k_conv_tc_reg)
        const int r = i >> 8, f = (i >> 2) & 63, j = i & 3;
        *reinterpret_cast<uint4 *>(sm + S2_B1 + r * 4096 + f * 64 + ((j ^ ((f >> 1) & 3)) << 4)) =
            *reinterpret_cast<const uint4 *>(p.w1 + f * 288 + r * 32 + j * 8);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    const uint32_t hi = ((8u * 64u) >> 4) | (2u << 30);   // K-major, 64-byte rows, 64B swizzle, SBO = 8 rows * 64 B
    const bool leaky0 = p.act == ACT_LEAKY, leaky1 = p.act1 == ACT_LEAKY;
    const int rl = 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);   // wgmma fragment: rows rl, rl + 8; columns 8 j + cq, + 1
    // The image patch of a tile (zeros outside the image): each thread loads PER values into registers, all issued back to
    // back, and stores them into `patch` later -- the next tile's loads are in flight while this tile's layer 1 runs.
    constexpr int PER = (3 * S2_PH * S2_PW + 255) / 256;
    auto patch_index = [&](int e, int &c, int &r, int &col) {
        if constexpr (U8) { r = e / (3 * S2_PW); const int b = e - r * 3 * S2_PW; col = b / 3; c = b - col * 3; }
        else { c = e / (S2_PH * S2_PW); const int b = e - c * S2_PH * S2_PW; r = b / S2_PW; col = b - r * S2_PW; }
    };
    auto load_patch = [&](int tile, float (&v)[PER]) {
        const int tx = tile % p.xt, rest = tile / p.xt, ty = rest % p.yt, n = rest / p.yt;
        const int py0 = 2 * ty * S2_TH - 2, px0 = 2 * tx * S2_TW - 2;   // image pixel of patch (0, 0)
        const size_t img = (size_t)n * 3 * p.H * p.W;   // first value of image n (both layouts); offsets in it fit 32 bits
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int e = t + 256 * k;
            int c, r, col;
            patch_index(e, c, r, col);
            const int y = py0 + r, x = px0 + col;
            const bool in_img = e < 3 * S2_PH * S2_PW && y >= 0 && y < p.H && x >= 0 && x < p.W;
            if constexpr (U8) v[k] = in_img ? lut[__ldg(p.in8 + img + (unsigned)((y * p.W + x) * 3 + c))] : 0.f;
            else v[k] = in_img ? __ldg(p.in + img + (unsigned)((c * p.H + y) * p.W + x)) : 0.f;
        }
    };
    float pv[PER];
    if ((int)blockIdx.x < p.ntiles) load_patch(blockIdx.x, pv);
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const int tx = tile % p.xt, rest = tile / p.xt, ty = rest % p.yt, n = rest / p.yt;
        const int ox0 = tx * S2_TW, oy0 = ty * S2_TH;
        const int gy0 = 2 * oy0 - 1, gx0 = 2 * ox0 - 1;   // stem pixel of region (0, 0)

        // ---- 1. the image patch -> shared memory (the previous tile's im2col, which read it, is behind two block barriers)
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int e = t + 256 * k;
            if (e >= 3 * S2_PH * S2_PW) break;
            int c, r, col;
            patch_index(e, c, r, col);
            patch[(c * S2_PH + r) * S2_PP + col] = pv[k];
        }
        __syncthreads();

        // ---- stem im2col rows, i = sy * 33 + sx: k_stem_tc's window (k = (ky*3 + kx)*3 + c, padded to 32) as bf16 pairs
        for (int i = t; i < S2_ROWS; i += 256) {
            const int sy = i / S2_RW, sx = i - sy * S2_RW;
            const float *w0 = patch + sy * S2_PP + sx;
            const bool ok = i < S2_RW * S2_RH;
            uint32_t packed[16];
            {
                float v[32];
#pragma unroll
                for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                        for (int c = 0; c < 3; ++c) v[(ky * 3 + kx) * 3 + c] = ok ? w0[(c * S2_PH + ky) * S2_PP + kx] : 0.f;
#pragma unroll
                for (int k = 27; k < 32; ++k) v[k] = 0.f;
#pragma unroll
                for (int k = 0; k < 16; ++k) packed[k] = pack_bf16x2(v[2 * k], v[2 * k + 1]);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
                *reinterpret_cast<uint4 *>(sm + S2_U + i * 64 + ((j ^ ((i >> 1) & 3)) << 4)) =
                    make_uint4(packed[4 * j], packed[4 * j + 1], packed[4 * j + 2], packed[4 * j + 3]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
        __syncthreads();

        // ---- 2. stem wgmmas
        float ds[5][16];
#pragma unroll
        for (int c = 0; c < 5; ++c)
#pragma unroll
            for (int i = 0; i < 16; ++i) ds[c][i] = 0.f;
#pragma unroll
        for (int c = 0; c < 5; ++c) wg_fence_operand(ds[c]);
        wg_fence();
#pragma unroll
        for (int c = 0; c < 5; ++c)
#pragma unroll
            for (int k = 0; k < 2; ++k)
                Wg<TC_BF16, 32>::mma(ds[c], wg_desc(U + (uint32_t)(5 * wg + c) * 4096u + 32u * k, hi), wg_desc(base + S2_BS + 32u * k, hi), (uint32_t)k);
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int c = 0; c < 5; ++c) wg_fence_operand(ds[c]);
        __syncthreads();   // every stem wgmma has read its rows: the sets may overwrite them

        // ---- stem epilogue into the sets.  Region column sx goes to set kx = 1 (sx odd), or to kx = 0 and / or kx = 2 (sx even).
        // (no "memory" clobbers on these stores: the bias loads may be scheduled freely around them; the barrier below orders them)
        {
#pragma unroll
            for (int c = 0; c < 5; ++c)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = 64 * (5 * wg + c) + rl + 8 * h;
                    if (i >= S2_RW * S2_RH) continue;
                    const int sy = i / S2_RW, sx = i - sy * S2_RW, y = gy0 + sy, x = gx0 + sx;
                    const bool in_img = y >= 0 && y < p.H && x >= 0 && x < p.W;
                    uint32_t v[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        float a = ds[c][4 * j + 2 * h] + bias0_s[8 * j + cq], b = ds[c][4 * j + 2 * h + 1] + bias0_s[8 * j + cq + 1];
                        if (leaky0) { a = fmaxf(a, 0.1f * a); b = fmaxf(b, 0.1f * b); }
                        v[j] = in_img ? pack_bf16x2(a, b) : 0u;
                    }
                    const uint32_t set = U + ((sy & 1) ? 9u * 1024u : 0u) + (uint32_t)(sy >> 1) * 1024u + 2u * (uint32_t)cq;
                    auto put = [&](int kx, int ox) {
                        const uint32_t row = set + (uint32_t)kx * S2_SETS_KX + (uint32_t)ox * 64u;
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(row + ((uint32_t)(j ^ ((ox >> 1) & 3)) << 4)), "r"(v[j]));
                    };
                    const bool odd = sx & 1, last = sx == 2 * S2_TW;
                    put(odd ? 1 : last ? 2 : 0, last ? (sx >> 1) - 1 : sx >> 1);
                    if (!odd && !last && sx >= 2) put(2, (sx >> 1) - 1);
                }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();

        if (tile + (int)gridDim.x < p.ntiles) load_patch(tile + gridDim.x, pv);

        // ---- 3. layer 1: 9 taps x two m64n64k16 into warpgroup wg's 64 rows (tile rows oy = 4 wg .. 4 wg + 3)
        float d[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) d[i] = 0.f;
        wg_fence_operand(d);
        wg_fence();
#pragma unroll
        for (int r = 0; r < 9; ++r) {
            const int ky = r / 3, kx = r % 3;
            const uint32_t a = U + (uint32_t)kx * S2_SETS_KX + ((ky & 1) ? 9u * 1024u : 0u) + (uint32_t)(ky >> 1) * 1024u + (uint32_t)wg * 4096u;
            const uint32_t b = base + S2_B1 + (uint32_t)r * 4096u;
#pragma unroll
            for (int k = 0; k < 2; ++k)
                Wg<TC_BF16, 64>::mma(d, wg_desc(a + 32u * k, hi), wg_desc(b + 32u * k, hi), (r > 0 || k > 0) ? 1u : 0u);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_operand(d);
        __syncthreads();   // both warpgroups are done with the sets: the staging tiles may overwrite them

        // ---- 4. epilogue: staging tile [64 pixels][128 B], 16-byte chunk j of row q at j ^ (q & 7)
        const uint32_t stg = U + S2_STG + (uint32_t)wg * 8192u;
        float b1[16];
#pragma unroll
        for (int j = 0; j < 8; ++j) { b1[2 * j] = bias1_s[8 * j + cq]; b1[2 * j + 1] = bias1_s[8 * j + cq + 1]; }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int q = rl + 8 * h;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float a = d[4 * j + 2 * h] + b1[2 * j], b = d[4 * j + 2 * h + 1] + b1[2 * j + 1];
                if (leaky1) { a = fmaxf(a, 0.1f * a); b = fmaxf(b, 0.1f * b); }   // == a > 0 ? a : 0.1a
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + (uint32_t)q * 128u + ((uint32_t)(j ^ (q & 7)) << 4) + 2u * (uint32_t)cq),
                             "r"(pack_bf16x2(a, b)) : "memory");
            }
        }
        if (wg == 0) named_bar_sync(1, 128);   // constant barrier ids: ptxas reserves 2 barriers, not all 16
        else named_bar_sync(2, 128);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int idx = (t & 127) + 128 * k, q = idx >> 3, ch = idx & 7;
            const int oy = oy0 + 4 * wg + (q >> 4), ox = ox0 + (q & 15);
            if (oy < p.OH && ox < p.OW) {
                uint4 o;
                asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w)
                             : "r"(stg + (uint32_t)q * 128u + ((uint32_t)(ch ^ (q & 7)) << 4)) : "memory");
                *reinterpret_cast<uint4 *>(p.out + ((size_t)(n * p.OHp + oy + 1) * p.OWp + ox + 1) * (size_t)p.out_ldc * 2 + ch * 16) = o;
            }
        }
        // the next tile writes this staging tile only after two block barriers, which every thread reaches after its stores
    }
}

// ------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
            fatal_throw("cuTensorMapEncodeTiled not available from the driver");
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

}  // namespace

// Both kernel families take the same parameters
using TcKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, TcParams);

struct TcPlan {
    CUtensorMap tmA, tmB, tmO, tmO1, tmR;   // activation, filters; TMA epilogue: output, its one-row view (stride 2), residual
    TcParams p;
    TcKernel kernel;                  // the instantiation the plan runs
    bool reg;                         // kernel is a k_conv_tc_reg (TCR_THREADS), else a k_conv_tc (TC_THREADS)
    int grid;
    size_t smem;                      // dynamic shared memory per CTA (tc_smem_layout)
    char desc[96];
    DevBuf<unsigned long long> stats;   // p.stats (YB_TC_STATS)
};

namespace {

int sm_count() {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

bool is_integer(int kind) { return kind == TC_S8 || kind == TC_S8_GPU || kind == TC_XNOR || kind == TC_XNOR_GPU || kind == TC_PM1Z_GPU; }
int elem_size(int kind) { return kind == TC_TF32 ? 4 : is_integer(kind) ? 1 : 2; }   // operand element size
// operand channels per pixel: the integer kinds read the s8 input's zero-padded channels (their weights are padded alike)
int operand_channels(const TcConv &c) { return is_integer(c.kind) ? c.in.ldc : c.l->c; }

// The filter geometries of the implicit GEMM: 3x3 / pad 1 and 1x1 / pad 0 at stride 1; 3x3 / pad 1 at stride 2 on even sizes
// (the 5-D view splits x and y into (half, parity))
bool geometry_ok(const Layer &l) {
    if (l.stride == 1) return (l.size == 3 && l.pad == 1) || (l.size == 1 && l.pad == 0);
    return l.stride == 2 && l.size == 3 && l.pad == 1 && l.h % 2 == 0 && l.w % 2 == 0;
}

// Channels per K-block: the widest 128 / 64 / 32-byte row (a TMA / wgmma swizzle width) that divides `channels` elements of
// esz bytes, or 0
int channel_row(int channels, int esz) {
    for (int bytes = 128; bytes >= 32; bytes /= 2)
        if (channels * esz % bytes == 0) return bytes / esz;
    return 0;
}

// k_conv_tc: at most 128 filters per tile -- the [128][BN + 4] f32 accumulator tile shares the 227 KB of shared memory with the ring
int pick_bn(int n) { return n <= 32 ? 32 : n <= 64 ? 64 : 128; }
// k_conv_tc_reg: BN in {32, 64, 128, 256} (no wider than the filters need) with the least wave-quantised cost
//     ceil(work items / SMs) * (K-blocks * (BN + 64) + 2 * BN).
// A K-block of a 128 x BN tile feeds 128 activation rows and BN filter rows for BN columns of MMA work: the + 64 charges the
// activation tile's share of the feed, 2 * BN the register epilogue.  E.g. 1x1 512 -> 256 at 38x38, batch 16: 380 work items
// at BN = 128 (3 waves) against 190 at BN = 256 (2 waves of double-length tiles), and BN = 128 is cheaper.
// forced > 0 (YB_TC_BN) takes that width instead (capped at the filters' width; A/B experiments).
int pick_bn_reg(int n, long m_tiles, int kblocks, int sms, int forced) {
    int cap = 32;
    while (cap < n && cap < 256) cap *= 2;
    if (forced > 0) {
        int bn = 32;
        while (bn * 2 <= std::min(forced, cap)) bn *= 2;
        return bn;
    }
    int best = 32; double best_cost = 1e300;
    for (int bn = 32; bn <= cap; bn *= 2) {
        const long items = m_tiles * ((n + bn - 1) / bn);
        const double cost = (double)((items + sms - 1) / sms) * ((double)kblocks * (bn + 64) + 2.0 * bn);
        if (cost < best_cost) { best_cost = cost; best = bn; }
    }
    return best;
}

// Persistent grid size of the tensor-core plans: one CTA per SM, or at most max_grid > 0 (YB_TC_GRID; tests: several work items
// per CTA reuse the epilogue buffers and flip the barrier phases many times on small layers).
int grid_cap(int sms, int max_grid) { return max_grid > 0 ? std::min(sms, max_grid) : sms; }

// Geometry, K-blocks, tile shape, filter tile width and the resident filter matrix.  reg: k_conv_tc_reg runs the plan.
void plan_tiles(TcParams &p, const TcConv &c, bool reg, int sms) {
    const Layer &l = *c.l;
    const bool s2 = l.stride == 2;
    const int esz = elem_size(c.kind), cin = operand_channels(c);
    p.kind = c.kind;
    p.N = c.in.N;
    p.OH = l.out_h; p.OW = l.out_w; p.OHp = c.out.Hp; p.OWp = c.out.Wp;
    p.size = l.size; p.BK = channel_row(cin, esz);
    p.kk = p.BK * esz / 32;
    p.cblocks = cin / p.BK; p.kblocks = l.size * l.size * p.cblocks;
    p.stride2 = s2 ? 1 : 0;
    p.xoff = 1 - l.pad; p.yoff = -l.pad;
    p.PR = s2 ? (c.in.Hp / 2) : c.in.Hp;
    p.row_off = s2 ? 0 : 1;
    // wgmma descriptor high word: SBO (8 rows * row bytes) >> 4 at bits 32..45, swizzle mode at 62..63 (1: 128B, 2: 64B, 3: 32B)
    const uint32_t row_bytes = 32u * (uint32_t)p.kk;
    p.desc_hi = ((8u * row_bytes) >> 4) | ((row_bytes == 128 ? 1u : row_bytes == 64 ? 2u : 3u) << 30);

    // tile width: power of two minimising padded work
    const long rows = (long)p.N * p.PR;
    auto padded = [&](int tw) {
        const int th = 128 / tw;
        return (double)((p.OW + tw - 1) / tw) * tw * (double)((rows + th - 1) / th) * th;
    };
    double best = 1e30; int tw = 1;
    for (int t = 1; t <= 128; t *= 2)
        if (padded(t) < best - 0.5) { best = padded(t); tw = t; }
    if (c.yolo_out) {
        // the epilogue scatters NCHW planes (fused [yolo]): a warp's 32 accumulator rows should be as few image-row runs as
        // possible, so take the widest tile whose padded work stays within 30 % of the minimum
        for (int t = 64; t > tw; t /= 2)
            if (padded(t) <= 1.3 * best) { tw = t; break; }
    }
    // a fused 2x2 max-pool needs 8 x 16 tiles that start one merged row down -- row 0 is a border row, and 2x2 windows then
    // never straddle tiles
    if (c.pool_fmt != SIDE_NONE) tw = 8;
    p.jshift = c.pool_fmt != SIDE_NONE ? 1 : 0;
    auto set_tw = [&](int t) {
        p.TW = t; p.TH = 128 / t;
        p.TWlog2 = 0; while ((1 << p.TWlog2) < p.TW) ++p.TWlog2;
        p.xt = (p.OW + p.TW - 1) / p.TW;
        p.jt = (int)((rows - p.jshift + p.TH - 1) / p.TH);
    };
    set_tw(tw);
    p.BN = reg ? pick_bn_reg(l.n, (long)p.xt * p.jt, p.kblocks, sms, c.sw.bn) : pick_bn(l.n);
    // k_conv_tc_reg stores straddling stride-2 half tiles one tile row at a time, from byte t * TW * 2 SW of a slab: with
    // 64-byte slab rows (SW = 32) and TW = 1 that is not 128-byte aligned, as bulk tensor copies need
    if (reg && s2 && p.BN == 32 && p.TW == 1) set_tw(2);
    p.nt = (l.n + p.BN - 1) / p.BN;
    p.num_work = p.xt * p.jt * p.nt;
    p.a_bytes = (uint32_t)(TC_BM * p.BK * esz);
    p.b_bytes = (uint32_t)(p.BN * p.BK * esz);
    // small filter matrices stay resident in shared memory for the whole kernel (one TMA pass per CTA)
    p.bstat = (p.nt == 1 && (size_t)p.kblocks * p.b_bytes <= 48 * 1024 && !c.sw.no_bstat) ? 1 : 0;
    p.bstat_bytes = p.bstat ? (uint32_t)p.kblocks * p.b_bytes : 0u;
}

// The epilogue: the output, the per-kind parameters, the fusions and the staging tiles.  k_conv_tc_reg (reg): bf16 slabs of 64
// columns (32 when BN == 32) stored by TMA, per consumer warpgroup one staging buffer of 64 pixels x BN (64 / 32 / 16 / 8 KB per
// CTA at BN = 256 / 128 / 64 / 32).  k_conv_tc: the stride-1 integer kinds store f32 slabs of 32 columns (128-byte rows) by TMA,
// one 128-pixel tile per warp group; the raw-accumulator dump (tests) and the float kinds store through per-warp LSU staging tiles.
void plan_epilogue(TcParams &p, const TcConv &c, bool reg) {
    const Layer &l = *c.l;
    p.tma_epi = reg ? (p.BN >= 64 ? 64 : 32) : (is_integer(c.kind) && !p.stride2 && !c.acc_out) ? 32 : 0;
    p.stg_bytes = reg ? 2u * 64u * (uint32_t)p.BN * 2u : p.tma_epi ? 2u * 16384u : 4096u * TC_EPI_WARPS;
    p.acc_pitch = p.BN + 4;
    p.out = c.out.base; p.out_ldc = c.out.ldc;
    p.n = l.n;
    p.res = c.res.base;
    p.bias = c.bias; p.act = l.activation; p.act2 = c.act2;
    p.alpha1 = c.alpha1;
    p.mean = c.mean;
    p.xK = l.size * l.size * l.c;
    p.acc_out = c.acc_out;
    p.yolo_out = c.yolo_out;
    p.yolo_per = c.yolo_out ? 4 + c.yolo_classes + 1 : 0;
    p.pool_fmt = c.pool_fmt; p.pool_mult = c.pool_mult;
    p.pool_out = reinterpret_cast<signed char *>(c.pool_next.base); p.pool_ldc = c.pool_next.ldc;
    p.pool_Hp = c.pool_next.Hp; p.pool_Wp = c.pool_next.Wp;
}

// Sizes of the epilogue's regions of shared memory (see tc_smem_layout).  reg: k_conv_tc_reg runs the plan.
struct TcEpiBytes {
    size_t bias, ymask, stg, acc;
    size_t sum() const { return bias + ymask + stg + acc; }
};
TcEpiBytes epi_bytes(const TcParams &p, bool reg) {
    const size_t f = (size_t)p.nt * p.BN;
    return {sizeof(float) * f,                                     // f32 bias of every filter tile
            reg ? 0 : f / 8,                                       // k_conv_tc's fused [yolo] mask: one bit per filter
            p.stg_bytes,                                           // epilogue staging or TMA-epilogue tiles
            reg ? 0 : (size_t)TC_BM * p.acc_pitch * sizeof(float)};   // k_conv_tc's accumulator tile (k_conv_tc_reg: registers)
}

// The operand ring: K-blocks per stage and stages, in what is left of 222 KB beside the resident filter matrix and the epilogue's
// regions.  The other 5 KB of the 227 KB cover the barriers and the alignment padding of tc_smem_layout.
void plan_ring(TcParams &p, bool reg) {
    const size_t ring_budget = (size_t)(227 - 5) * 1024 - epi_bytes(p, reg).sum();
    // several K-blocks per stage when they are small: fewer barrier round trips per K
    const uint32_t ring_blk = p.a_bytes + (p.bstat ? 0u : p.b_bytes);
    p.sps = (int)std::max<uint32_t>(1, std::min<uint32_t>(4, 32u * 1024u / std::max(ring_blk, 1u)));
    p.sps = std::min(p.sps, p.kblocks);
    if (ring_budget < p.bstat_bytes + 2 * (size_t)ring_blk) fatal_throw("tc plan: tile does not fit shared memory");
    const size_t avail = ring_budget - p.bstat_bytes;
    while (p.sps > 1 && avail / ((size_t)p.sps * ring_blk) < 3) --p.sps;   // keep the ring at least 3 stages deep
    p.stage_bytes = (uint32_t)p.sps * ring_blk;
    p.stages = (int)std::min<size_t>(8, avail / p.stage_bytes);
    if (p.stages < 2) fatal_throw("tc plan: tile does not fit shared memory");
}

// The dynamic shared memory of a plan whose sizes are decided: places every region (TcParams::sm) at its alignment, in this
// order, and returns the bytes the launch asks for -- the regions plus 1024 bytes of slack for aligning the kernel's base.
//   resident filter matrix   bstat_bytes                  1024 (128B swizzle atoms)
//   operand ring             stages x stage_bytes         1024
//   mbarriers                full[stages], empty[stages], the resident-filter barrier; k_conv_tc_reg:
//                            stg_full[2][TCR_MAX_SLABS], stg_ready[2]            8
//   bias, [yolo] mask        epi_bytes                    16, 4
//   staging                  stg_bytes                    1024 with the TMA epilogue (swizzled tiles), else 128
//   accumulator tile         epi_bytes                    16
size_t tc_smem_layout(TcParams &p, bool reg) {
    const TcEpiBytes epi = epi_bytes(p, reg);
    size_t top = 0;
    auto place = [&](size_t bytes, size_t align) {
        const size_t off = (top + align - 1) / align * align;
        top = off + bytes;
        return (uint32_t)off;
    };
    // the A and B boxes of every ring stage, and the filter matrix's boxes, are swizzled tiles: they keep the 1024-byte alignment
    if (p.a_bytes % 1024 || p.b_bytes % 1024) fatal_throw("tc plan: operand tiles break the 1024-byte swizzle alignment");
    place(p.bstat_bytes, 1024);
    p.sm.ring = place((size_t)p.stages * p.stage_bytes, 1024);
    const int nbars = 2 * p.stages + 1 + (reg ? 2 * TCR_MAX_SLABS + 2 : 0);
    p.sm.full = place(8 * (size_t)nbars, 8);
    p.sm.empty = p.sm.full + 8u * (uint32_t)p.stages;
    p.sm.bstat_bar = p.sm.empty + 8u * (uint32_t)p.stages;
    p.sm.stg_full = reg ? p.sm.bstat_bar + 8u : 0u;
    p.sm.stg_ready = reg ? p.sm.stg_full + 8u * 2u * TCR_MAX_SLABS : 0u;
    p.sm.bias = place(epi.bias, 16);
    p.sm.ymask = reg ? 0u : place(epi.ymask, 4);
    p.sm.stg = place(epi.stg, p.tma_epi ? 1024 : 128);
    p.sm.acc = reg ? 0u : place(epi.acc, 16);
    const size_t smem = 1024 + top;
    if (smem > 227 * 1024) fatal_throw("tc plan: shared memory budget exceeded");
    return smem;
}

// The tensor maps: activation boxes of a K-block, filter boxes and, for the TMA epilogue, the output and residual slabs
void encode_maps(TcPlan &plan, const TcConv &c, bool reg) {
    const TcParams &p = plan.p;
    const TV &in = c.in;
    const int esz = elem_size(c.kind), cin = operand_channels(c);
    const CUtensorMapSwizzle swz = p.kk == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : p.kk == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    const CUtensorMapDataType dtype = c.kind == TC_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                    : is_integer(c.kind) ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    EncodeTiledFn enc = encode_fn();
    auto check = [](CUresult r, const char *what) {
        if (r != CUDA_SUCCESS) fatal_throw(std::string("cuTensorMapEncodeTiled(") + what + ") failed: " + std::to_string((int)r));
    };
    if (!p.stride2) {
        // activation view (c, x_padded, merged padded rows)
        cuuint64_t dims[3] = {(cuuint64_t)cin, (cuuint64_t)in.Wp, (cuuint64_t)in.N * in.Hp};
        cuuint64_t strides[2] = {(cuuint64_t)in.ldc * esz, (cuuint64_t)in.Wp * in.ldc * esz};
        cuuint32_t box[3] = {(cuuint32_t)p.BK, (cuuint32_t)p.TW, (cuuint32_t)p.TH};
        cuuint32_t es[3] = {1, 1, 1};
        check(enc(&plan.tmA, dtype, 3, in.base, dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE), "A");
    } else {
        // stride 2: (c, x parity, x half, y parity, merged y half)
        cuuint64_t dims[5] = {(cuuint64_t)cin, 2, (cuuint64_t)in.Wp / 2, 2, (cuuint64_t)in.N * in.Hp / 2};
        cuuint64_t strides[4] = {(cuuint64_t)in.ldc * esz, (cuuint64_t)in.ldc * 2 * esz, (cuuint64_t)in.Wp * in.ldc * esz,
                                 (cuuint64_t)in.Wp * in.ldc * 2 * esz};
        cuuint32_t box[5] = {(cuuint32_t)p.BK, 1, (cuuint32_t)p.TW, 1, (cuuint32_t)p.TH};
        cuuint32_t es[5] = {1, 1, 1, 1, 1};
        check(enc(&plan.tmA, dtype, 5, in.base, dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE), "A");
    }
    {
        const cuuint64_t K = (cuuint64_t)p.size * p.size * cin;
        cuuint64_t dims[2] = {K, (cuuint64_t)c.ldn};
        cuuint64_t strides[1] = {K * esz};
        cuuint32_t box[2] = {(cuuint32_t)p.BK, (cuuint32_t)p.BN};
        cuuint32_t es[2] = {1, 1};
        check(enc(&plan.tmB, dtype, 2, const_cast<void *>(c.w), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE), "B");
    }
    plan.tmO = plan.tmA; plan.tmO1 = plan.tmA; plan.tmR = plan.tmA;   // valid placeholders when unused
    if (p.tma_epi && c.out.base) {   // a plan with a fused max-pool has no output to map
        const int oesz = c.out_bf16 ? 2 : 4;
        auto encode_px = [&](CUtensorMap *tm, const TV &t, const char *what, int box_rows) {
            // (channels, padded x, merged padded rows) of a padded-NHWC tensor (bf16, or f32 for the integer kinds); box = one
            // slab of a pixel tile (k_conv_tc_reg: half a tile, the 64 pixels of one consumer warpgroup), box_rows rows of it
            cuuint64_t dims[3] = {(cuuint64_t)p.n, (cuuint64_t)t.Wp, (cuuint64_t)t.N * t.Hp};
            cuuint64_t strides[2] = {(cuuint64_t)t.ldc * oesz, (cuuint64_t)t.Wp * t.ldc * oesz};
            cuuint32_t box[3] = {(cuuint32_t)p.tma_epi, (cuuint32_t)std::min(p.TW, reg ? 64 : 128), (cuuint32_t)box_rows};
            cuuint32_t es[3] = {1, 1, 1};
            check(enc(tm, c.out_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, t.base, dims, strides, box, es,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, p.tma_epi * oesz == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE), what);
        };
        const int box_rows = reg ? std::max(p.TH / 2, 1) : p.TH;
        encode_px(&plan.tmO, c.out, "output", box_rows);
        if (reg && p.stride2) encode_px(&plan.tmO1, c.out, "output row", 1);   // straddling half tiles, one tile row per store
        if (c.res.base) encode_px(&plan.tmR, c.res, "residual", box_rows);
    }
}

}  // namespace

int tc_conv_supported(const TcConv &c) {
    const Layer &l = *c.l;
    const bool integer = is_integer(c.kind);
    // every view it reads or writes must be one TMA can address: a vec16_view
    if (!geometry_ok(l) || l.n < 8 || (l.activation != YB_LEAKY && l.activation != YB_LINEAR)) return 0;
    if (channel_row(operand_channels(c), elem_size(c.kind)) == 0 || c.in.P != 1 || !vec16_view(c.in, elem_size(c.kind))) return 0;
    // bf16 output: the bf16 kind only, whole 16-byte filter groups
    if (c.out_bf16 && (c.kind != TC_BF16 || l.n % 8 != 0)) return 0;
    if (c.out.base ? (c.out.P != 1 || !vec16_view(c.out, c.out_bf16 ? 2 : 4)) : !(c.yolo_out || c.pool_fmt != SIDE_NONE)) return 0;
    // fused shortcut: k_conv_tc_reg at stride 1
    if (c.res.base && !(c.kind == TC_BF16 && c.out_bf16 && l.stride == 1 && c.res.H == l.out_h && c.res.W == l.out_w &&
                        c.res.C == l.n && vec16_view(c.res, 2)))
        return 0;
    // fused [yolo]: the f32 epilogue of k_conv_tc
    if (c.yolo_out && (integer || c.out_bf16)) return 0;
    // fused max-pool: the 8 x 16 tiles of the stride-1 3x3 integer layers start one merged row down, so 2x2 windows never
    // straddle tiles when the padded height and the output size are even; the epilogue writes whole 32-filter groups of bytes
    if (c.pool_fmt != SIDE_NONE && !(integer && (side_s8(c.pool_fmt) || c.pool_fmt == SIDE_PM1_S8) && !c.acc_out && l.size == 3 && l.stride == 1 &&
                         l.h % 2 == 0 && l.out_h % 2 == 0 && l.out_w % 2 == 0 && l.n % 32 == 0 &&
                         c.pool_next.H == l.out_h / 2 && c.pool_next.W == l.out_w / 2 && vec16_view(c.pool_next, 1)))
        return 0;
    return 1;
}

TcPlanPtr tc_make_plan(const TcConv &c) {
    const Layer &l = *c.l;
    if (!tc_conv_supported(c)) fatal_throw("tc plan: convolution not supported by the tensor-core kernels");
    TcPlanPtr plan(new TcPlan());
    TcParams &p = plan->p;
    const bool reg = c.kind == TC_BF16 && c.out_bf16;   // bf16 NHWC output: the register-accumulator kernel with its TMA epilogue
    const int sms = sm_count();
    plan_tiles(p, c, reg, sms);
    plan_epilogue(p, c, reg);
    plan_ring(p, reg);
    plan->smem = tc_smem_layout(p, reg);
    p.dbg = c.sw.dbg;
    snprintf(plan->desc, sizeof(plan->desc), "%dx%dx%d -> n%d k%d s%d%s", l.c, l.h, l.w, l.n, l.size, l.stride, reg ? " reg" : "");
    encode_maps(*plan, c, reg);
    plan->grid = std::min(p.num_work, grid_cap(sms, c.sw.grid));
    // the integer kinds compile EPI 2, the float kinds EPI 0; YB_TC_STATS runs the role-counter instantiations
    const bool st = c.sw.stats;
    plan->reg = reg;
    if (reg) plan->kernel = st ? k_conv_tc_reg<true> : k_conv_tc_reg<false>;
    else if (is_integer(c.kind)) plan->kernel = st ? k_conv_tc<true, 2> : k_conv_tc<false, 2>;
    else plan->kernel = st ? k_conv_tc<true, 0> : k_conv_tc<false, 0>;
    // the largest any plan may ask for: other plans of the same kernel rely on it
    if (cudaFuncSetAttribute((const void *)plan->kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
        fatal_throw("cudaFuncSetAttribute(k_conv_tc) failed");
    if (st) {
        plan->stats.ensure(TC_NSTATS * (size_t)plan->grid);
        p.stats = plan->stats.get();
        cudaMemset(p.stats, 0, sizeof(unsigned long long) * TC_NSTATS * plan->grid);
    }
    return plan;
}

struct StemPlan { StemTcP p; int grid; bool s2; };   // s2: k_stem_s2_tc (stem + layer 1)
int tc_stem_supported(const Layer &l, const TV &out) {
    return l.c == 3 && l.size == 3 && l.stride == 1 && l.pad == 1 && (l.n == 16 || l.n == 32) &&
           (l.activation == YB_LEAKY || l.activation == YB_LINEAR) && out.base && vec16_view(out, 2);
}
// d_w: device buffer of 32*32 bf16 ([filter][k], k = (ky,kx,c), zero padded), d_bias: device f32[>= n]
StemPlanPtr tc_stem_make_plan(const Layer &l, const TV &out, const void *d_w, const float *d_bias) {
    StemPlanPtr sp(new StemPlan());
    StemTcP &p = sp->p;
    p.out = out.base; p.out_ldc = out.ldc; p.w = reinterpret_cast<const __nv_bfloat16 *>(d_w); p.bias = d_bias;
    p.N = out.N; p.H = l.h; p.W = l.w; p.OHp = out.Hp; p.OWp = out.Wp; p.nf = l.n; p.act = l.activation;
    p.npix = (long)out.N * l.h * l.w;
    if (p.npix >= (1L << 31) - 256) fatal_throw("stem plan: more than 2^31 pixels per batch");
    p.ntiles = (int)((p.npix + 127) / 128);
    sp->grid = std::min(p.ntiles, sm_count() * 8);
    return sp;
}
int tc_stem_s2_supported(const Layer &l0, const Layer &l1, const TV &out1) {
    return l0.n == 32 && l1.c == 32 && l1.n == 64 && l1.size == 3 && l1.stride == 2 && l1.pad == 1 && l1.h == l0.h && l1.w == l0.w &&
           l0.h % 2 == 0 && l0.w % 2 == 0 && (l1.activation == YB_LEAKY || l1.activation == YB_LINEAR) && out1.base && out1.P == 1 &&
           out1.H == l0.h / 2 && out1.W == l0.w / 2 && vec16_view(out1, 2);
}
// d_w1: layer 1's bf16 [64][9 * 32] filter matrix (K ordered (ky, kx, c)), d_bias1: its f32 bias
StemPlanPtr tc_stem_s2_make_plan(const Layer &l0, const Layer &l1, const TV &out1, const void *d_w, const float *d_bias,
                                 const void *d_w1, const float *d_bias1, int max_grid) {
    StemPlanPtr sp(new StemPlan());
    sp->s2 = true;
    StemTcP &p = sp->p;
    p.out = out1.base; p.out_ldc = out1.ldc; p.w = reinterpret_cast<const __nv_bfloat16 *>(d_w); p.bias = d_bias;
    p.N = out1.N; p.H = l0.h; p.W = l0.w; p.OHp = out1.Hp; p.OWp = out1.Wp; p.nf = l0.n; p.act = l0.activation;
    p.w1 = reinterpret_cast<const __nv_bfloat16 *>(d_w1); p.bias1 = d_bias1; p.act1 = l1.activation;
    p.OH = out1.H; p.OW = out1.W;
    p.xt = (p.OW + S2_TW - 1) / S2_TW; p.yt = (p.OH + S2_TH - 1) / S2_TH;
    const long ntiles = (long)p.N * p.xt * p.yt;
    if (ntiles >= INT_MAX) fatal_throw("stem plan: too many tiles");
    p.ntiles = (int)ntiles;
    sp->grid = std::min(p.ntiles, grid_cap(2 * sm_count(), max_grid));
    for (const void *f : {(const void *)k_stem_s2_tc<false>, (const void *)k_stem_s2_tc<true>}) {
        if (cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S2_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, 100) != cudaSuccess)
            fatal_throw("cudaFuncSetAttribute(k_stem_s2_tc) failed");
    }
    return sp;
}
void tc_stem_launch(const StemPlan &sp, const float *d_in_nchw, cudaStream_t s) {
    StemTcP p = sp.p;
    p.in = d_in_nchw;
    if (sp.s2) k_stem_s2_tc<false><<<sp.grid, 256, S2_SMEM, s>>>(p);
    else k_stem_tc<false><<<sp.grid, 128, 0, s>>>(p);
}
// 8-bit HWC frames of exactly the network size (3 channels): no planar-float staging
void tc_stem_launch_u8(const StemPlan &sp, const unsigned char *d_in_hwc, cudaStream_t s) {
    StemTcP p = sp.p;
    p.in8 = d_in_hwc;
    if (sp.s2) k_stem_s2_tc<true><<<sp.grid, 256, S2_SMEM, s>>>(p);
    else k_stem_tc<true><<<sp.grid, 128, 0, s>>>(p);
}

namespace {
int copy_fields(const int (&f)[TC_PLAN_NFIELDS], int *fields, int n) {
    const int k = std::max(0, std::min(n, (int)TC_PLAN_NFIELDS));
    for (int i = 0; i < k; ++i) fields[i] = f[i];
    return k;
}
}  // namespace

int tc_plan_fields(const TcPlan &plan, int *fields, int n) {
    const TcParams &p = plan.p;
    const int f[TC_PLAN_NFIELDS] = {plan.reg ? TC_PLAN_CONV_REG : TC_PLAN_CONV, p.kind, p.TW, p.TH, p.BN, p.BK,
                                    p.nt, p.bstat, p.stages, p.sps, plan.grid, p.num_work, p.tma_epi, p.jshift,
                                    p.out ? (int)p.out_ldc : 0};
    return copy_fields(f, fields, n);
}

int tc_stem_plan_fields(const StemPlan &sp, int *fields, int n) {
    const int f[TC_PLAN_NFIELDS] = {sp.s2 ? TC_PLAN_STEM_S2 : TC_PLAN_STEM, TC_BF16, sp.s2 ? S2_TW : -1, sp.s2 ? S2_TH : -1,
                                    sp.s2 ? 64 : -1, -1, -1, -1, -1, -1, sp.grid, sp.p.ntiles, -1, -1, (int)sp.p.out_ldc};
    return copy_fields(f, fields, n);
}

void tc_launch(const TcPlan &P, cudaStream_t s) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)P.grid); cfg.blockDim = dim3((unsigned)(P.reg ? TCR_THREADS : TC_THREADS));
    cfg.dynamicSmemBytes = P.smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];   // programmatic dependent launch: this kernel's prologue runs while the previous kernel drains
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, P.kernel, P.tmA, P.tmB, P.tmO, P.tmO1, P.tmR, P.p);
}

void TcPlanDelete::operator()(TcPlan *plan) const {
    if (plan->p.stats) {   // diagnostic dump: mean cycles per CTA of the LAST launch
        std::vector<unsigned long long> h(TC_NSTATS * (size_t)plan->grid);
        cudaDeviceSynchronize();
        cudaMemcpy(h.data(), plan->p.stats, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
        double m[TC_NSTATS] = {0};
        for (int b = 0; b < plan->grid; ++b) for (int k = 0; k < TC_NSTATS; ++k) m[k] += (double)h[TC_NSTATS * b + k] / plan->grid;
        fprintf(stderr, "TCSTATS %-28s tiles/cta %.1f kb %d sps %d BN %d | producer: wait_empty %.0f tma_issue %.0f total %.0f | ",
                plan->desc, (double)plan->p.num_work / plan->grid, plan->p.kblocks, plan->p.sps, plan->p.BN,
                m[STAT_PROD_WAIT_EMPTY], m[STAT_PROD_TMA_ISSUE], m[STAT_PROD_TOTAL]);
        if (plan->reg)   // k_conv_tc_reg: the consumers' wait on stg_ready (first work item apart) and the store warps
            fprintf(stderr, "consumers: wait_full %.0f wait_ready %.0f (first item %.0f) total %.0f | store: wait_full %.0f wait_read %.0f\n",
                    m[STAT_CONS_WAIT_FULL], m[STAT_CONS_WAIT_READY], m[STAT_CONS_FIRST_READY], m[STAT_CONS_TOTAL],
                    m[STAT_STORE_WAIT_FULL], m[STAT_STORE_WAIT_READ]);
        else fprintf(stderr, "consumers: wait_full %.0f total %.0f\n", m[STAT_CONS_WAIT_FULL], m[STAT_CONS_TOTAL]);
    }
    delete plan;
}
void TcPlanDelete::operator()(StemPlan *plan) const { delete plan; }

}  // namespace yb
