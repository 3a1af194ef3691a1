// yb_kernels.cuh -- CUDA-core (SIMT) kernels of the engine: layout converters, the generic FP32 / XNOR / INT8
// convolution and all small layers.  sm_90a only.  The tensor-core (wgmma) convolutions live in
// yb_conv_tc.cuh.
//
// Device activation layout ("padded NHWC"): element (n, y, x, c) of a tensor with logical dims N,H,W,C lives at
//     base + (((n*(H+2P) + y+P) * (W+2P) + x+P) * ldc + c) * sizeof(T)
// with a P=1 pixel border that is zero-filled once at allocation and never written -- 3x3/pad-1 convolutions
// (and their TMA loads) read the border instead of bounds-checking.  ldc >= C lets a tensor be a channel slice
// of a wider concat buffer (route layers become aliasing).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/yolo2_light_b200.h"   // YB_FRAME_*
#include "yb_device.cuh"

namespace yb {

// ------------------------------------------------------------------------------------------------------
// input: NCHW f32 (host contract, reference additionally.c:3093-3103) -> padded NHWC
// ------------------------------------------------------------------------------------------------------
template <typename TOut>
__global__ void k_input_nchw_to_nhwc(const float *__restrict__ in, TV out) {
    const long total = (long)out.N * out.H * out.W;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < total; p += (long)gridDim.x * blockDim.x) {
        const int x = (int)(p % out.W);
        const int y = (int)((p / out.W) % out.H);
        const int n = (int)(p / ((long)out.W * out.H));
        TOut *o = tv_px<TOut>(out, n, y, x);
        const float *src = in + ((size_t)n * out.C * out.H + y) * out.W + x;
        for (int c = 0; c < out.C; ++c) o[c] = from_f32<TOut>(src[(size_t)c * out.H * out.W]);
    }
}

// any padded-NHWC activation -> NCHW f32 (diagnostic fetch)
template <typename TIn>
__global__ void k_nhwc_to_nchw_f32(TV in, float *__restrict__ out) {
    const long total = (long)in.N * in.C * in.H * in.W;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % in.W);
        const int y = (int)((i / in.W) % in.H);
        const int c = (int)((i / ((long)in.W * in.H)) % in.C);
        const int n = (int)(i / ((long)in.W * in.H * in.C));
        out[i] = to_f32(tv_px<TIn>(in, n, y, x)[c]);
    }
}

// ------------------------------------------------------------------------------------------------------
// input pipeline of the reference app on the device (SURVEY 8f row 2): a batch of u8 HWC frames (what stbi_load
// returns), each of its own size -> planar float /255. (load_image_stb, additionally.c:3080-3103) -> resize_image's
// two-pass bilinear to the network size (additionally.c:3021-3064).  Every product and sum is rounded to float exactly
// where the reference rounds (no FMA contraction), so the result is bit-identical to the reference's scalar build.
//
// One block = RS_ROWS output rows of one image (grid.y = image).  Per output row it stages the byte span of the one or
// two source rows that row reads into shared memory with 16-byte loads, then every thread makes one output pixel for all
// c channels (the x-interpolation is computed once per pixel, not once per channel) and the planes are written with
// coalesced stores.  The /255. conversion is a 256-entry table (`unit`, made on the host with load_image_stb's own double
// divide) read into shared memory: no divide in the kernel.  A span wider than RS_SPAN bytes (frames several thousand pixels wide) is read from global memory
// directly; both ways give the same values.
//
// The source format F is a template parameter (YB_FRAME_*, include/yolo2_light_b200.h); every image carries its own
// pointer(s) and row pitch.  Host frames are staged as packed RGB (c = net.c bytes per pixel).  For the caller's device
// frames (c = 3): BGR swaps R and B when a byte is read; planar stages the three plane spans; NV12 stages the Y span and
// the chroma span of each source row and converts them to RGB bytes in shared memory, once per source pixel, with
// BT.601 limited-range fixed-point arithmetic (OpenCV's COLOR_YUV2RGB_NV12 constants).  The interpolation that follows
// is the same for every format, so a device frame gives bit-for-bit what its RGB equivalent gives through the host path.
//
// Letterboxing (darknet's letterbox_image: resize to the letterbox size, fill_image(.5), embed_image): each image resizes
// to its target nw x nh (ImageGeo), placed at (dx, dy) of the out_w x out_h input.  Rows outside [dy, dy + nh) are 0.5 in
// every channel and stage nothing; inside, the columns outside [dx, dx + nw) are 0.5.  Without letterboxing the target is
// the whole input at (0, 0), and the kernel computes exactly the stretched resize.
// ------------------------------------------------------------------------------------------------------
struct ImageGeo {               // one image of a batch (device table, uploaded with the frames)
    const unsigned char *src;   // RGB / BGR: first pixel; planar: the R plane; NV12: the Y plane
    const unsigned char *chroma;   // NV12: the interleaved U, V plane (h / 2 rows, same pitch as Y)
    long long plane;            // planar: bytes from one plane to the next
    int pitch;                  // bytes from one row to the next
    int w, h;                   // frame size
    int new_w, new_h;           // correct_yolo_boxes' embedded size (the network size unless `letter`)
    int nw, nh, dx, dy;         // resize target and its offset in the network input: the network size at (0, 0), or with
                                // letterboxing on the letterbox size at ((W - nw) / 2, (H - nh) / 2)
    float w_scale, h_scale;     // resize_image's (w - 1) / (nw - 1), (h - 1) / (nh - 1): IEEE float divides, made
                                // on the host so that the kernel has no divide
};

constexpr int RS_THREADS = 256, RS_ROWS = 4, RS_COLS = 1024, RS_SPAN = 12288, RS_PLANE = RS_SPAN / 3;
static_assert(RS_THREADS == 256, "one thread per entry of the /255. table");

// frame bytes [p, p + len) -> smem; returns the smem offset of byte p.  The 16-byte vectors are aligned in memory: the ones
// wholly inside the span are read with one 16-byte load, the (at most two) that straddle its ends byte by byte, and only
// the span's own bytes of them.  So no byte outside [p, p + len) is read, and a frame may start at any address and end on
// the last byte of its allocation.  The smem bytes of a straddling vector that lie outside the span stay unwritten; nothing
// reads them.
__device__ __forceinline__ int rs_stage(const unsigned char *__restrict__ p, int len, uint4 *smem) {
    const uintptr_t s = reinterpret_cast<uintptr_t>(p), e = s + (uintptr_t)len, a = s & ~(uintptr_t)15;
    const int nvec = (int)((e - a + 15) >> 4);
    for (int i = threadIdx.x; i < nvec; i += RS_THREADS) {
        const uintptr_t v = a + 16 * (uintptr_t)i;
        if (v >= s && v + 16 <= e) {
            smem[i] = __ldg(reinterpret_cast<const uint4 *>(v));
        } else {
            unsigned char *d = reinterpret_cast<unsigned char *>(smem + i);
            for (int j = 0; j < 16; ++j)
                if (v + j >= s && v + j < e) d[j] = __ldg(reinterpret_cast<const unsigned char *>(v + j));
        }
    }
    return (int)(s - a);
}

// BT.601 limited range -> 8-bit RGB, OpenCV's fixed-point form (cvtColor COLOR_YUV2RGB_NV12).  Every intermediate fits in
// an int: |yy| + |1673527 * v| + 2^19 < 2^30.
__device__ __forceinline__ int nv12_clamp(int x) { return min(255, max(0, x)); }
__device__ __forceinline__ int nv12_ch(int Y, int U, int V, int k) {
    const int yy = max(0, Y - 16) * 1220542 + (1 << 19), u = U - 128, v = V - 128;
    return nv12_clamp((k == 0 ? yy + 1673527 * v : k == 1 ? yy - 852492 * v - 409993 * u : yy + 2116026 * u) >> 20);
}

// 8-bit RGB -> BT.601 limited-range Y, U, V, integer form with 8 fractional bits (the direction opposite to nv12_ch; the
// rule of include/yolo2_light_b200.h, YB_FRAME_NV12).  >> is an arithmetic shift; the results lie in 16..235 / 16..240.
__device__ __forceinline__ void rgb_to_yuv601(int R, int G, int B, unsigned char *yuv) {
    yuv[0] = (unsigned char)(((66 * R + 129 * G + 25 * B + 128) >> 8) + 16);
    yuv[1] = (unsigned char)(((-38 * R - 74 * G + 112 * B + 128) >> 8) + 128);
    yuv[2] = (unsigned char)(((112 * R - 94 * G - 18 * B + 128) >> 8) + 128);
}

struct RsSrc {                  // one source row of a chunk; index 0 is column `lo`
    const unsigned char *q[3];  // RGB / BGR / NV12 staged (converted): q[0]; planar: the three planes; NV12 read
                                // directly: the Y row (q[0]) and the chroma row from column lo & ~1 (q[1])
    int odd;                    // NV12 read directly: lo & 1
};

// byte of channel k of pixel lo + x
template <int F>
__device__ __forceinline__ int rs_px(const RsSrc &s, bool staged, int c, int x, int k) {
    if (F == YB_FRAME_RGB) return s.q[0][x * c + k];
    if (F == YB_FRAME_BGR) return s.q[0][x * 3 + 2 - k];
    if (F == YB_FRAME_RGB_PLANAR) return s.q[k][x];
    if (staged) return s.q[0][x * 3 + k];
    const int uv = (x + s.odd) & ~1;
    return nv12_ch(__ldg(s.q[0] + x), __ldg(s.q[1] + uv), __ldg(s.q[1] + uv + 1), k);
}

template <int F>
static __global__ void __launch_bounds__(RS_THREADS) k_resize_frames(const ImageGeo *__restrict__ geo,
                                                                      const float *__restrict__ unit_tab, int c_,
                                                                      float *__restrict__ dst, int out_w, int out_h) {
    constexpr bool NV12 = F == YB_FRAME_NV12;
    __shared__ uint4 stage[2][RS_SPAN / 16];
    __shared__ uint4 raw[NV12 ? 2 : 1][2][NV12 ? (RS_PLANE + 32) / 16 : 1];   // NV12: the Y and chroma spans of each row
    __shared__ float unit[256];
    unit[threadIdx.x] = unit_tab[threadIdx.x];   // RS_THREADS == 256; published by the first barrier
    const int c = F == YB_FRAME_RGB ? c_ : 3;
    const int n = blockIdx.y;
    const ImageGeo g = geo[n];
    const int w = g.w, h = g.h, tw = g.nw, th = g.nh;   // frame and resize target
    float *out = dst + (size_t)n * c * out_h * out_w;
    const size_t plane = (size_t)out_h * out_w;
    const bool same = (tw == w && th == h);
    const float w_scale = g.w_scale, h_scale = g.h_scale;
    const int r0 = blockIdx.x * RS_ROWS, r_end = min(out_h, r0 + RS_ROWS);
    // letterbox: 0.5 in the bands above and below the image and in the columns left and right of it (none when stretched)
    for (int r = r0; r < r_end; ++r) {
        const bool band = r < g.dy || r >= g.dy + th;
        const int nfill = band ? out_w : out_w - tw;
        for (int cc = threadIdx.x; cc < nfill; cc += RS_THREADS) {
            const int x = band || cc < g.dx ? cc : cc + tw;
#pragma unroll 1
            for (int k = 0; k < c; ++k) out[k * plane + (size_t)r * out_w + x] = 0.5f;
        }
    }
    for (int r = max(r0, g.dy), r1 = min(r_end, g.dy + th); r < r1; ++r) {   // the image's rows
        const int tr = r - g.dy;                            // row of the target
        float *orow = out + (size_t)r * out_w + g.dx;
        int iy = tr;
        float dy = 0.f;
        bool two = false;
        if (!same) {
            const float sy = __fmul_rn((float)tr, h_scale);
            iy = (int)sy;
            dy = __fsub_rn(sy, (float)iy);
            two = !(tr == th - 1 || h == 1);
        }
        for (int cc0 = 0; cc0 < tw; cc0 += RS_COLS) {
            const int cc1 = min(tw, cc0 + RS_COLS) - 1;         // last column of this chunk
            // source columns the chunk reads: ix(cc0) .. ix(cc1) + 1, or the last column
            int lo, hi;
            if (same) { lo = cc0; hi = cc1; }
            else if (w == 1) { lo = hi = 0; }
            else {
                lo = cc0 == tw - 1 ? w - 1 : (int)__fmul_rn((float)cc0, w_scale);
                hi = cc1 == tw - 1 ? w - 1 : (int)__fmul_rn((float)cc1, w_scale) + 1;
            }
            const int npix = hi - lo + 1, len = npix * c;
            const unsigned char *row[2] = {g.src + (size_t)iy * g.pitch, g.src + (size_t)(iy + two) * g.pitch};
            bool staged;
            if (F == YB_FRAME_RGB || F == YB_FRAME_BGR)
                staged = (int)(reinterpret_cast<uintptr_t>(row[0] + lo * c) & 15) + len <= RS_SPAN &&
                         (!two || (int)(reinterpret_cast<uintptr_t>(row[1] + lo * c) & 15) + len <= RS_SPAN);
            else   // per plane (planar) or per staged span (NV12: Y, and chroma of at most npix + 2 bytes in RS_PLANE + 32)
                staged = npix + 15 <= RS_PLANE;
            RsSrc src[2];                       // rows iy / iy + 1 (the same row when !two)
            int oy[2] = {0, 0}, ouv[2] = {0, 0};   // NV12 staged: smem offsets of the Y and chroma spans in raw[t]
            __syncthreads();                    // the previous chunk is done with the staging buffers
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                if (t && !two) break;
                unsigned char *s = reinterpret_cast<unsigned char *>(stage[t]);
                if (F == YB_FRAME_RGB || F == YB_FRAME_BGR) {
                    src[t].q[0] = staged ? s + rs_stage(row[t] + lo * c, len, stage[t]) : row[t] + lo * c;
                } else if (F == YB_FRAME_RGB_PLANAR) {
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        const unsigned char *p = row[t] + k * g.plane + lo;
                        src[t].q[k] = staged ? s + k * RS_PLANE + rs_stage(p, npix, stage[t] + k * (RS_PLANE / 16)) : p;
                    }
                } else {
                    const unsigned char *yr = row[t] + lo, *cr = g.chroma + (size_t)((iy + t) >> 1) * g.pitch + (lo & ~1);
                    if (staged) {
                        src[t].q[0] = s;
                        oy[t] = rs_stage(yr, npix, raw[t][0]);
                        ouv[t] = rs_stage(cr, ((hi | 1) - (lo & ~1)) + 1, raw[t][1]);
                    } else {
                        src[t].q[0] = yr; src[t].q[1] = cr;
                    }
                    src[t].odd = lo & 1;
                }
            }
            if (!two) src[1] = src[0];
            if (staged) __syncthreads();
            if (NV12 && staged) {               // staged Y / chroma -> RGB bytes, once per source pixel
#pragma unroll
                for (int t = 0; t < 2; ++t) {
                    if (t && !two) break;
                    unsigned char *d = reinterpret_cast<unsigned char *>(stage[t]);
                    const unsigned char *ys = reinterpret_cast<const unsigned char *>(raw[t][0]) + oy[t];
                    const unsigned char *uvs = reinterpret_cast<const unsigned char *>(raw[t][1]) + ouv[t];
                    for (int x = threadIdx.x; x < npix; x += RS_THREADS) {
                        const int Y = ys[x], uv = (x + (lo & 1)) & ~1, U = uvs[uv], V = uvs[uv + 1];
                        for (int k = 0; k < 3; ++k) d[x * 3 + k] = (unsigned char)nv12_ch(Y, U, V, k);
                    }
                }
                __syncthreads();
            }
            const RsSrc &p0 = src[0], &p1 = src[1];
            for (int cc = cc0 + threadIdx.x; cc <= cc1; cc += RS_THREADS) {
                float *o = orow + cc;
                if (same) {
                    for (int k = 0; k < c; ++k) o[k * plane] = unit[rs_px<F>(p0, staged, c, cc - lo, k)];
                    continue;
                }
                // the reference's `part` image at (cc, row): the last column (or a 1-pixel-wide frame) copies the edge
                const bool edge = cc == tw - 1 || w == 1;
                int xa = w - 1 - lo;
                float dx = 0.f;
                if (!edge) {
                    const float sx = __fmul_rn((float)cc, w_scale);
                    const int ix = (int)sx;
                    dx = __fsub_rn(sx, (float)ix);
                    xa = ix - lo;
                }
                const float ndx = __fsub_rn(1.f, dx), ndy = __fsub_rn(1.f, dy);
                for (int k = 0; k < c; ++k) {
                    float part0 = unit[rs_px<F>(p0, staged, c, xa, k)];
                    if (!edge) part0 = __fadd_rn(__fmul_rn(ndx, part0), __fmul_rn(dx, unit[rs_px<F>(p0, staged, c, xa + 1, k)]));
                    float val = __fmul_rn(ndy, part0);
                    if (two) {
                        float part1 = unit[rs_px<F>(p1, staged, c, xa, k)];
                        if (!edge) part1 = __fadd_rn(__fmul_rn(ndx, part1), __fmul_rn(dx, unit[rs_px<F>(p1, staged, c, xa + 1, k)]));
                        val = __fadd_rn(val, __fmul_rn(dy, part1));
                    }
                    o[k * plane] = val;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// The convolutions on CUDA cores: one implicit GEMM, 64 pixels x 64 filters per CTA, 256 threads, a 4x4 accumulator tile per
// thread, K streamed through shared memory.  Taps outside the image read a zero element.  A policy V gives the K element, its
// loaders, the multiply-accumulate and the epilogue:
//   SimtF32<TIn, TOut, TRes, EXACT>  f32 values: forward_convolutional_layer_cpu FP32 branch (reference
//       yolov2_forward_network.c:204-261), out = act(sum_{c,ky,kx} w*in + bias) with zero padding; optional fused shortcut
//       (reference :443-449), out = act2(act(..) + residual).  Validation precision (YB_PREC_FP32), the FP32 layers of XNOR /
//       INT8 networks, the bf16 layers the tensor cores refuse, and the XNOR layers of the float-GEMM fallback.
//   SimtPopc<A>  words of 32 sign bits (reference yolov2_forward_network.c:116-203): count = sum popc(~(a ^ w)) - (pad bits),
//       out = IntEpi<A>::finish(2*count - K, mean[f], bias[f]).  SimtXnor (AR_XNOR): the XNOR layers off the s8 wgmma with more
//       than 2 words per tap; SimtXnorGpu (AR_XNOR_GPU): the XNOR layers with c % 32 == 0 of the GPU XNOR rule, of any size,
//       stride and pad, off the s8 wgmma and the small-K kernel.
//   SimtDp4a<A>  words of 4 s8 values: acc32 = sum xq*wq (dp4a, exact), out = IntEpi<A>::finish(acc32, ..).  SimtInt8 (AR_INT8,
//       reference yolov2_forward_network_quantized.c:527-631) and SimtInt8Gpu (AR_INT8_GPU): the INT8 layers the s8 wgmma tile
//       refuses; SimtPm1zGpu (AR_PM1Z_GPU), over +-1 bytes (SIDE_PM1Z_S8, +-1 weights): the XNOR layers below 32 channels of the
//       GPU XNOR rule that the s8 wgmma tile does not take.  Out-of-image taps read 0.
// The integer inputs are written by k_int_input or by the fused kernels in front of the convolution.
// ------------------------------------------------------------------------------------------------------
struct SimtP {
    TV in, out, res;           // in: f32 / bf16 activations or the integer side input; res.base == nullptr: no residual
    const void *w;             // f32: [K][ldw], ldw = filters rounded up to 64; integer: [filters rounded up to 64][K] words
    const float *bias;
    const float *mean;         // XNOR
    float alpha1;              // INT8: ALPHA1 of the rule's epilogue
    int n;                     // filters
    int ldw;
    int size, stride, pad;
    int act, act2;
    int K;                     // GEMM depth: size*size*C f32 values, or size*size*CW words ordered (ky, kx, word)
    int CW;                    // integer: words per input pixel
    int bits, padbits;         // XNOR: true bit count size*size*C, and (CW*32 - C) * size*size
    long M;                    // N*out_h*out_w
    int32_t *counts;           // integer: optional raw popcounts / s32 accumulators, NCHW (tests)
};

// the image and window origin of an A-loader's output pixel; valid = false past the last pixel
struct SimtRow {
    bool valid;
    int n, iy0, ix0;
};

// (iy, ix): the input pixel of row r under tap t; false where it falls outside the image
__device__ __forceinline__ bool simt_tap(const SimtP &p, const SimtRow &r, int tap, int &iy, int &ix) {
    const int ky = tap / p.size, kx = tap - ky * p.size;
    iy = r.iy0 + ky;
    ix = r.ix0 + kx;
    return iy >= 0 && iy < p.in.H && ix >= 0 && ix < p.in.W;
}

// EXACT = true (f32 activations: the exact nets and YB_PREC_FP32): K runs in the reference's own order (c, ky, kx) --
// weights [K][ldw] stored in that order -- and every product and sum is rounded separately (__fmul_rn / __fadd_rn), i.e.
// gemm_nn's `C[j] += A_PART * B[k][j]` of the scalar build (additionally.c:1272-1286): the result is bit-identical to the
// reference, so a last-bit difference can never flip `x > 0` / `(int16)(x * m)` in a following integer layer.  Otherwise K
// is ordered (ky, kx, c) and summed with fmaf.
template <typename TIn, typename TOut_, typename TRes_, bool EXACT = false>
struct SimtF32 {
    using E = float;
    using Acc = float;
    using TOut = TOut_;
    using TRes = TRes_;
    static constexpr int BK = 16, SKEW = 4;
    static constexpr bool RAW = false;
    // A: pixel tid/4, 4 consecutive k from (tid%4)*4; B: k row tid/16, 4 consecutive filters (tid%16)*4 in one float4
    static __device__ __forceinline__ void load(const SimtP &p, const SimtRow &r, E (*As)[64 + SKEW], E (*Bs)[64 + SKEW], int k0,
                                                int n0) {
        const int tid = threadIdx.x, lp = tid >> 2, lk = (tid & 3) * 4;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int k = k0 + lk + q;
            float v = 0.f;
            if (r.valid && k < p.K) {
                const int taps = p.size * p.size, C = p.in.C;
                const int tap = EXACT ? k % taps : k / C, ch = EXACT ? k / taps : k - tap * C;
                int iy, ix;
                if (simt_tap(p, r, tap, iy, ix)) v = to_f32(tv_px<TIn>(p.in, r.n, iy, ix)[ch]);
            }
            As[lk + q][lp] = v;
        }
        const int bk = tid >> 4, bn = (tid & 15) * 4, k = k0 + bk;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < p.K) v = *reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(p.w) + (size_t)k * p.ldw + n0 + bn);
        Bs[bk][bn + 0] = v.x; Bs[bk][bn + 1] = v.y; Bs[bk][bn + 2] = v.z; Bs[bk][bn + 3] = v.w;
    }
    static __device__ __forceinline__ void mac(float &acc, float a, float b) {
        if constexpr (EXACT) acc = __fadd_rn(acc, __fmul_rn(b, a));
        else acc = fmaf(a, b, acc);
    }
    static __device__ __forceinline__ float finish(const SimtP &p, float acc, int f, const TRes *r) {
        float v = act_exact(__fadd_rn(acc, p.bias[f]), p.act);
        if (r) v = act_exact(__fadd_rn(v, to_f32(r[f])), p.act2);
        return v;
    }
};

// the integer policies' shared part: 64 rows x 8 words per operand, 2 words per thread -- A: pixel tid/4 of the side input
// (element type T), B: filter n0 + tid/4 of [ldn][K]; the K tail pads A with 0 and B with KPAD, which contribute nothing
template <typename T, uint32_t KPAD>
struct SimtWords {
    using E = uint32_t;
    using Acc = int;
    using TOut = float;
    using TRes = float;
    static constexpr int BK = 8, SKEW = 1;
    static constexpr bool RAW = true;
    static __device__ __forceinline__ void load(const SimtP &p, const SimtRow &r, E (*As)[64 + SKEW], E (*Bs)[64 + SKEW], int k0,
                                                int n0) {
        const int lr = threadIdx.x >> 2, lw = (threadIdx.x & 3) * 2;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int k = k0 + lw + q;
            uint32_t a = 0, b = KPAD;
            if (k < p.K) {
                const int tap = k / p.CW, wd = k - tap * p.CW;
                int iy, ix;
                if (r.valid && simt_tap(p, r, tap, iy, ix)) a = reinterpret_cast<const uint32_t *>(tv_px<T>(p.in, r.n, iy, ix))[wd];
                b = reinterpret_cast<const uint32_t *>(p.w)[(size_t)(n0 + lr) * p.K + k];
            }
            As[lw + q][lr] = a;
            Bs[lw + q][lr] = b;
        }
    }
};

// the integer policies' epilogue: IntEpi<A> on the signed result r of filter f
template <Arith A>
__device__ __forceinline__ float simt_int_finish(const SimtP &p, int r, int f) {
    return IntEpi<A>::finish(r, IntEpi<A>::MEAN ? p.mean[f] : p.alpha1, p.bias[f], p.act);
}

// xor + popc over sign words (AR_XNOR, AR_XNOR_GPU): r = 2*(count - padbits) - bits
template <Arith A>
struct SimtPopc : SimtWords<uint32_t, 0xffffffffu> {   // a ^ b all ones in the tail: xnor counts 0
    static __device__ __forceinline__ void mac(int &acc, uint32_t a, uint32_t b) { acc += __popc(~(a ^ b)); }
    static __device__ __forceinline__ int dot(const SimtP &p, int acc) { return 2 * (acc - p.padbits) - p.bits; }
    static __device__ __forceinline__ int raw(const SimtP &p, int acc) { return IntEpi<A>::raw(dot(p, acc), p.bits); }
    static __device__ __forceinline__ float finish(const SimtP &p, int acc, int f, const float *) { return simt_int_finish<A>(p, dot(p, acc), f); }
};

// dp4a over s8 or +-1 bytes (AR_INT8, AR_INT8_GPU, AR_PM1Z_GPU): r = the s32 accumulator
template <Arith A>
struct SimtDp4a : SimtWords<int8_t, 0u> {
    static __device__ __forceinline__ void mac(int &acc, uint32_t a, uint32_t b) { acc = __dp4a((int)a, (int)b, acc); }
    static __device__ __forceinline__ int raw(const SimtP &p, int acc) { return IntEpi<A>::raw(acc, p.bits); }
    static __device__ __forceinline__ float finish(const SimtP &p, int acc, int f, const float *) { return simt_int_finish<A>(p, acc, f); }
};

// the integer policies by the names their k_conv_simt instantiations carry (Network.op_kernels)
struct SimtXnor : SimtPopc<AR_XNOR> {};
struct SimtXnorGpu : SimtPopc<AR_XNOR_GPU> {};
struct SimtPm1zGpu : SimtDp4a<AR_PM1Z_GPU> {};
struct SimtInt8 : SimtDp4a<AR_INT8> {};
struct SimtInt8Gpu : SimtDp4a<AR_INT8_GPU> {};

template <typename V>
__global__ void __launch_bounds__(256) k_conv_simt(SimtP p) {
    constexpr int BM = 64, BN = 64;
    using E = typename V::E;
    __shared__ E As[V::BK][BM + V::SKEW];
    __shared__ E Bs[V::BK][BN + V::SKEW];
    const int tid = threadIdx.x;
    const long m0 = (long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int OH = p.out.H, OW = p.out.W;

    SimtRow row{m0 + (tid >> 2) < p.M, 0, 0, 0};   // A-load role: pixel tid/4
    if (row.valid) {
        const long m = m0 + (tid >> 2);
        const int ox = (int)(m % OW);
        const int oy = (int)((m / OW) % OH);
        row.n = (int)(m / ((long)OW * OH));
        row.iy0 = oy * p.stride - p.pad;
        row.ix0 = ox * p.stride - p.pad;
    }
    const int tx = tid & 15, ty = tid >> 4;   // compute role: pixels ty*4.., filters tx*4..
    typename V::Acc acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0;

    for (int k0 = 0; k0 < p.K; k0 += V::BK) {
        V::load(p, row, As, Bs, k0, n0);
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < V::BK; ++kk) {
            E a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) V::mac(acc[i][j], a[i], b[j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long m = m0 + ty * 4 + i;
        if (m >= p.M) continue;
        const int ox = (int)(m % OW);
        const int oy = (int)((m / OW) % OH);
        const int n = (int)(m / ((long)OW * OH));
        typename V::TOut *o = tv_px<typename V::TOut>(p.out, n, oy, ox);
        const typename V::TRes *r = p.res.base ? tv_px<typename V::TRes>(p.res, n, oy, ox) : nullptr;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int f = n0 + tx * 4 + j;
            if (f >= p.n) continue;
            if constexpr (V::RAW)
                if (p.counts) p.counts[(((size_t)n * p.n + f) * OH + oy) * OW + ox] = V::raw(p, acc[i][j]);
            o[f] = from_f32<typename V::TOut>(V::finish(p, acc[i][j], f, r));
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// stem convolution (network input, 3 channels): 3x3 / stride 1 / pad 1 straight from the caller's NCHW f32 image
// (reference input contract additionally.c:3093-3103) to padded-NHWC output -- fuses the layout conversion, so
// the image is read exactly once and no NHWC copy of it is ever written.  One thread per output pixel, all NF
// filters in registers, weights [27][NF] broadcast from shared memory.  Accumulation order (ky, kx, c) matches
// k_conv_simt.
// ------------------------------------------------------------------------------------------------------
template <int NF>
struct StemW {            // passed by value as a kernel parameter: lives in the constant bank, so every FFMA takes
    float w[27 * NF];     // its weight operand straight from c[][] -- no shared-memory traffic at all
    float b[NF];
};

// EXACT (f32 output = the exact nets): reference order (c, ky, kx) with separately rounded products and sums, see
// k_conv_simt -- the INT8 / XNOR layers behind the stem then see bit-identical inputs.
template <int NF, typename TOut, bool EXACT = false>
__global__ void __launch_bounds__(128) k_conv_stem(const float *__restrict__ in, TV out, const __grid_constant__ StemW<NF> sw,
                                                   int act, int H, int W) {
    const long total = (long)out.N * H * W;
    const long p = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (p >= total) return;
    const int x = (int)(p % W);
    const int y = (int)((p / W) % H);
    const int n = (int)(p / ((long)W * H));
    const float *img = in + (size_t)n * 3 * H * W;
    float acc[NF];
#pragma unroll
    for (int f = 0; f < NF; ++f) acc[f] = 0.f;
    if constexpr (EXACT) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = y + ky - 1;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int ix = x + kx - 1;
                    const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
                    const float v = ok ? __ldg(img + ((size_t)c * H + iy) * W + ix) : 0.f;
#pragma unroll
                    for (int f = 0; f < NF; ++f)
                        acc[f] = __fadd_rn(acc[f], __fmul_rn(sw.w[((ky * 3 + kx) * 3 + c) * NF + f], v));
                }
            }
    } else {
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int iy = y + ky - 1;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int ix = x + kx - 1;
            const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float v = ok ? __ldg(img + ((size_t)c * H + iy) * W + ix) : 0.f;
#pragma unroll
                for (int f = 0; f < NF; ++f) acc[f] = fmaf(v, sw.w[((ky * 3 + kx) * 3 + c) * NF + f], acc[f]);
            }
        }
    }
    }
    TOut *o = tv_px<TOut>(out, n, y, x);
    if constexpr (sizeof(TOut) == 2) {
        uint4 *op = reinterpret_cast<uint4 *>(o);     // 8 filters per store: the layer plan checks vec16_view(out, 2)
#pragma unroll
        for (int g = 0; g < NF / 8; ++g) {
            float t[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float a = acc[g * 8 + j] + sw.b[g * 8 + j];
                t[j] = (act == ACT_LEAKY) ? ((a > 0.f) ? a : 0.1f * a) : act_exact(a, act);
            }
            __nv_bfloat162 h0 = __floats2bfloat162_rn(t[0], t[1]), h1 = __floats2bfloat162_rn(t[2], t[3]);
            __nv_bfloat162 h2 = __floats2bfloat162_rn(t[4], t[5]), h3 = __floats2bfloat162_rn(t[6], t[7]);
            uint4 v;
            v.x = *reinterpret_cast<uint32_t *>(&h0); v.y = *reinterpret_cast<uint32_t *>(&h1);
            v.z = *reinterpret_cast<uint32_t *>(&h2); v.w = *reinterpret_cast<uint32_t *>(&h3);
            op[g] = v;
        }
    } else {
        float4 *op = reinterpret_cast<float4 *>(o);   // NF*4 bytes per pixel, 16-byte aligned: the layer plan checks vec16_view(out, 4)
#pragma unroll
        for (int g = 0; g < NF / 4; ++g)
            op[g] = make_float4(act_exact(__fadd_rn(acc[g * 4 + 0], sw.b[g * 4 + 0]), act), act_exact(__fadd_rn(acc[g * 4 + 1], sw.b[g * 4 + 1]), act),
                                act_exact(__fadd_rn(acc[g * 4 + 2], sw.b[g * 4 + 2]), act), act_exact(__fadd_rn(acc[g * 4 + 3], sw.b[g * 4 + 3]), act));
    }
}

// ------------------------------------------------------------------------------------------------------
// BIT1-XNOR path (reference yolov2_forward_network.c:116-203; SURVEY Appendix A).  The sign-bit and +-1 byte inputs of
// the XNOR convolutions are written by k_int_input (or by the fused kernels in front of them).
// ------------------------------------------------------------------------------------------------------
// binarize_cpu (additionally.c:128-134): x > 0 ? +1 : -1 as floats -- the input of the XNOR layers that take the reference's
// float-GEMM fallback (stride != 1 or pad != 1).  The zero border of the destination stays zero (im2col's padding value).
static __global__ void k_binarize_pm1(TV in, TV out) {
    const long total = (long)in.N * in.H * in.W * in.C;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % in.C);
        const long px = i / in.C;
        const int x = (int)(px % in.W), y = (int)((px / in.W) % in.H), n = (int)(px / ((long)in.W * in.H));
        tv_px<float>(out, n, y, x)[c] = tv_px<float>(in, n, y, x)[c] > 0.f ? 1.f : -1.f;
    }
}

struct XnorP {                // the small-K XNOR convolutions, 3x3 / stride 1 / pad 1
    TV bits;                  // input bits, C = words per pixel (CW)
    TV out;                   // f32
    const uint32_t *w;        // [ldn filters][9 taps][CW] sign bits
    const float *mean, *bias;
    int n;
    int K;                   // true bit count size*size*C
    int padbits;              // (CW*32 - C) * size*size
    int act;
    long M;
    int32_t *counts;          // optional raw popcounts, NCHW (tests)
};

// The same convolution with the following 2x2 / stride-2 max-pool and the next XNOR layer's input conversion fused in: one thread
// per POOLED pixel computes the four popcount outputs of its window for every filter, takes the reference's max (max-pool
// semantics: elements outside the image are skipped) and writes only the sign the next layer would have extracted, in its side
// format F: SIDE_PM1_S8 (next layer runs as +-1 on the s8 wgmma) or SIDE_BITS (next layer on the popcount kernels).  The f32
// activation and the pooled f32 tensor are never written.  Bit-identical to conv -> max-pool -> k_int_input.  A: AR_XNOR or
// AR_XNOR_GPU, whose IntEpi finishes each dot.
template <int CW, SideFmt F, Arith A>
__device__ __forceinline__ void xnor_smallk_pool(const XnorP &p, const TV &q) {
    extern __shared__ uint32_t wsm[];            // [n][9*CW]
    constexpr int KW = 9 * CW;
    for (int i = threadIdx.x; i < p.n * KW; i += blockDim.x) wsm[i] = p.w[i];
    __syncthreads();
    const int H = p.out.H, W = p.out.W, PH = q.H, PW = q.W;
    const long m = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (m >= (long)q.N * PH * PW) return;
    const int px = (int)(m % PW), py = (int)((m / PW) % PH), n = (int)(m / ((long)PW * PH));
    uint32_t a[16 * CW];                          // 4x4 window of input words around the 2x2 outputs
#pragma unroll
    for (int t = 0; t < 16; ++t) {
        const int iy = 2 * py + t / 4 - 1, ix = 2 * px + t % 4 - 1;
        const bool in = iy >= -1 && iy <= H && ix >= -1 && ix <= W;      // the 1-pixel border exists in memory (words 0 == -1)
        const uint32_t *src = tv_px<uint32_t>(p.bits, n, in ? iy : -1, in ? ix : -1);
#pragma unroll
        for (int c = 0; c < CW; ++c) a[t * CW + c] = in ? src[c] : 0u;
    }
    uint32_t word = 0;
    for (int f = 0; f < p.n; ++f) {
        const uint32_t *wf = wsm + f * KW;
        float mx = -3.402823466e+38f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {             // window order of the reference: rows, then columns
            const int dy = k >> 1, dx = k & 1;
            if (2 * py + dy >= H || 2 * px + dx >= W) continue;
            int cnt = 0;
#pragma unroll
            for (int t = 0; t < 9; ++t)
#pragma unroll
                for (int c = 0; c < CW; ++c) cnt += __popc(~(a[((t / 3 + dy) * 4 + t % 3 + dx) * CW + c] ^ wf[t * CW + c]));
            const int dot = 2 * (cnt - p.padbits) - p.K;
            const float v = IntEpi<A>::finish(dot, p.mean[f], p.bias[f], p.act);
            mx = v > mx ? v : mx;
        }
        // one store per word (+-1 bytes: the filter count of an XNOR layer feeding the tensor-core path is a multiple of 16)
        constexpr int V = side_per_word(F);
        word |= side_place<F>(side_code<F>(mx, 0.f), f % V);
        if (f % V == V - 1 || f + 1 == p.n) { side_px<F>(q, n, py, px)[f / V] = word; word = 0; }
    }
}

// XNOR convolution for small K (one or two words per tap): one thread per output pixel keeps its 9 x CW input
// words in registers and walks all filters, whose sign words sit in shared memory (broadcast reads).  Whole groups of 4
// filters are stored as one float4: the output must be a vec16_view (16-byte aligned pixels), which the layer plan checks.  A: as
// in xnor_smallk_pool.
template <int CW, Arith A>
__device__ __forceinline__ void xnor_smallk(const XnorP &p) {
    extern __shared__ uint32_t wsm[];            // [n][9*CW]
    constexpr int KW = 9 * CW;
    for (int i = threadIdx.x; i < p.n * KW; i += blockDim.x) wsm[i] = p.w[i];
    __syncthreads();
    const int H = p.out.H, W = p.out.W;
    const long m = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (m >= p.M) return;
    const int x = (int)(m % W);
    const int y = (int)((m / W) % H);
    const int n = (int)(m / ((long)W * H));
    uint32_t a[KW];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
        const uint32_t *src = tv_px<uint32_t>(p.bits, n, y + t / 3 - 1, x + t % 3 - 1);   // border words are 0 (== -1)
#pragma unroll
        for (int c = 0; c < CW; ++c) a[t * CW + c] = src[c];
    }
    float *o = tv_px<float>(p.out, n, y, x);
    for (int f0 = 0; f0 < p.n; f0 += 4) {
        float r[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int f = f0 + j;
            int cnt = 0;
            if (f < p.n) {
                const uint32_t *wf = wsm + f * KW;
#pragma unroll
                for (int k = 0; k < KW; ++k) cnt += __popc(~(a[k] ^ wf[k]));
            }
            const int dot = 2 * (cnt - p.padbits) - p.K;
            if (p.counts && f < p.n) p.counts[(((size_t)n * p.n + f) * H + y) * W + x] = IntEpi<A>::raw(dot, p.K);
            const float mean = (f < p.n) ? p.mean[f] : 0.f, bias = (f < p.n) ? p.bias[f] : 0.f;
            r[j] = IntEpi<A>::finish(dot, mean, bias, p.act);
        }
        if (f0 + 3 < p.n) *reinterpret_cast<float4 *>(o + f0) = make_float4(r[0], r[1], r[2], r[3]);
        else for (int j = 0; j < 4 && f0 + j < p.n; ++j) o[f0 + j] = r[j];
    }
}

// the kernels, by arithmetic: AR_XNOR k_conv_xnor_smallk[_pool], AR_XNOR_GPU k_conv_xnor_smallk[_pool]_gpu
template <int CW>
__global__ void __launch_bounds__(128) k_conv_xnor_smallk(XnorP p) { xnor_smallk<CW, AR_XNOR>(p); }
template <int CW>
__global__ void __launch_bounds__(128) k_conv_xnor_smallk_gpu(XnorP p) { xnor_smallk<CW, AR_XNOR_GPU>(p); }
template <int CW, SideFmt F>
__global__ void __launch_bounds__(128) k_conv_xnor_smallk_pool(XnorP p, TV q /* next layer's input */) { xnor_smallk_pool<CW, F, AR_XNOR>(p, q); }
template <int CW, SideFmt F>
__global__ void __launch_bounds__(128) k_conv_xnor_smallk_pool_gpu(XnorP p, TV q) { xnor_smallk_pool<CW, F, AR_XNOR_GPU>(p, q); }

// ------------------------------------------------------------------------------------------------------
// small layers (one thread per output element, channels innermost -> coalesced)
// ------------------------------------------------------------------------------------------------------

// The max-pool window of forward_maxpool_layer_avx's scalar build (reference additionally.c:1448-1482), for output pixel
// (n, y, x) and channels c0 .. c0+V-1: m[k] starts at -FLT_MAX and takes each in-image tap of the window (origin
// o*stride - pad/2, out-of-image taps skipped) that is strictly greater.  Channels past in.C keep -FLT_MAX.  With vec (the
// input is a vec16_view) a group wholly inside in.C is read with 16-byte loads, all issued together; otherwise value by value.
// The window is walked by one loop per load form, so the 16-byte loop carries no per-tap branch and unrolls.
template <typename T, int V>
__device__ __forceinline__ void pool_window(const TV &in, int n, int y, int x, int c0, int size, int stride, int pad, bool vec,
                                            float (&m)[V]) {
#pragma unroll
    for (int k = 0; k < V; ++k) m[k] = -3.402823466e+38f;
    auto window = [&](auto fold) {   // fold(src) for each in-image tap, src: channel c0 of the tap's pixel
        const int off = -pad / 2;
        for (int a = 0; a < size; ++a) {
            const int iy = off + y * stride + a;
            if (iy < 0 || iy >= in.H) continue;
            for (int b = 0; b < size; ++b) {
                const int ix = off + x * stride + b;
                if (ix < 0 || ix >= in.W) continue;
                fold(tv_px<T>(in, n, iy, ix) + c0);
            }
        }
    };
    constexpr int L = (V * sizeof(T) + 15) / 16;   // 16-byte loads per group, where the group is whole ones
    if (V * sizeof(T) % 16 == 0 && vec && c0 + V <= in.C) {
        window([&](const T *src) {
            uint4 raw[L];
#pragma unroll
            for (int k = 0; k < L; ++k) raw[k] = __ldg(reinterpret_cast<const uint4 *>(src) + k);
            const T *v = reinterpret_cast<const T *>(raw);
#pragma unroll
            for (int k = 0; k < V; ++k) { const float f = to_f32(v[k]); m[k] = f > m[k] ? f : m[k]; }
        });
    } else {
        window([&](const T *src) {
#pragma unroll
            for (int k = 0; k < V; ++k)
                if (c0 + k < in.C) { const float f = to_f32(src[k]); m[k] = f > m[k] ? f : m[k]; }
        });
    }
}

// Max-pool: one thread per element, or with VEC one per 16 bytes of channels (4 f32 / 8 bf16), which the engine runs on
// vec16_view input and output whose channel rows are whole 16-byte groups.
template <typename T, bool VEC>
__device__ __forceinline__ void maxpool(const TV &in, const TV &out, int size, int stride, int pad) {
    constexpr int V = VEC ? 16 / sizeof(T) : 1;   // channels per thread
    const int groups = out.C / V;
    const long total = (long)out.N * out.H * out.W * groups;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int g = (int)(i % groups);
        const long pxl = i / groups;
        const int x = (int)(pxl % out.W);
        const int y = (int)((pxl / out.W) % out.H);
        const int n = (int)(pxl / ((long)out.W * out.H));
        float m[V];
        pool_window<T>(in, n, y, x, g * V, size, stride, pad, VEC, m);
        T *dst = tv_px<T>(out, n, y, x) + g * V;
        if constexpr (VEC) {
            uint4 o;
            T *ov = reinterpret_cast<T *>(&o);
#pragma unroll
            for (int k = 0; k < V; ++k) ov[k] = from_f32<T>(m[k]);
            *reinterpret_cast<uint4 *>(dst) = o;
        } else {
            *dst = from_f32<T>(m[0]);
        }
    }
}
// the kernels, by form: k_maxpool (one thread per element), k_maxpool_vec (16 bytes per thread)
template <typename T>
__global__ void k_maxpool(TV in, TV out, int size, int stride, int pad) { maxpool<T, false>(in, out, size, stride, pad); }
template <typename T>
__global__ void k_maxpool_vec(TV in, TV out, int size, int stride, int pad) { maxpool<T, true>(in, out, size, stride, pad); }

// The input conversion of an integer convolution: f32 activation -> side format F (yb_device.cuh), optionally behind a max-pool.
// With a 1x1 window (size 1, stride 1, pad 0) it is the conversion alone (the reference's quantisation / binarize_cpu /
// float_to_bit); with the max-pool's window it is that max-pool (pool_window) followed by the conversion, so the f32 pooled
// tensor never goes to HBM.  Either way the bytes are those of the unfused layers: a NaN or -inf input leaves -FLT_MAX, which
// converts as they do.  One thread per int_input_channels(F) channels: 16 s8 channels (one 16-byte store; s8 pixel strides are
// multiples of 32) or one word of 32 sign bits.  In the last group, channels past in.C keep -FLT_MAX (s8 0, +-1 byte -1, bit
// 0); the 16-channel groups wholly past in.C are not written and keep the values the engine placed there (s8 0, +-1 byte -1),
// the same bytes.  The input is read with 16-byte loads when it is a vec16_view, with scalar loads otherwise.
__host__ __device__ constexpr int int_input_channels(SideFmt f) { return f == SIDE_BITS ? 32 : 16; }
// k_int_input's threads per pixel of an input of C channels
__host__ __device__ constexpr int int_input_groups(SideFmt f, int C) { return (C + int_input_channels(f) - 1) / int_input_channels(f); }

template <SideFmt F>
__global__ void k_int_input(TV in /* f32 */, TV q, int size, int stride, int pad, float mult) {
    constexpr int V = int_input_channels(F);                     // channels per thread
    const int groups = int_input_groups(F, in.C);                // threads per pixel
    const int OH = q.H, OW = q.W;
    const long total = (long)q.N * OH * OW * groups;
    const bool vec = vec16_view(in, 4);
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int g = (int)(i % groups);
        const long pxl = i / groups;
        const int x = (int)(pxl % OW);
        const int y = (int)((pxl / OW) % OH);
        const int n = (int)(pxl / ((long)OW * OH));
        float m[V];
        pool_window<float>(in, n, y, x, g * V, size, stride, pad, vec, m);
        if constexpr (F == SIDE_BITS) side_px<F>(q, n, y, x)[g] = side_word<F>(m, mult);
        else reinterpret_cast<uint4 *>(side_px<F>(q, n, y, x))[g] = side_word4<F>(m, mult);
    }
}

// Pairs of f32 lanes (filter 2j, 2j + 1) in one 64-bit value, each lane rounded on its own: exactly __fmul_rn / __fadd_rn
// twice.  __fmul_rn / __fadd_rn are never contracted into an FMA, which keeps the reference's separately rounded gemm_nn order.
__device__ __forceinline__ unsigned long long f2_pack(float lo, float hi) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void f2_unpack(unsigned long long v, float &lo, float &hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ unsigned long long f2_mul(unsigned long long a, unsigned long long b) {
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1); f2_unpack(b, b0, b1);
    return f2_pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ unsigned long long f2_add(unsigned long long a, unsigned long long b) {
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1); f2_unpack(b, b0, b1);
    return f2_pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}

// ------------------------------------------------------------------------------------------------------
// Exact nets (INT8 / XNOR tiny models): stem convolution + 2x2/2 max-pool + the next integer layer's input conversion in ONE
// kernel.  Layers 0-2 of yolov3-tiny / tiny-yolo-obj_xnor are conv 3->16 (f32), maxpool 2/2, integer conv: unfused, the f32 stem
// output (709 MB at 416x416 batch 64) is written once and read once just to be reduced 4:1 and narrowed to one byte (or bit)
// per value.  One thread per POOLED pixel: the 4x4x3 input window (48 loads), four stem outputs x 16 filters in the
// reference's exact order (c, ky, kx; separately rounded products and sums: k_conv_stem<EXACT>), bias + activation, the
// reference's max (forward_maxpool_layer_avx scalar semantics: -FLT_MAX start, strict >), then quant_i8 / quant_i8_sat / sign exactly as
// k_int_input, in the side format F of the integer layer.  Bit-identical to the three separate kernels.  s8 formats: q.ldc bytes
// per pixel, of which the first 16 are written; sign bits: one word per pixel.
// ------------------------------------------------------------------------------------------------------
// ACT is a template parameter: act_exact() with a run-time activation drags the double-precision logistic (exp) into each of the 64
// call sites -- 19 k SASS instructions, 300 KB of code that no instruction cache holds.
template <SideFmt F, int ACT>
__global__ void __launch_bounds__(128) k_stem_pool(const float *__restrict__ in, TV q, const __grid_constant__ StemW<16> sw, int /*act*/,
                                                   int H, int W, float mult) {
    constexpr int NF = 16;
    const int OH = q.H, OW = q.W;
    const long total = (long)q.N * OH * OW;
    const long pidx = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (pidx >= total) return;
    const int px = (int)(pidx % OW), py = (int)((pidx / OW) % OH), n = (int)(pidx / ((long)OW * OH));
    const float *img = in + (size_t)n * 3 * H * W;
    unsigned long long acc2[4][NF / 2];          // (filter 2j, filter 2j + 1) pairs: mul.rn.f32x2 / add.rn.f32x2
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int j = 0; j < NF / 2; ++j) acc2[k][j] = 0ull;
    const int y0 = 2 * py - 1, x0 = 2 * px - 1;            // top-left of the 4x4 input window
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        unsigned long long win2[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const int iy = y0 + a, ix = x0 + b;
                const float v = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? __ldg(img + ((size_t)c * H + iy) * W + ix) : 0.f;
                win2[a][b] = f2_pack(v, v);
            }
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                for (int j = 0; j < NF / 2; ++j) {
                    const float *wp = &sw.w[((ky * 3 + kx) * 3 + c) * NF + 2 * j];
                    const unsigned long long w2 = f2_pack(wp[0], wp[1]);
#pragma unroll
                    for (int k = 0; k < 4; ++k)     // output pixel (dy, dx) = (k >> 1, k & 1); per accumulator the order is (c, ky, kx)
                        acc2[k][j] = f2_add(acc2[k][j], f2_mul(w2, win2[(k >> 1) + ky][(k & 1) + kx]));
                }
    }
    float acc[4][NF];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int j = 0; j < NF / 2; ++j) f2_unpack(acc2[k][j], acc[k][2 * j], acc[k][2 * j + 1]);
    float m[NF];
#pragma unroll
    for (int f = 0; f < NF; ++f) {
        float mx = -3.402823466e+38f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {                       // window order of the reference: rows, then columns
            const bool inside = (2 * py + (k >> 1)) < H && (2 * px + (k & 1)) < W;
            float v = __fadd_rn(acc[k][f], sw.b[f]);
            if (ACT == ACT_LEAKY) v = (v > 0.f) ? v : (float)(0.1 * (double)v);     // activate(), additionally.h:91 (scalar build)
            if (inside) mx = v > mx ? v : mx;
        }
        m[f] = mx;
    }
    uint32_t *dst = side_px<F>(q, n, py, px);
    if constexpr (F == SIDE_BITS) {
        dst[0] = side_word<F, NF>(m, mult);
    } else {
        *reinterpret_cast<uint4 *>(dst) = side_word4<F>(m, mult);
    }
}

// upsample_cpu forward (reference yolov2_forward_network.c:380-394): out = scale * in[y/stride][x/stride].  One thread per
// element, or with VEC one per 16 bytes of channels, which the engine runs at scale 1 only -- a copy of the bits, exact for
// any dtype -- on vec16_view input and output whose channel rows are whole 16-byte groups.
template <typename T, bool VEC>
__device__ __forceinline__ void upsample(const TV &in, const TV &out, int stride, float scale) {
    constexpr int V = VEC ? 16 / sizeof(T) : 1;   // channels per thread
    const int groups = out.C / V;
    const long total = (long)out.N * out.H * out.W * groups;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int g = (int)(i % groups);
        const long pxl = i / groups;
        const int x = (int)(pxl % out.W);
        const int y = (int)((pxl / out.W) % out.H);
        const int n = (int)(pxl / ((long)out.W * out.H));
        const T *src = tv_px<T>(in, n, y / stride, x / stride) + g * V;
        T *dst = tv_px<T>(out, n, y, x) + g * V;
        if constexpr (VEC) *reinterpret_cast<uint4 *>(dst) = __ldg(reinterpret_cast<const uint4 *>(src));
        else *dst = from_f32<T>(__fmul_rn(scale, to_f32(*src)));
    }
}
// the kernels, by form: k_upsample (one thread per element), k_upsample_vec16 (16 bytes per thread, scale 1)
template <typename T>
__global__ void k_upsample(TV in, TV out, int stride, float scale) { upsample<T, false>(in, out, stride, scale); }
template <typename T>
__global__ void k_upsample_vec16(TV in, TV out, int stride) { upsample<T, true>(in, out, stride, 1.f); }

// forward_shortcut_layer_cpu (reference yolov2_forward_network.c:443-449, shortcut_cpu :410-432):
// out = act(in + from) with the general stride/sample subsampling of shortcut_cpu.
template <typename T>
__global__ void k_shortcut(TV in, TV from, TV out, int stride, int sample, int minw, int minh, int minc, int act) {
    const long total = (long)out.N * out.H * out.W * out.C;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % out.C);
        const long pxl = i / out.C;
        const int x = (int)(pxl % out.W);
        const int y = (int)((pxl / out.W) % out.H);
        const int n = (int)(pxl / ((long)out.W * out.H));
        float v = to_f32(tv_px<T>(in, n, y, x)[c]);
        if (c < minc && (y % sample) == 0 && (x % sample) == 0) {
            const int j = y / sample, ii = x / sample;
            if (j < minh && ii < minw) v = __fadd_rn(v, to_f32(tv_px<T>(from, n, j * stride, ii * stride)[c]));
        }
        tv_px<T>(out, n, y, x)[c] = from_f32<T>(act_exact(v, act));
    }
}

// route: copy one source into its channel slice of the concat buffer (reference yolov2_forward_network.c:318)
template <typename T>
__global__ void k_copy_channels(TV in, TV out /* view of the slice: C == in.C */) {
    const long total = (long)in.N * in.H * in.W * in.C;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % in.C);
        const long pxl = i / in.C;
        const int x = (int)(pxl % in.W);
        const int y = (int)((pxl / in.W) % in.H);
        const int n = (int)(pxl / ((long)in.W * in.H));
        tv_px<T>(out, n, y, x)[c] = tv_px<T>(in, n, y, x)[c];
    }
}

// forward_reorg_layer_cpu (reference yolov2_forward_network.c:337-373), darknet's space-to-depth flavour:
// out[n][k][j][i] = x_flat[ w2 + (out_w*stride) * (h2 + (out_h*stride) * (c2 + in_c*n)) ] with the whole batch of the input
// reinterpreted as [N][in_c][out_h*stride][out_w*stride] where in_c = out_c/stride^2.  When stride does not divide the input's
// height or width, that view is smaller than an image, so image n > 0 reads from a flat offset inside the images before it, as
// the reference does; the index stays below N*in.C*in.H*in.W.
template <typename T>
__global__ void k_reorg(TV in, TV out, int stride) {
    const long total = (long)out.N * out.H * out.W * out.C;
    const int in_c = out.C / (stride * stride);
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int k = (int)(i % out.C);
        const long pxl = i / out.C;
        const int x = (int)(pxl % out.W);
        const int y = (int)((pxl / out.W) % out.H);
        const int n = (int)(pxl / ((long)out.W * out.H));
        const int c2 = k % in_c, offset = k / in_c;
        const int w2 = x * stride + offset % stride, h2 = y * stride + offset / stride;
        // flat index into the batch viewed as [N][in_c][out.H*stride][out.W*stride]
        const long flat = w2 + (long)out.W * stride * (h2 + (long)out.H * stride * (c2 + (long)in_c * n));
        // map the flat NCHW index back onto the real source dims [N][in.C][in.H][in.W]
        const int sx = (int)(flat % in.W);
        const int sy = (int)((flat / in.W) % in.H);
        const int sc = (int)((flat / ((long)in.W * in.H)) % in.C);
        const int sn = (int)(flat / ((long)in.W * in.H * in.C));
        tv_px<T>(out, n, y, x)[k] = tv_px<T>(in, sn, sy, sx)[sc];
    }
}

// forward_yolo_layer_cpu (reference yolov2_forward_network.c:453-472): copy + logistic on entries 0,1 and
// 4..4+classes of each anchor block.  Reads the head conv's NHWC activation, writes the NCHW f32 tensor the
// reference decoder expects (additionally.c:4200 entry_index).
template <typename TIn>
__global__ void __launch_bounds__(256) k_yolo(TV in, float *__restrict__ out, int classes, int fast) {
    // 32 pixels x 32 channels per tile: channel-contiguous reads (NHWC), pixel-contiguous writes (NCHW)
    __shared__ float tile[32][33];
    const int HW = in.H * in.W;
    const int ptiles = (HW + 31) / 32, ctiles = (in.C + 31) / 32;
    const long ntiles = (long)in.N * ptiles * ctiles;
    const int per = 4 + classes + 1;
    const int lane = threadIdx.x & 31, wy = threadIdx.x >> 5;   // 8 warps
    for (long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int ct = (int)(t % ctiles);
        const int pt = (int)((t / ctiles) % ptiles);
        const int n = (int)(t / ((long)ctiles * ptiles));
        const int c = ct * 32 + lane;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int pl = wy * 4 + k;
            const int hw = pt * 32 + pl;
            float v = 0.f;
            if (hw < HW && c < in.C) {
                v = to_f32(tv_px<TIn>(in, n, hw / in.W, hw % in.W)[c]);
                const int e = c % per;
                // exact nets: the reference's double-precision logistic; bf16 tensor-core nets: f32 (error ~1e-7,
                // far below the path's 1e-3 bar)
                if (e != 2 && e != 3) v = fast ? 1.f / (1.f + __expf(-v)) : (float)(1.0 / (1.0 + exp(-(double)v)));
            }
            tile[pl][lane] = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int cl = wy * 4 + k;
            const int cc = ct * 32 + cl;
            const int hw = pt * 32 + lane;
            if (hw < HW && cc < in.C) out[((size_t)n * in.C + cc) * HW + hw] = tile[lane][cl];
        }
        __syncthreads();
    }
}

// forward_region_layer_cpu (reference yolov2_forward_network.c:511-575): per image HWC flatten (== our NHWC
// order), float logistic on entry 4, softmax over classes (softmax_cpu :476) when softmax=1.
// One thread per (image, cell, anchor).
template <typename TIn>
__global__ void k_region(TV in, float *__restrict__ out, int nanchors, int classes, int coords, int softmax) {
    const int size = coords + classes + 1;
    const long total = (long)in.N * in.H * in.W * nanchors;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int a = (int)(i % nanchors);
        const long pxl = i / nanchors;
        const int x = (int)(pxl % in.W);
        const int y = (int)((pxl / in.W) % in.H);
        const int n = (int)(pxl / ((long)in.W * in.H));
        const TIn *src = tv_px<TIn>(in, n, y, x) + a * size;
        float *o = out + (((size_t)n * in.H + y) * in.W + x) * (size_t)(nanchors * size) + (size_t)a * size;
        for (int k = 0; k < coords; ++k) o[k] = to_f32(src[k]);
        o[coords] = 1.0f / (1.0f + expf(-to_f32(src[coords])));
        if (softmax) {
            float largest = -3.402823466e+38f;
            for (int k = 0; k < classes; ++k) { const float v = to_f32(src[coords + 1 + k]); if (v > largest) largest = v; }
            float sum = 0.f;
            for (int k = 0; k < classes; ++k) {
                const float e = expf(to_f32(src[coords + 1 + k]) - largest);
                sum += e;
                o[coords + 1 + k] = e;
            }
            for (int k = 0; k < classes; ++k) o[coords + 1 + k] = __fdiv_rn(o[coords + 1 + k], sum);
        } else {
            for (int k = 0; k < classes; ++k) o[coords + 1 + k] = to_f32(src[coords + 1 + k]);
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// INT8 input calibration (SURVEY 8f row 3): histogram of |x| over the logical elements of image `img` of an
// activation tensor, binned exactly like the reference (yolov2_forward_network_quantized.c:1308-1316:
// lround(fabs(x) / bin_width) in double, saturated into the last bin).  Per-block shared-memory histogram,
// integer atomics -> exact counts.  max_bin <= 4096.
// ------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_abs_hist(TV in, int img, float bin_width, int max_bin, unsigned *__restrict__ hist) {
    __shared__ unsigned sh[4096];
    for (int i = threadIdx.x; i < max_bin; i += 256) sh[i] = 0u;
    __syncthreads();
    const long per = (long)in.C * in.H * in.W;
    const int last_bin = max_bin - 1;
    for (long e = (long)blockIdx.x * 256 + threadIdx.x; e < per; e += (long)gridDim.x * 256) {
        const int c = (int)(e % in.C);
        const long px = e / in.C;
        const int x = (int)(px % in.W), y = (int)(px / in.W);
        const float v = to_f32(tv_px<T>(in, img, y, x)[c]);
        const long b = lround(fabs((double)v) / (double)bin_width);
        atomicAdd(&sh[b >= last_bin ? last_bin : (int)b], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < max_bin; i += 256)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
}
// the network input (NCHW f32, as the caller passes it)
static __global__ void __launch_bounds__(256) k_abs_hist_flat(const float *__restrict__ src, long n, float bin_width, int max_bin,
                                                              unsigned *__restrict__ hist) {
    __shared__ unsigned sh[4096];
    for (int i = threadIdx.x; i < max_bin; i += 256) sh[i] = 0u;
    __syncthreads();
    const int last_bin = max_bin - 1;
    for (long e = (long)blockIdx.x * 256 + threadIdx.x; e < n; e += (long)gridDim.x * 256) {
        const long b = lround(fabs((double)src[e]) / (double)bin_width);
        atomicAdd(&sh[b >= last_bin ? last_bin : (int)b], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < max_bin; i += 256)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

}  // namespace yb
