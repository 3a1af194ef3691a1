// yb_detect.cuh -- batched detection decode + NMS on the device (SURVEY 8f row 1).
//
// Replaces, for every image of the batch at once and without moving the yolo / region tensors to the host,
//   get_network_boxes            src/additionally.c:4403  (make_network_boxes :4381, fill_network_boxes :4391)
//     get_yolo_detections        src/additionally.c:4317-4357   (objectness > thresh, get_yolo_box :4263)
//     custom_get_region_detections src/additionally.c:4363      (every box; get_region_box_cpu, yolov2_forward_network.c:653)
//     correct_yolo_boxes         src/additionally.c:4281-4315
//   do_nms_sort                  src/box.c:296-328  (box_iou :46-70)
//
// Pipeline per image (4 launches for the first nimg images of the batch, grid.y = image):
//   k_det_count  : candidates per 256-box block, boxes enumerated in the reference's order (layer, cell, anchor)
//   k_det_emit   : stable compaction (block offsets + ballot scan), decode, row = {x, y, w, h, objectness, prob[classes]}
//   k_det_iou    : bit matrix  M[i][j] = box_iou(i, j) > nms   (once per image, shared by all classes)
//   k_det_nms    : one block per (class, image): sort candidates by prob[class] (bitonic, shared memory), then the
//                  reference's greedy scan with row-wise bit clears; suppressed entries get prob = 0 like box.c:319
// Arithmetic follows the reference expression by expression (double where C promotes to double, float divides and
// multiplies without FMA contraction) so that thresholds and IoU comparisons decide identically.
#pragma once
#include <climits>
#include <cuda_runtime.h>

#include "yb_kernels.cuh"   // ImageGeo

namespace yb {

constexpr int DET_MAX_LAYERS = 8;
constexpr int DET_MAX_ANCHORS = 16;

struct DetLayer {
    const float *p;          // device tensor of the layer, all images ([b][outputs])
    int type;                // YB_YOLO / YB_REGION
    int w, h, n, classes, outputs;
    int base, nbox;          // first candidate ordinal of this layer, number of boxes (w*h*n)
    float aw[DET_MAX_ANCHORS], ah[DET_MAX_ANCHORS];   // anchors (already through the yolo mask)
};

struct DetParams {
    DetLayer L[DET_MAX_LAYERS];
    int nl, total, classes;
    const ImageGeo *geo;     // per image: frame size and correct_yolo_boxes' embedded size
    int netw, neth, relative;
    float thresh, nms;
    int max_rows, nblk;
};

__device__ __forceinline__ bool det_locate(const DetParams &P, int ord, int &li, int &cell, int &a) {
    if (ord >= P.total) return false;
    li = 0;
    while (li + 1 < P.nl && ord >= P.L[li + 1].base) ++li;
    const int r = ord - P.L[li].base;
    cell = r / P.L[li].n;
    a = r - cell * P.L[li].n;
    return true;
}

__device__ __forceinline__ bool det_flag(const DetParams &P, int b, int ord, int &li, int &cell, int &a) {
    if (!det_locate(P, ord, li, cell, a)) return false;
    const DetLayer &l = P.L[li];
    if (l.type == YB_REGION) return true;                       // custom_get_region_detections keeps every box
    const int hw = l.w * l.h;
    const float obj = l.p[(size_t)b * l.outputs + (size_t)a * hw * (l.classes + 5) + (size_t)4 * hw + cell];
    return obj > P.thresh;                                      // additionally.c:4331
}

static __global__ void __launch_bounds__(256) k_det_count(DetParams P, int *blkcnt) {
    const int b = blockIdx.y;
    int li, cell, a;
    const bool f = det_flag(P, b, blockIdx.x * 256 + threadIdx.x, li, cell, a);
    const int c = __syncthreads_count(f ? 1 : 0);
    if (threadIdx.x == 0) blkcnt[b * P.nblk + blockIdx.x] = c;
}

static __global__ void __launch_bounds__(256) k_det_emit(DetParams P, const int *blkcnt, float *rows, int *counts) {
    __shared__ int warp_tot[8];
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int li = 0, cell = 0, a = 0;
    const bool f = det_flag(P, b, blockIdx.x * 256 + threadIdx.x, li, cell, a);
    // candidates of the blocks before this one: summed by the whole block (a serial loop over up to 89 dependent global loads in
    // every thread made this kernel ~20 us of pure latency on the compute stream)
    __shared__ int s_off;
    if (threadIdx.x == 0) s_off = 0;
    __syncthreads();
    {
        int part = 0;
        for (int k = threadIdx.x; k < (int)blockIdx.x; k += 256) part += blkcnt[b * P.nblk + k];
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        if (lane == 0 && part) atomicAdd(&s_off, part);
    }
    __syncthreads();
    const int offset = s_off;
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    int pre = __popc(bal & ((1u << lane) - 1u));
    for (int k = 0; k < warp; ++k) pre += warp_tot[k];
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
        int tot = offset;
        for (int k = 0; k < 8; ++k) tot += warp_tot[k];
        counts[b] = tot;
    }
    const int slot = offset + pre;
    if (!f || slot >= P.max_rows) return;
    const DetLayer &l = P.L[li];
    const int stride = 5 + P.classes;
    float *o = rows + ((size_t)b * P.max_rows + slot) * stride;
    const float *p = l.p + (size_t)b * l.outputs;
    const int row = cell / l.w, col = cell - (cell / l.w) * l.w;
    float x, y, w, h, obj, scale;
    if (l.type == YB_YOLO) {
        const int hw = l.w * l.h;
        const float *q = p + (size_t)a * hw * (l.classes + 5) + cell;
        obj = q[(size_t)4 * hw];
        // get_yolo_box, additionally.c:4263-4271: float adds/divides; exp() in double, product in double
        x = __fdiv_rn(__fadd_rn((float)col, q[0]), (float)l.w);
        y = __fdiv_rn(__fadd_rn((float)row, q[(size_t)hw]), (float)l.h);
        w = (float)(exp((double)q[(size_t)2 * hw]) * (double)l.aw[a] / (double)P.netw);
        h = (float)(exp((double)q[(size_t)3 * hw]) * (double)l.ah[a] / (double)P.neth);
        scale = obj;
        for (int j = 0; j < l.classes; ++j) {
            const float prob = __fmul_rn(scale, q[(size_t)(5 + j) * hw]);
            o[5 + j] = (prob > P.thresh) ? prob : 0.f;            // additionally.c:4343-4345
        }
    } else {
        const int index = cell * l.n + a;
        const float *q = p + (size_t)index * (l.classes + 5);
        // get_region_box_cpu, yolov2_forward_network.c:653-661: logistic_activate evaluates in double but RETURNS float
        // (additionally.h:85); the add and the divide are then float operations
        const float lx = (float)(1. / (1. + exp(-(double)q[0]))), ly = (float)(1. / (1. + exp(-(double)q[1])));
        x = __fdiv_rn(__fadd_rn((float)col, lx), (float)l.w);
        y = __fdiv_rn(__fadd_rn((float)row, ly), (float)l.h);
        w = __fdiv_rn(__fmul_rn(expf(q[2]), l.aw[a]), (float)l.w);
        h = __fdiv_rn(__fmul_rn(expf(q[3]), l.ah[a]), (float)l.h);
        obj = 1.f;
        scale = q[4];
        for (int j = 0; j < l.classes; ++j) {
            const float prob = __fmul_rn(scale, q[5 + j]);
            o[5 + j] = (prob > P.thresh) ? prob : 0.f;
        }
    }
    // correct_yolo_boxes, additionally.c:4281-4315 (mixed float / double exactly as written there), for image b's frame
    const ImageGeo &G = P.geo[b];
    x = (float)(((double)x - (double)(P.netw - G.new_w) / 2. / (double)P.netw) / (double)__fdiv_rn((float)G.new_w, (float)P.netw));
    y = (float)(((double)y - (double)(P.neth - G.new_h) / 2. / (double)P.neth) / (double)__fdiv_rn((float)G.new_h, (float)P.neth));
    w = __fmul_rn(w, __fdiv_rn((float)P.netw, (float)G.new_w));
    h = __fmul_rn(h, __fdiv_rn((float)P.neth, (float)G.new_h));
    if (!P.relative) {
        x = __fmul_rn(x, (float)G.w); w = __fmul_rn(w, (float)G.w);
        y = __fmul_rn(y, (float)G.h); h = __fmul_rn(h, (float)G.h);
    }
    o[0] = x; o[1] = y; o[2] = w; o[3] = h; o[4] = obj;
}

__device__ __forceinline__ float det_overlap(float x1, float w1, float x2, float w2) {   // box.c:46-55
    const float l1 = __fsub_rn(x1, __fdiv_rn(w1, 2.f)), l2 = __fsub_rn(x2, __fdiv_rn(w2, 2.f));
    const float left = l1 > l2 ? l1 : l2;
    const float r1 = __fadd_rn(x1, __fdiv_rn(w1, 2.f)), r2 = __fadd_rn(x2, __fdiv_rn(w2, 2.f));
    const float right = r1 < r2 ? r1 : r2;
    return __fsub_rn(right, left);
}

// mask[b][i][wd] bit j: box_iou(i, 32*wd + j) > nms
static __global__ void __launch_bounds__(128) k_det_iou(DetParams P, const float *rows, const int *counts, unsigned *mask) {
    const int b = blockIdx.z;
    const int n = min(counts[b], P.max_rows);
    const int words = (P.max_rows + 31) / 32;
    const int wd = blockIdx.x * 128 + threadIdx.x;
    if (wd >= words || wd * 32 >= n) return;
    const int stride = 5 + P.classes;
    for (int i = blockIdx.y; i < n; i += gridDim.y) {        // grid.y is capped: the pipelined path sizes it without knowing n
    const float *ri = rows + ((size_t)b * P.max_rows + i) * stride;
    const float ax = ri[0], ay = ri[1], aw = ri[2], ah = ri[3];
    unsigned m = 0;
    for (int j = 0; j < 32; ++j) {
        const int k = wd * 32 + j;
        if (k >= n) break;
        const float *rk = rows + ((size_t)b * P.max_rows + k) * stride;
        const float bx = rk[0], by = rk[1], bw = rk[2], bh = rk[3];
        const float ow = det_overlap(ax, aw, bx, bw), oh = det_overlap(ay, ah, by, bh);
        const float inter = (ow < 0.f || oh < 0.f) ? 0.f : __fmul_rn(ow, oh);                        // box.c:57-64
        const float uni = __fsub_rn(__fadd_rn(__fmul_rn(aw, ah), __fmul_rn(bw, bh)), inter);         // box.c:66-70
        if (__fdiv_rn(inter, uni) > P.nms) m |= 1u << j;
    }
    mask[((size_t)b * P.max_rows + i) * words + wd] = m;
    }
}

// Block-wide bitonic sort of (key, idx)[0 .. np2) in shared memory, np2 a power of two, NT threads: afterwards before(a, b)
// holds for every earlier entry a and later entry b, given that `before` is a strict total order on the entries.  Ends with a
// barrier.
template <int NT, class Before>
__device__ __forceinline__ void block_bitonic_sort(float *key, int *idx, int np2, Before before) {
    for (int k = 2; k <= np2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < np2; i += NT) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const float ka = key[i], kb = key[ixj];
                    const int ia = idx[i], ib = idx[ixj];
                    const bool a_first = before(ka, ia, kb, ib);    // a belongs before b
                    const bool up = (i & k) == 0;
                    if (up ? !a_first : a_first) { key[i] = kb; key[ixj] = ka; idx[i] = ib; idx[ixj] = ia; }
                }
            }
            __syncthreads();
        }
    }
}
struct DescThenIndex {   // descending key, equal keys by ascending index
    __device__ bool operator()(float ka, int ia, float kb, int ib) const { return ka > kb || (ka == kb && ia < ib); }
};
struct AscThenIndex {    // ascending key, equal keys by ascending index
    __device__ bool operator()(float ka, int ia, float kb, int ib) const { return ka < kb || (ka == kb && ia < ib); }
};

// one block per (class, image); dynamic smem: keys float[P2], idx int[P2], alive unsigned[words]
static __global__ void __launch_bounds__(256) k_det_nms(DetParams P, float *rows, const int *counts, const unsigned *mask, int P2) {
    extern __shared__ unsigned char det_smem[];
    float *key = reinterpret_cast<float *>(det_smem);
    int *idx = reinterpret_cast<int *>(key + P2);
    unsigned *alive = reinterpret_cast<unsigned *>(idx + P2);
    __shared__ int s_m;
    const int c = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
    const int n = min(counts[b], P.max_rows);
    if (n == 0) return;
    const int words = (P.max_rows + 31) / 32;
    const int stride = 5 + P.classes;
    float *rb = rows + (size_t)b * P.max_rows * stride;
    int np2 = 1; while (np2 < n) np2 <<= 1;
    if (t == 0) s_m = 0;
    __syncthreads();
    int local = 0;
    for (int i = t; i < np2; i += 256) {
        const float pr = (i < n) ? rb[(size_t)i * stride + 5 + c] : 0.f;
        key[i] = pr > 0.f ? pr : -1.f;
        idx[i] = i;
        local += pr > 0.f ? 1 : 0;
    }
    for (int i = t; i < words; i += 256) alive[i] = 0xffffffffu;
    atomicAdd(&s_m, local);
    __syncthreads();
    const int m = s_m;
    if (m == 0) return;
    // descending by (prob, then lower index first) -- qsort's tie order in box.c:311 is unspecified
    block_bitonic_sort<256>(key, idx, np2, DescThenIndex{});
    // greedy scan (box.c:313-322): a live candidate clears every box whose IoU with it exceeds nms
    for (int k = 0; k < m; ++k) {
        const int i = idx[k];
        const bool live = (alive[i >> 5] >> (i & 31)) & 1u;
        __syncthreads();
        if (live) {
            const unsigned *mr = mask + ((size_t)b * P.max_rows + i) * words;
            for (int wd = t; wd * 32 < n; wd += 256) {
                unsigned mm = mr[wd];
                if (wd == (i >> 5)) mm &= ~(1u << (i & 31));     // the candidate itself stays
                alive[wd] &= ~mm;
            }
        } else if (t == 0) {
            rb[(size_t)i * stride + 5 + c] = 0.f;                 // suppressed by an earlier, stronger box
        }
        __syncthreads();
    }
}

// ---- drawing the detections into the caller's device frames (draw_detections_v3, src/main.c:80-148) ---------------------
//   k_det_select : one block per image: get_actual_detections (main.c:38-62) on the image's post-NMS candidate rows, then
//                  the selected list in compare_by_lefts order (main.c:65-70) and the boxes in compare_by_probs order
//                  (main.c:73-78, :107), each with its clamped corners (main.c:109-143) and colour (get_color,
//                  additionally.c:3247); equal keys by candidate position, like the NMS
//   k_det_draw<F>: one block per band of rows of an image walks the boxes in draw order, with a barrier after each, so a later
//                  box overwrites an earlier one wherever they share pixels; draw_box_width / draw_box (additionally.c:2945-2988)
//                  in format F

constexpr int DET_DRAW_BANDS = 8;   // k_det_draw's blocks per image

struct DetDraw {                  // one box in draw order
    int x1, y1, x2, y2;           // draw_box_width's corners: left, top, right, bot after draw_detections_v3's clamp
    unsigned char rgb[3], yuv[3]; // its colour as save_image_png writes it, and as NV12 bytes (rgb_to_yuv601)
};

// x86's cvttsd2si, which the reference's double -> int conversions compile to: truncation, and INT_MIN for NaN and for every
// value whose truncation is outside int (CUDA's conversion saturates instead)
__device__ __forceinline__ int det_d2i_x86(double v) {
    return (v > -2147483649.0 && v < 2147483648.0) ? (int)v : INT_MIN;
}
// int + / - as the reference's x86 build computes draw_box_width's x1 + i, x2 - i: two's complement, wrapping
__device__ __forceinline__ int det_wrap_add(int a, int b) { return (int)((unsigned)a + (unsigned)b); }

__constant__ float c_det_colors[6][3] = {{1, 0, 1}, {0, 0, 1}, {0, 1, 1}, {0, 1, 0}, {1, 1, 0}, {1, 0, 0}};

// get_color(c, x, max), additionally.c:3247-3257: float arithmetic, floor / ceil of the float promoted to double, no contraction
__device__ __forceinline__ float det_get_color(int c, int x, int max) {
    float ratio = __fmul_rn(__fdiv_rn((float)x, (float)max), 5.f);
    const int i = (int)floor((double)ratio), j = (int)ceil((double)ratio);
    ratio = __fsub_rn(ratio, (float)i);
    return __fadd_rn(__fmul_rn(__fsub_rn(1.f, ratio), c_det_colors[i][c]), __fmul_rn(ratio, c_det_colors[j][c]));
}

// one block per image; dynamic smem: key float[P2], idx int[P2], sel int[P2] (row | best class << 14), P2 >= max_rows
// sel: yb_detection[batch][max_rows] in list order, nsel[batch], draw: DetDraw[batch][max_rows] in draw order
static __global__ void __launch_bounds__(256) k_det_select(DetParams P, const float *rows, const int *counts, yb_detection *sel,
                                                           int *nsel, DetDraw *draw, int P2) {
    extern __shared__ unsigned char det_smem[];
    float *key = reinterpret_cast<float *>(det_smem);
    int *idx = reinterpret_cast<int *>(key + P2);
    int *pick = idx + P2;
    __shared__ int s_wsum[8], s_m;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int n = min(counts[b], P.max_rows);
    const int stride = 5 + P.classes;
    const float *rb = rows + (size_t)b * P.max_rows * stride;
    if (t == 0) s_m = 0;
    __syncthreads();
    // get_actual_detections: the best class is the first j with prob[j] > best, best starting at thresh; stable compaction
    for (int c0 = 0; c0 < n; c0 += 256) {
        const int i = c0 + t;
        int best = -1;
        if (i < n) {
            float bp = P.thresh;
            const float *pr = rb + (size_t)i * stride + 5;
            for (int j = 0; j < P.classes; ++j) {
                const float p = pr[j];
                if (p > bp) { best = j; bp = p; }
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, best >= 0);
        if (lane == 0) s_wsum[warp] = __popc(bal);
        __syncthreads();
        int pos = s_m + __popc(bal & ((1u << lane) - 1u));
        for (int k = 0; k < warp; ++k) pos += s_wsum[k];
        if (best >= 0) pick[pos] = i | best << 14;
        __syncthreads();
        if (t == 0) for (int k = 0; k < 8; ++k) s_m += s_wsum[k];
        __syncthreads();
    }
    const int m = s_m;
    if (t == 0) nsel[b] = m;
    if (m == 0) return;
    int np2 = 1; while (np2 < m) np2 <<= 1;
    // list order, compare_by_lefts: ascending float x - w / 2 (a NaN key sorts as +inf), equal keys by candidate position
    for (int i = t; i < np2; i += 256) {
        float k = __int_as_float(0x7f800000);
        if (i < m) {
            const float *r = rb + (size_t)(pick[i] & 16383) * stride;
            k = __fsub_rn(r[0], __fdiv_rn(r[2], 2.f));
            if (k != k) k = __int_as_float(0x7f800000);
        }
        key[i] = k;
        idx[i] = i;
    }
    __syncthreads();
    block_bitonic_sort<256>(key, idx, np2, AscThenIndex{});
    yb_detection *so = sel + (size_t)b * P.max_rows;
    for (int k = t; k < m; k += 256) {
        const int row = pick[idx[k]] & 16383, cls = pick[idx[k]] >> 14;
        const float *r = rb + (size_t)row * stride;
        so[k] = yb_detection{r[0], r[1], r[2], r[3], r[5 + cls], cls, row};
    }
    __syncthreads();
    // draw order, compare_by_probs: ascending prob[best class], equal keys by candidate position
    for (int i = t; i < np2; i += 256) {
        key[i] = i < m ? rb[(size_t)(pick[i] & 16383) * stride + 5 + (pick[i] >> 14)] : __int_as_float(0x7f800000);
        idx[i] = i;
    }
    __syncthreads();
    block_bitonic_sort<256>(key, idx, np2, AscThenIndex{});
    const ImageGeo &G = P.geo[b];
    const double imw = (double)G.w, imh = (double)G.h;
    DetDraw *dd = draw + (size_t)b * P.max_rows;
    for (int k = t; k < m; k += 256) {
        const int row = pick[idx[k]] & 16383, cls = pick[idx[k]] >> 14;
        const float *r = rb + (size_t)row * stride;
        const double x = r[0], y = r[1], w = r[2], h = r[3];
        // main.c:125-133, in double without contraction
        int left = det_d2i_x86(__dmul_rn(__dsub_rn(x, __ddiv_rn(w, 2.)), imw));
        int right = det_d2i_x86(__dmul_rn(__dadd_rn(x, __ddiv_rn(w, 2.)), imw));
        int top = det_d2i_x86(__dmul_rn(__dsub_rn(y, __ddiv_rn(h, 2.)), imh));
        int bot = det_d2i_x86(__dmul_rn(__dadd_rn(y, __ddiv_rn(h, 2.)), imh));
        if (left < 0) left = 0;
        if (right > G.w - 1) right = G.w - 1;
        if (top < 0) top = 0;
        if (bot > G.h - 1) bot = G.h - 1;
        DetDraw D;
        D.x1 = left; D.y1 = top; D.x2 = right; D.y2 = bot;
        const int offset = cls * 123457 % P.classes;           // main.c:116 (the caller bounds classes so that this fits)
        for (int c = 0; c < 3; ++c)                            // red = get_color(2, ...), green (1, ...), blue (0, ...)
            D.rgb[c] = (unsigned char)(int)__fmul_rn(255.f, det_get_color(2 - c, offset, P.classes));   // additionally.c:3226
        rgb_to_yuv601(D.rgb[0], D.rgb[1], D.rgb[2], D.yuv);
        dd[k] = D;
    }
}

// pixel (x, y) of frame g in colour D
template <int F>
__device__ __forceinline__ void det_put(const ImageGeo &g, int x, int y, const DetDraw &D) {
    unsigned char *p = const_cast<unsigned char *>(g.src);
    if (F == YB_FRAME_RGB || F == YB_FRAME_BGR) {
        unsigned char *q = p + (size_t)y * g.pitch + 3 * x;
        q[0] = D.rgb[F == YB_FRAME_RGB ? 0 : 2]; q[1] = D.rgb[1]; q[2] = D.rgb[F == YB_FRAME_RGB ? 2 : 0];
    } else if (F == YB_FRAME_RGB_PLANAR) {
        unsigned char *q = p + (size_t)y * g.pitch + x;
        q[0] = D.rgb[0]; q[g.plane] = D.rgb[1]; q[2 * g.plane] = D.rgb[2];
    } else {   // NV12: the pixel's Y and the chroma pair of its 2x2 block
        p[(size_t)y * g.pitch + x] = D.yuv[0];
        unsigned char *c = const_cast<unsigned char *>(g.chroma) + (size_t)(y >> 1) * g.pitch + (x & ~1);
        c[0] = D.yuv[1]; c[1] = D.yuv[2];
    }
}

// draw_box_width(im, left, top, right, bot, width, ...) for every box in draw order.  Block (b, k) owns the rows of band k
// of image b -- gridDim.y bands of an even number of rows, so a band also owns the NV12 chroma rows of its pixels -- and
// walks all boxes in draw order with a barrier after each, so that a later box overwrites an earlier one on every pixel
// where the reference's loop does.
template <int F>
static __global__ void __launch_bounds__(256) k_det_draw(const ImageGeo *__restrict__ geo, const DetDraw *__restrict__ draw,
                                                         const int *__restrict__ nsel, int max_rows) {
    const int b = blockIdx.x;
    const ImageGeo g = geo[b];
    const int bh = ((g.h + (int)gridDim.y - 1) / (int)gridDim.y + 1) & ~1;
    const int r0 = blockIdx.y * bh, r1 = min(g.h, r0 + bh) - 1;    // the band's rows r0 .. r1
    if (r0 >= g.h) return;
    const int m = nsel[b];
    int width = (int)((double)g.h * .006);                     // main.c:109-111
    if (width < 1) width = 1;
    for (int d = 0; d < m; ++d) {
        const DetDraw D = draw[(size_t)b * max_rows + d];
        for (int i = 0; i < width; ++i) {
            // draw_box(a, x1 + i, y1 + i, x2 - i, y2 - i): each corner clamped into the frame, then rows y1 and y2 over
            // x1 .. x2 and columns x1 and x2 over y1 .. y2 (none where the range is empty); here their pixels in the band
            int x1 = det_wrap_add(D.x1, i), y1 = det_wrap_add(D.y1, i), x2 = det_wrap_add(D.x2, -i), y2 = det_wrap_add(D.y2, -i);
            x1 = min(max(x1, 0), g.w - 1); x2 = min(max(x2, 0), g.w - 1);
            y1 = min(max(y1, 0), g.h - 1); y2 = min(max(y2, 0), g.h - 1);
            const int nx = max(0, x2 - x1 + 1);
            const int ha = (y1 >= r0 && y1 <= r1) ? nx : 0, hb = (y2 >= r0 && y2 <= r1) ? nx : 0;
            const int ya = max(y1, r0), ny = max(0, min(y2, r1) - ya + 1);
            for (int p = threadIdx.x; p < ha + hb + 2 * ny; p += 256) {
                if (p < ha) det_put<F>(g, x1 + p, y1, D);
                else if (p < ha + hb) det_put<F>(g, x1 + p - ha, y2, D);
                else det_put<F>(g, ((p - ha - hb) & 1) ? x2 : x1, ya + ((p - ha - hb) >> 1), D);
            }
        }
        __syncthreads();   // the next box overwrites this one where they meet
    }
}
}  // namespace yb
