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
    // bitonic sort, descending by (prob, then lower index first) -- qsort's tie order in box.c:311 is unspecified
    for (int k = 2; k <= np2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = t; i < np2; i += 256) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const float ka = key[i], kb = key[ixj];
                    const int ia = idx[i], ib = idx[ixj];
                    const bool a_first = (ka > kb) || (ka == kb && ia < ib);     // a belongs before b in descending order
                    const bool up = (i & k) == 0;
                    if (up ? !a_first : a_first) { key[i] = kb; key[ixj] = ka; idx[i] = ib; idx[ixj] = ia; }
                }
            }
            __syncthreads();
        }
    }
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

}  // namespace yb
