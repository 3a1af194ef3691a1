// yb_engine.cu -- builds and runs the device execution plan of a prepared network.
//
// Mirrors the layer loop of the reference (yolov2_forward_network_cpu, src/yolov2_forward_network.c:581-628 and
// yolov2_forward_network_q, src/yolov2_forward_network_quantized.c:1027-1089) as a flat list of kernel
// launches with pre-resolved device pointers, replayed as a CUDA graph.  See yb_kernels.cuh for the device
// layout.  No CPU fallback: everything here requires a compute-capability-9.0 device (H100).
#include "yb_engine.h"

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "yb_conv_tc.cuh"
#include "yb_cuda.h"
#include "yb_kernels.cuh"
#include "yb_detect.cuh"

namespace yb {

const char *op_kind_name(int k) {
    static const char *names[] = {"input", "conv_simt", "conv_tc", "binarize", "conv_xnor", "quantize",
                                  "conv_int8", "maxpool", "upsample", "shortcut", "route_copy", "reorg",
                                  "yolo", "region", "conv_tc_i8", "conv_tc_tf32"};
    return (k >= 0 && k < 16) ? names[k] : "?";
}

enum { DT_F32 = 0, DT_BF16 = 1, DT_S8 = 2, DT_BITS = 3 };
static inline size_t dt_size(int dt) { return dt == DT_F32 ? 4 : dt == DT_BF16 ? 2 : dt == DT_S8 ? 1 : 4; }
// the <float> or <__nv_bfloat16> instantiation of kernel template k, for activations of dtype dt
#define BY_DT(k, dt) ((dt) == DT_F32 ? k<float> : k<__nv_bfloat16>)

// One launch of the op list.  `launch` is given the caller's NCHW images of the call, which only ops[0] reads: their pointer
// changes per call, so ops[0] runs outside the CUDA graph.  ops[0] may also read 8-bit HWC frames of the network size instead
// (`launch_u8`, when set).  `kernel` is the kernel an op launches directly (null for the ops that launch through a plan).
struct Op {
    int kind;
    int layer;
    std::function<void(const float *, cudaStream_t)> launch;
    std::function<void(const unsigned char *, cudaStream_t)> launch_u8;
    const void *kernel = nullptr;
};

struct ConvWeights {   // offsets into the weight arena
    size_t w = (size_t)-1;         // the filters in the layout of the layer's kernel (pack_weights)
    size_t bias = (size_t)-1, mean = (size_t)-1;
    int ldw = 0;      // f32 [K][ldw]
    int ldn = 0;      // rows of the [ldn][...] layouts
    int cpad = 0;     // padded channels of the s8 / bits / bf16 layouts
};

// The diagnostic YB_* switches of the library (DESIGN, appendix), read once when an engine is built; nothing else in the engine
// reads the environment (YB_XNOR_RULE, a network's initial XNOR rule, is read when the network is created).
struct Switches {
    bool no_graph, no_nccl, no_tc, no_tf32, no_stem, no_stem_tc, no_stem_u8, no_stem_pool_fuse, no_stem_s2_fuse,
         no_conv_pool_fuse, no_pool_fuse, no_yolo_fuse;
    bool no_fuse;       // YB_NO_FUSE=1: EngineOptions::fuse off
    bool xnor_tc;       // YB_XNOR_TC=0 puts every XNOR layer on the popcount kernels
    int xnor_tc_minc;   // narrowest XNOR layer on the tensor cores
    TcSwitches tc;      // the tensor-core plans'
    static Switches read() {
        auto set = [](const char *name) { return getenv(name) != nullptr; };
        auto num = [](const char *name) { const char *v = getenv(name); return v ? atoi(v) : 0; };
        const char *xtc = getenv("YB_XNOR_TC"), *minc = getenv("YB_XNOR_TC_MINC"), *nf = getenv("YB_NO_FUSE");
        return Switches{set("YB_NO_GRAPH"), set("YB_NO_NCCL"), set("YB_NO_TC"), set("YB_NO_TF32"), set("YB_NO_STEM"),
                        set("YB_NO_STEM_TC"), set("YB_NO_STEM_U8"), set("YB_NO_STEM_POOL_FUSE"), set("YB_NO_STEM_S2_FUSE"),
                        set("YB_NO_CONV_POOL_FUSE"), set("YB_NO_POOL_FUSE"), set("YB_NO_YOLO_FUSE"),
                        nf && nf[0] == '1', !(xtc && xtc[0] == '0'), minc ? atoi(minc) : 16,
                        // YB_TC_BN set to anything below 32 means 32
                        TcSwitches{set("YB_TC_BN") ? std::max(num("YB_TC_BN"), 1) : 0, num("YB_TC_GRID"), set("YB_TC_NO_BSTAT"),
                                   set("YB_TC_STATS"), num("YB_TC_DBG")}};
    }
};

struct Engine {
    EngineOptions opt;
    Switches sw{};
    int batch = 0;
    int act_dt = DT_F32;
    Stream stream;
    DevBuf<char> act_arena, w_arena;
    DevBuf<float> d_input;             // staging of the caller's images
    std::vector<TV> out_tv;            // per layer (base == nullptr: no NHWC output, or one that exists only in a fused form)
    std::vector<int> out_dt;
    struct Final { DevBuf<float> d; PinnedBuf<float> h; };   // a layer's f32 NCHW output and its pinned host mirror
    std::vector<Final> finals;         // per layer: the yolo / region outputs and the last layer's (empty for the others)
    std::vector<DevBuf<int32_t>> counts;   // per layer: optional raw integer results of a convolution
    std::vector<Op> ops;
    TV in0{};                          // NHWC copy of the caller's images (base == nullptr: the stem reads them directly)
    int in0_dt = DT_F32;
    GraphExec graph_exec;
    bool graph_failed = false;
    std::vector<std::pair<int, TcPlanPtr>> tc_plans;   // (layer, its tensor-core plan)
    int n_tc = 0;
    StemPlanPtr stem_plan;
    struct FrameStage {                 // the caller's 8-bit frames of one batch on the device, packed back to back
        DevBuf<unsigned char> buf;
        DevBuf<ImageGeo> d_geo; PinnedBuf<ImageGeo> h_geo;   // per-image table (batch entries) and its pinned host twin
    };
    FrameStage u8;                      // device-side input pipeline + decode geometry of the synchronous calls
    DevBuf<float> d_unit;               // byte value -> float /255. (k_resize_frames)
    // hand-off of the caller's device frames: produced on the caller's stream (ev_frames_ready) / read (ev_frames_read) /
    // drawn into (ev_frames_drawn)
    Event ev_frames_ready, ev_frames_read, ev_frames_drawn;
    // ---- pipelined end-to-end path: H2D(k+1) | compute(k) | D2H(k-1) on three streams -----------------
    struct DetWs {                      // decode + NMS workspace for `cap` candidate rows of `stride` floats per image
        DevBuf<float> rows; DevBuf<unsigned> mask; DevBuf<int> blkcnt, counts;
        int cap = 0, stride = 0;
    };
    struct Slot {
        DevBuf<float> d_in;
        std::vector<Final> out;         // raw tensors (mode 0), made by the first engine_submit on this slot
        Event ev_in, ev_comp, ev_done, ev_det;
        bool busy = false;
        // device-side input pipeline + decode of the pipelined detection path (engine_submit_frames)
        FrameStage u8;
        DetWs det;
        PinnedBuf<float> h_rows; PinnedBuf<int> h_counts;
        int mode = 0;                   // 0: raw tensors (engine_submit), 1: detections (engine_submit_frames)
        int nimg = 0;                   // images of the batch in this slot (mode 1)
        // drawing tickets (mode 1 with draw): the selected list in list order and the boxes in draw order (k_det_select),
        // and the list's pinned host copy, valid from the collect (collect_seq) until the slot is taken again
        bool draw = false;
        DevBuf<yb_detection> d_sel; DevBuf<DetDraw> d_draw; DevBuf<int> d_nsel;
        PinnedBuf<yb_detection> h_sel; PinnedBuf<int> h_nsel;
        unsigned long long collect_seq = 0;   // 0: no collected list
    };
    std::vector<Slot> slots;
    Stream s_in, s_out, s_det;
    int next_slot = 0;
    DetWs det;                          // workspace of the synchronous engine_detect
    ~Engine();
};

// Work may still be queued for uncollected tickets, or on a caller's stream (engine_forward); the members free themselves
// once it has finished.
Engine::~Engine() {
    cudaSetDevice(opt.device);
    cudaDeviceSynchronize();
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int grid_for(long total, int block = 256) {
    long g = (total + block - 1) / block;
    const long cap = 132L * 32;   // grid-stride kernels: a few waves of the 132 SMs
    return (int)std::max<long>(1, std::min(g, cap));
}

static TV make_tv(char *base, int N, int H, int W, int C, int ldc, int P, int dt, int coff) {
    TV t;
    t.base = base + (size_t)coff * dt_size(dt);
    t.N = N; t.H = H; t.W = W; t.C = C; t.ldc = ldc; t.P = P; t.Hp = H + 2 * P; t.Wp = W + 2 * P;
    return t;
}
static size_t tv_bytes(int N, int H, int W, int ldc, int P, int dt) {
    return (size_t)N * (H + 2 * P) * (W + 2 * P) * ldc * dt_size(dt);
}

// which layers read layer j's output
static std::vector<std::vector<int>> consumers_of(const Network &net) {
    const int nl = (int)net.layers.size();
    std::vector<std::vector<int>> cons(nl);
    for (int i = 0; i < nl; ++i) {
        const Layer &l = net.layers[i];
        if (l.type == YB_ROUTE) {
            for (int s : l.input_layers) cons[s].push_back(i);
        } else if (l.type != YB_BLANK) {
            if (i > 0) cons[i - 1].push_back(i);
            if (l.type == YB_SHORTCUT) cons[l.index].push_back(i);
        }
    }
    return cons;
}

template <typename T> struct same_type { using type = T; };   // keeps a parameter out of template argument deduction

// ---- engine build --------------------------------------------------------------------------------------------------------
// Four passes, in this order: plan_layers decides every kernel path and fusion, each layer output's dtype and home, and which
// outputs are materialised, and rejects the networks the engine cannot run; place allocates the activation buffers that some op
// writes; pack_weights fills the weight arena; the emit_* functions turn the plan into the op list in layer order, reading the
// plan only: each picks its kernel instantiation and launch shape once, and the op repeats that launch.

enum FirstOp { FIRST_NHWC, FIRST_STEM_SIMT, FIRST_STEM_TC, FIRST_STEM_S2, FIRST_STEM_POOL };

// The kernel family that runs a convolution
enum ConvKern { KERN_TC, KERN_SIMT, KERN_SMALLK };   // tensor-core plan, k_conv_simt, k_conv_xnor_smallk*

// What each arithmetic computes with: its converted input on the tensor-core tile and on the word kernels (k_conv_simt, the
// small-K kernels), the tile's kind (TC_BF16 stands for TC_TF32 under f32 activations), its k_conv_simt policy (null: the
// SimtF32 policy of the layer's activation types), the op kind of its CUDA-core convolution, and the numerator of the ALPHA1
// its epilogue reads besides the bias (0: none; the XNOR arithmetics read the filters' mean instead, arith_mean) --
// ..._quantized.c:598 (CPU rule, R_MULT), yolov2_forward_network_gpu.cu:200 (GPU rule, no R_MULT).
struct ArithRow {
    SideFmt side_tc, side_words;
    TcKind tc;
    void (*simt)(SimtP);
    int simt_op;
    int alpha1_num;
};
static const ArithRow kArith[] = {
    /* AR_F32          */ {SIDE_NONE, SIDE_NONE, TC_BF16, nullptr, OP_CONV_SIMT, 0},
    /* AR_XNOR_PM1_F32 */ {SIDE_PM1_F32, SIDE_PM1_F32, TC_BF16, nullptr, OP_CONV_SIMT, 0},
    /* AR_XNOR         */ {SIDE_PM1_S8, SIDE_BITS, TC_XNOR, k_conv_simt<SimtXnor>, OP_CONV_XNOR, 0},
    /* AR_XNOR_GPU     */ {SIDE_PM1_S8, SIDE_BITS, TC_XNOR_GPU, k_conv_simt<SimtXnorGpu>, OP_CONV_XNOR, 0},
    /* AR_PM1Z_GPU     */ {SIDE_PM1Z_S8, SIDE_PM1Z_S8, TC_PM1Z_GPU, k_conv_simt<SimtPm1zGpu>, OP_CONV_XNOR, 0},
    /* AR_INT8         */ {SIDE_S8, SIDE_S8, TC_S8, k_conv_simt<SimtInt8>, OP_CONV_INT8, 32},
    /* AR_INT8_GPU     */ {SIDE_S8_SAT, SIDE_S8_SAT, TC_S8_GPU, k_conv_simt<SimtInt8Gpu>, OP_CONV_INT8, 1},
};

struct LayerPlan {
    Arith arith = AR_F32;       // convolutions
    ConvKern kern = KERN_SIMT;  // convolutions
    int fused_into = -1;        // conv + shortcut: this convolution writes the shortcut's output
    bool fused_sc = false;      // shortcut computed in the epilogue of the convolution in front of it
    bool yolo_fused = false;    // conv: writes the [yolo] layer behind it from its epilogue; [yolo]: written that way
    SideFmt pool = SIDE_NONE;   // conv: runs the max-pool behind it and writes layer i+2's converted input (in its side format)
    bool pool_in_conv = false;  // max-pool: runs in the epilogue of the convolution in front of it
    bool pool_to_side = false;  // max-pool: writes the next convolution's converted input instead of its own output
    bool sc_bin = false;        // shortcut: behind a GPU-rule XNOR layer, whose bit GEMM adds it without its activation
    bool prefilled = false;     // conv: its converted input is written by the op in front of it
    bool in_first_op = false;   // computed by the op that reads the caller's images
    int out_dt = DT_F32;
    SideFmt side = SIDE_NONE;   // converted input of a convolution
    bool has_out = false;       // has an NHWC output: own buffer, channel slice of a route's buffer, or alias
    bool materialised = false;  // ... and some op writes it
    int owner = -1, coff = 0;   // channel slice at `coff` of route `owner`'s buffer (owner -1: own buffer or alias)
    int ldc = 0;                // pixel stride of an own buffer
};

// Stands in for the activation arena while the plan is made.  Every buffer starts 1024-byte aligned in the arena, so the
// predicates that check a view's alignment answer the same for views rooted here as for the placed ones.
static char *const kLayoutBase = reinterpret_cast<char *>(uintptr_t(1) << 40);

// calls put(filter, channel, tap, index into l.weights) for every weight of convolution l
template <typename F>
static void for_each_weight(const Layer &l, F &&put) {
    const int taps = l.size * l.size;
    for (int f = 0; f < l.n; ++f)
        for (int c = 0; c < l.c; ++c)
            for (int t = 0; t < taps; ++t) put(f, c, t, ((size_t)f * l.c + c) * taps + t);
}

// stem weights as by-value kernel constants: [27 = (ky,kx,c)][NF] + bias
template <int NF>
static StemW<NF> stem_weights(const Layer &l0) {
    StemW<NF> w{};
    for_each_weight(l0, [&](int f, int c, int t, size_t k) { w.w[(t * 3 + c) * NF + f] = l0.weights[k]; });
    for (int f = 0; f < l0.n; ++f) w.b[f] = l0.biases[f];
    return w;
}

namespace {
constexpr int P = 1;   // border of every activation buffer

struct Builder {
    Network &net;
    const EngineOptions &opt;
    Engine &e;
    const Switches &sw;
    const int B, nl;
    int ADT = DT_F32;
    std::vector<std::vector<int>> cons;
    std::vector<LayerPlan> L;
    int first = FIRST_NHWC;
    std::vector<size_t> buf_off, side_off;
    std::vector<ConvWeights> cw;
    size_t stem_w_off = (size_t)-1;

    Builder(Network &n, Engine &en)
        : net(n), opt(en.opt), e(en), sw(en.sw), B(n.batch), nl((int)n.layers.size()), cons(consumers_of(n)), L(nl),
          buf_off(nl, (size_t)-1), side_off(nl, (size_t)-1), cw(nl) {}

    const Layer &layer(int i) const { return net.layers[i]; }
    bool is_conv(int i) const { return layer(i).type == YB_CONVOLUTIONAL; }
    bool sole_reader(int i, int r) const { return cons[i].size() == 1 && cons[i][0] == r; }
    bool is_alias(int i) const { return layer(i).type == YB_ROUTE && layer(i).n == 1 && opt.fuse; }

    // The arithmetic of convolution i.  INT8 first, XNOR layers included: the CPU rule's yolov2_forward_network_q
    // (yolov2_forward_network_quantized.c:1036), the GPU rule's l.quantized (forward_network_gpu_cudnn_quantized,
    // yolov2_forward_network_gpu.cu:494-507).
    // CPU XNOR rule: XNOR layers with stride != 1 or pad != 1 never reach the bit GEMM in the reference:
    // forward_convolutional_layer_cpu binarises the input to +-1 floats (binarize_cpu, additionally.c:128-134), swaps in the +-mean
    // weights (binarize_weights, :113-126) and runs the ordinary im2col + gemm_nn (yolov2_forward_network.c:40-50, :204) --
    // out-of-image taps count 0 there, not -1.  Same here: k_binarize_pm1 + the exact-order float convolution.
    // GPU XNOR rule (forward_convolutional_layer_gpu_cudnn, yolov2_forward_network_gpu.cu:23-139): an XNOR layer below 32 channels
    // is a zero-padded +-1 convolution (path B); one with c % 32 == 0 runs the bit GEMM (path A), at every geometry.
    Arith conv_arith(int i) const {
        const Layer &l = layer(i);
        if (opt.rule == YB_QUANT_CPU && (i + opt.q_index_offset) >= 1 && l.activation != YB_LINEAR) return AR_INT8;
        if (opt.rule == YB_QUANT_GPU && l.quantized) return AR_INT8_GPU;
        if (!l.xnor) return AR_F32;
        if (opt.xnor_rule == YB_XNOR_GPU) return l.c < 32 ? AR_PM1Z_GPU : AR_XNOR_GPU;
        return l.stride == 1 && l.pad == 1 ? AR_XNOR : AR_XNOR_PM1_F32;
    }
    // XNOR layers with enough channels run on the tensor cores as +-1 int8 (dot == 2*count - K, exact); the small ones stay on
    // the popcount kernels.  Channels are padded to a multiple of 32 with zero WEIGHT bytes (whatever the activation pad bytes
    // hold contributes 0), so even the 16- and 32-channel layers run there: the popcount kernels are bound by the 16 POPC/clk/SM
    // of the integer pipe, while the same layers as +-1 bytes on the s8 tensor cores are not.  Under the GPU XNOR rule only
    // where the tile takes the activation; the others stay on the CUDA cores.
    bool xnor_tc(int i) const {
        const Layer &l = layer(i);
        return sw.xnor_tc && l.c % 16 == 0 && l.c >= sw.xnor_tc_minc && l.size == 3 && l.stride == 1 && l.pad == 1 && l.n >= 8 &&
               (L[i].arith == AR_XNOR || l.activation == YB_LEAKY || l.activation == YB_LINEAR);
    }
    // a [shortcut] the GPU build folds into XNOR layer i's bit GEMM (calculate_binary_weights, additionally.c:326-338)
    bool bin_shortcut(int i) const {
        if (opt.xnor_rule != YB_XNOR_GPU || !layer(i).xnor || i + 1 >= nl) return false;
        const Layer &s = layer(i + 1);
        return s.type == YB_SHORTCUT && s.w == s.out_w && s.h == s.out_h && s.c == s.out_c;
    }

    // conv i -> 2x2/2 max-pool i+1 -> integer conv i+2, nothing else reading i or i+1: the pool and the next layer's input
    // conversion may run in conv i's epilogue.  Returns layer i+2's side format, or SIDE_NONE.
    SideFmt conv_pool_fmt(int i) const {
        if (!opt.fuse || opt.keep_counts || sw.no_conv_pool_fuse || i + 2 >= nl) return SIDE_NONE;
        const Layer &mp = layer(i + 1);
        if (mp.type != YB_MAXPOOL || mp.size != 2 || mp.stride != 2 || mp.pad != 1 || !is_conv(i + 2)) return SIDE_NONE;
        if (!sole_reader(i, i + 1) || !sole_reader(i + 1, i + 2)) return SIDE_NONE;
        return side_int(L[i + 2].side) ? L[i + 2].side : SIDE_NONE;
    }

    // layer i's NHWC output view; buf(j) is the start of layer j's own buffer
    template <typename F>
    TV out_view(int i, F &&buf) const {
        const Layer &l = layer(i);
        if (is_alias(i)) return out_view(l.input_layers[0], buf);
        if (L[i].owner >= 0)
            return make_tv(buf(L[i].owner), B, l.out_h, l.out_w, l.out_c, L[L[i].owner].ldc, P, ADT, L[i].coff);
        return make_tv(buf(i), B, l.out_h, l.out_w, l.out_c, L[i].ldc, P, L[i].out_dt, 0);
    }
    TV layout_view(int i) const { return L[i].has_out ? out_view(i, [](int) { return kLayoutBase; }) : TV{}; }
    TV in0_view(char *base) const { return make_tv(base, B, net.h, net.w, net.c, net.c, P, ADT, 0); }
    TV layout_in(int i) const { return i == 0 ? in0_view(kLayoutBase) : layout_view(i - 1); }
    int in_dt(int i) const { return i == 0 ? ADT : L[i - 1].out_dt; }
    // pixel stride of convolution i's converted input: +-1 floats, sign words, or bytes over channels padded to a multiple of 32
    int side_ld(int i) const {
        const int c = layer(i).c;
        return L[i].side == SIDE_PM1_F32 ? c : (int)align_up(c, 32) / (L[i].side == SIDE_BITS ? 32 : 1);
    }
    TV side_view(int i, char *base) const {
        const Layer &l = layer(i);
        const int ld = side_ld(i);
        if (L[i].side == SIDE_PM1_F32) return make_tv(base, B, l.h, l.w, l.c, ld, P, DT_F32, 0);
        if (L[i].side == SIDE_BITS) return make_tv(base, B, l.h, l.w, ld, ld, P, DT_BITS, 0);
        return make_tv(base, B, l.h, l.w, l.c, ld, P, DT_S8, 0);
    }
    TV side_placed(int i) const { return side_view(i, e.act_arena.get() + side_off[i]); }
    // the multiplier of layer i's side conversion: the input multiplier of an INT8 layer, unused otherwise
    float side_mult(int i) const { return side_s8(L[i].side) ? layer(i).input_quant_multipler : 0.f; }
    float alpha1(int i) const {
        const Layer &l = layer(i);
        return kArith[L[i].arith].alpha1_num / (l.input_quant_multipler * l.weights_quant_multipler);
    }
    TcKind tc_kind(int i) const { return L[i].arith == AR_F32 && ADT == DT_F32 ? TC_TF32 : kArith[L[i].arith].tc; }

    // Convolution i as a tensor-core convolution, with the shortcut and [yolo] fusions of its plan and the max-pool fusion `pool`
    // (layer i+2's side format, or SIDE_NONE).  placed == false: views rooted at kLayoutBase and no device pointers, for the
    // queries of the layer plan; true: the placed buffers, the packed weights and the raw-count buffer (keep_counts) that
    // counts_buffer made.
    TcConv tc_conv(int i, bool placed, SideFmt pool) const {
        const Layer &l = layer(i);
        const LayerPlan &p = L[i];
        const int tgt = p.fused_into >= 0 ? p.fused_into : i;
        auto out = [&](int j) { return placed ? e.out_tv[j] : layout_view(j); };
        auto side = [&](int j) { return placed ? side_placed(j) : side_view(j, kLayoutBase); };
        TcConv c;
        c.kind = tc_kind(i);
        c.l = &l;
        c.in = p.side != SIDE_NONE ? side(i) : !placed ? layout_in(i) : i == 0 ? e.in0 : e.out_tv[i - 1];
        c.out = out(tgt);
        c.out_bf16 = L[tgt].out_dt == DT_BF16;
        if (p.fused_into >= 0) {
            c.res = out(layer(tgt).index);
            c.act2 = layer(tgt).activation;
        }
        c.pool_fmt = pool;
        if (pool != SIDE_NONE) {
            c.pool_mult = side_mult(i + 2);
            c.pool_next = side(i + 2);
        }
        c.sw = sw.tc;
        if (!placed) return c;
        // filters: [ldn][K] bf16, f32 (K-major copy) or s8 / +-1 bytes ([taps][cpad] per filter)
        c.w = e.w_arena.get() + cw[i].w;
        c.ldn = cw[i].ldn;
        c.bias = bias(i);
        if (kArith[p.arith].alpha1_num) c.alpha1 = alpha1(i);
        if (arith_mean(p.arith)) c.mean = mean(i);
        c.acc_out = e.counts[i].get();
        if (p.yolo_fused) {
            c.yolo_out = e.finals[i + 1].d.get();
            c.yolo_classes = layer(i + 1).classes;
        }
        return c;
    }

    // ---- pass 1: the layer plan ------------------------------------------------------------------------------------------
    void plan_layers() {
        // no reference binary runs the CPU build's INT8 forward with the GPU build's XNOR arithmetic
        if (opt.rule == YB_QUANT_CPU && opt.xnor_rule == YB_XNOR_GPU)
            fatal_throw("engine: the GPU XNOR rule runs with quantized = 0 or 2 (YB_QUANT_GPU), not with the CPU INT8 rule (quantized = 1)");
        bool any_xnor = false;
        for (int i = 0; i < nl; ++i) {
            const Layer &l = layer(i);
            if (l.type != YB_CONVOLUTIONAL) continue;
            if (l.batch_normalize) fatal_throw("engine: batch-norm not folded -- call yb_fuse_conv_batchnorm first");
            L[i].arith = conv_arith(i);
            if (l.xnor) {
                any_xnor = true;
                if (!l.has_mean_arr) fatal_throw("engine: xnor layer without mean_arr -- call yb_calculate_binary_weights first");
            }
            // the CPU rule reads every convolution's int8 weights (yolov2_forward_network_q), the GPU rule its INT8 layers'
            if ((opt.rule == YB_QUANT_CPU || L[i].arith == AR_INT8_GPU) && !l.has_int8)
                fatal_throw("engine: -quantized rule without int8 weights -- call yb_quantinization_and_get_multipliers first");
        }
        // f32 activations whenever an integer path must see exactly the reference's inputs; the GPU rule keeps float tensors
        // between layers as the reference's GPU build does
        ADT = (opt.rule != YB_QUANT_NONE || any_xnor || opt.precision == YB_PREC_FP32) ? DT_F32 : DT_BF16;

        // conv i + same-shape shortcut i+1 whose only reader is that shortcut
        if (opt.fuse) {
            for (int i = 0; i + 1 < nl; ++i) {
                const Layer &l = layer(i), &s = layer(i + 1);
                if (l.type != YB_CONVOLUTIONAL || s.type != YB_SHORTCUT) continue;
                if (L[i].arith != AR_F32) continue;
                if (l.stride != 1) continue;   // the tensor-core stride-2 path stores straddling tiles row by row, without a residual
                if (!sole_reader(i, i + 1)) continue;
                if (s.index == i) continue;
                if (!(s.w == s.out_w && s.h == s.out_h && s.c == s.out_c)) continue;
                L[i].fused_into = i + 1;
                L[i + 1].fused_sc = true;
            }
        }

        for (int i = 0; i + 1 < nl; ++i)
            if (is_conv(i) && bin_shortcut(i)) L[i + 1].sc_bin = true;

        // output dtypes and homes (own buffer, or a channel slice of a concat buffer)
        for (int i = 0; i < nl; ++i) {
            const Layer &l = layer(i);
            L[i].has_out = !(l.type == YB_YOLO || l.type == YB_REGION || l.type == YB_BLANK) && L[i].fused_into < 0 &&
                           l.out_h > 0 && l.out_w > 0 && l.out_c > 0;
            L[i].materialised = L[i].has_out;   // until a fusion below takes the output away
            L[i].out_dt = ADT;
            if (l.type == YB_CONVOLUTIONAL && !cons[i].empty()) {
                bool all_final = true;
                for (int c : cons[i]) if (layer(c).type != YB_YOLO && layer(c).type != YB_REGION) all_final = false;
                if (all_final) L[i].out_dt = DT_F32;   // detection heads stay f32 (bf16 would cost ~1e-3 rel by itself)
            }
            if (l.type == YB_CONVOLUTIONAL && cons[i].empty()) L[i].out_dt = DT_F32;
            // pixel stride rounded up to 8 channels: 16-byte aligned rows for TMA / vector stores (e.g. 255 -> 256)
            L[i].ldc = (int)align_up(l.out_c, 8);
        }
        if (opt.fuse) {
            for (int r = 0; r < nl; ++r) {
                const Layer &l = layer(r);
                if (l.type != YB_ROUTE || l.n < 2 || l.out_c <= 0) continue;
                int off = 0;
                for (int k = 0; k < l.n; ++k) {
                    const int j = l.input_layers[k];
                    if (L[j].has_out && L[j].owner < 0 && layer(j).type != YB_ROUTE && L[j].out_dt == ADT) {
                        L[j].owner = r;
                        L[j].coff = off;
                    }
                    off += layer(j).out_c;
                }
            }
        }
        for (int i = 0; i < nl; ++i)
            if (L[i].has_out && is_alias(i)) L[i].out_dt = L[layer(i).input_layers[0]].out_dt;

        // each convolution's kernel family, then its converted input: the tile's format is what the tile is asked about
        for (int i = 0; i < nl; ++i) {
            if (!is_conv(i)) continue;
            LayerPlan &p = L[i];
            p.side = kArith[p.arith].side_tc;
            p.kern = conv_kern(i);
            if (p.kern != KERN_TC) p.side = kArith[p.arith].side_words;
        }
        plan_first_op();
        plan_fusions();
        for (int i = 0; i < nl; ++i)
            if (is_alias(i)) L[i].materialised = L[i].has_out && L[layer(i).input_layers[0]].materialised;
        reject_unsupported();
    }

    // the networks the op list cannot express, rejected before anything is allocated
    void reject_unsupported() const {
        for (int i = 0; i < nl; ++i) {
            const Layer &l = layer(i);
            const LayerPlan &p = L[i];
            // a fused shortcut reads the output of the convolution in front of it as that convolution's accumulators
            const bool reads_prev = l.type == YB_CONVOLUTIONAL || l.type == YB_MAXPOOL || l.type == YB_UPSAMPLE || l.type == YB_REORG ||
                                    l.type == YB_YOLO || l.type == YB_REGION || (l.type == YB_SHORTCUT && !p.fused_sc);
            if (reads_prev && i > 0 && !L[i - 1].has_out) fatal_throw("engine: layer " + std::to_string(i) + " has no image input");
            switch (l.type) {
            case YB_CONVOLUTIONAL: {
                if (!L[p.fused_into >= 0 ? p.fused_into : i].has_out) fatal_throw("engine: conv output not placed");
                if (opt.xnor_rule == YB_XNOR_GPU && l.xnor) reject_gpu_xnor_rule(i);
                const int in_c = i == 0 ? net.c : layer(i - 1).out_c, in_h = i == 0 ? net.h : layer(i - 1).out_h,
                          in_w = i == 0 ? net.w : layer(i - 1).out_w;
                if (in_c != l.c || in_h != l.h || in_w != l.w) fatal_throw("engine: conv input shape mismatch");
                break;
            }
            case YB_UPSAMPLE:
                if (l.reverse) fatal_throw("engine: reverse upsample (downsample) is not supported");
                break;
            case YB_REORG:
                if (l.reverse) fatal_throw("engine: reverse reorg is not supported");
                break;
            case YB_SHORTCUT:
                if (!L[l.index].materialised) fatal_throw("engine: shortcut source not placed");
                // shortcut_cpu's asserts (yolov2_forward_network.c:414-415): the subsampling step taken from the widths must
                // also be the one of the heights, or the rows read from `from` run past it
                if (l.w / l.out_w != l.h / l.out_h || l.out_w / l.w != l.out_h / l.h)
                    fatal_throw("engine: shortcut from layer " + std::to_string(l.index) + " (" + std::to_string(l.w) + "x" +
                                std::to_string(l.h) + ") onto " + std::to_string(l.out_w) + "x" + std::to_string(l.out_h) +
                                ": the two scale by different factors in width and height");
                break;
            case YB_REGION:
                // the reference's forward and both decoders take the objectness at entry 4 and the classes from entry 5
                if (l.coords != 4) fatal_throw("engine: [region] coords=" + std::to_string(l.coords) + " is not supported (only 4)");
                break;
            case YB_ROUTE:
                if (!p.has_out) fatal_throw("engine: route over layers of different spatial size is not supported");
                if (is_alias(i)) break;
                for (int j : l.input_layers)
                    if (L[j].owner != i && !L[j].materialised) fatal_throw("engine: route source not placed");
                break;
            default:
                break;
            }
        }
    }

    // the XNOR layers the GPU XNOR rule cannot state as a convolution
    void reject_gpu_xnor_rule(int i) const {
        const Layer &l = layer(i);
        const std::string at = "engine: GPU XNOR rule: XNOR layer " + std::to_string(i) + " (" + std::to_string(l.c) + " channels) ";
        // the bit GEMM without the weight inversion (additionally.c:221-261): a sign-flipped, offset value read from
        // alignment bits of an uninitialised workspace
        if (l.c >= 32 && l.c % 32 != 0) fatal_throw(at + "has c >= 32 and c % 32 != 0, where the reference computes no convolution");
        if (!(i + 1 < nl && L[i + 1].sc_bin)) return;
        // the GPU build turns the shortcut into a blank layer and only the bit GEMM writes its output
        if (L[i].arith == AR_INT8_GPU) fatal_throw(at + "runs in INT8, so nothing writes the output of the [shortcut] behind it");
        if (L[i].arith == AR_PM1Z_GPU) fatal_throw(at + "is a +-1 convolution below 32 channels, so nothing writes the output of the [shortcut] behind it");
        // the sum takes the leaky-only value, which the engine keeps as the layer's output for leaky and linear layers only
        if (l.activation != YB_LEAKY && l.activation != YB_LINEAR)
            fatal_throw(at + "is followed by a [shortcut] and has an activation other than leaky or linear, which is not supported");
    }

    // the kernel family of convolution i, with L[i].side the tile's input format
    ConvKern conv_kern(int i) const {
        const Layer &l = layer(i);
        const LayerPlan &p = L[i];
        const int tgt = p.fused_into >= 0 ? p.fused_into : i;
        const TV tin = layout_in(i), tout = layout_view(tgt);
        const int idt = in_dt(i), odt = L[tgt].out_dt;
        const TcConv tc_query = tc_conv(i, false, SIDE_NONE);
        if (p.arith == AR_F32) {
            bool tc = ADT == DT_BF16 && idt == DT_BF16 && tc_conv_supported(tc_query);
            // float detection heads of the INT8 / XNOR networks (default precision): tf32 wgmma.  Only layers whose every
            // reader is a yolo / region layer -- nothing they compute can reach an integer layer, which stays bit-exact
            // against the CPU reference.  The GPU rule's float layers are cuDNN convolutions in the reference, which no
            // summation order reproduces bit for bit: all of them that the tensor cores take run on tf32.
            if (ADT == DT_F32 && opt.precision == YB_PREC_BF16_TC && idt == DT_F32 && odt == DT_F32 && p.fused_into < 0 &&
                !cons[i].empty() && !sw.no_tf32) {
                bool heads_only = true;
                for (int r : cons[i]) heads_only &= layer(r).type == YB_YOLO || layer(r).type == YB_REGION;
                if ((heads_only || opt.rule == YB_QUANT_GPU) && tc_conv_supported(tc_query)) tc = true;
            }
            return tc && !sw.no_tc ? KERN_TC : KERN_SIMT;
        }
        const bool int8 = p.arith == AR_INT8 || p.arith == AR_INT8_GPU;
        if (idt != DT_F32 || odt != DT_F32)
            fatal_throw(int8 ? "engine: int8 path needs f32 activations" : "engine: xnor path needs f32 activations");
        if (int8) return (!sw.no_tc && tc_conv_supported(tc_query)) ? KERN_TC : KERN_SIMT;
        if (p.arith == AR_PM1Z_GPU) return (xnor_tc(i) && tc_conv_supported(tc_query)) ? KERN_TC : KERN_SIMT;
        if (p.arith == AR_XNOR_PM1_F32) return KERN_SIMT;
        if (xnor_tc(i) && vec16_view(tin, 4)) {
            if (!tc_conv_supported(tc_query)) fatal_throw("engine: xnor tensor-core layer not supported by the i8 tile");
            return KERN_TC;
        }
        // small K: one thread per pixel, all filters (weights broadcast from shared memory), over CW sign words per tap.  It
        // stores 4 filters per float4, so every pixel of its output must be 16-byte aligned: a channel slice of a route's
        // buffer may not be.
        const int CW = (l.c + 31) / 32;
        if (CW <= 2 && l.size == 3 && l.stride == 1 && l.pad == 1 && (size_t)l.n * 9 * CW * 4 <= 40 * 1024 && vec16_view(tout, 4))
            return KERN_SMALLK;
        return KERN_SIMT;
    }

    // ops[0] consumes the caller's NCHW f32 images.  Usually that is the stem convolution itself (3 input channels, 3x3/1/1),
    // reading NCHW directly; otherwise a plain NCHW -> padded-NHWC conversion.  The stems store whole 16-byte groups of
    // filters (k_conv_stem: float4 / 8 bf16; k_stem_tc: 16-byte rows), so each output pixel must start 16-byte aligned; a stem
    // writing a channel slice of a route's buffer at an unaligned offset runs as a plain convolution behind the conversion.
    void plan_first_op() {
        const Layer &l0 = layer(0);
        const TV out0 = layout_view(0);
        const bool out_vec = vec16_view(out0, (int)dt_size(L[0].out_dt));
        const bool stem_ok = l0.type == YB_CONVOLUTIONAL && L[0].arith == AR_F32 && L[0].kern == KERN_SIMT && l0.c == 3 &&
                             l0.size == 3 && l0.stride == 1 && l0.pad == 1 && (l0.n == 16 || l0.n == 32) && L[0].fused_into < 0 &&
                             L[0].has_out && !sw.no_stem && out_vec;
        // exact nets: stem + 2x2/2 max-pool + the integer layer's input conversion in one kernel (k_stem_pool): layers 0 and 1
        // are then never written to HBM
        bool pool_ok = stem_ok && opt.fuse && L[0].out_dt == DT_F32 && l0.n == 16 && nl > 2 && !sw.no_stem_pool_fuse &&
                       (l0.activation == YB_LEAKY || l0.activation == YB_LINEAR);
        if (pool_ok) {
            const Layer &mp = layer(1), &c2 = layer(2);
            pool_ok = mp.type == YB_MAXPOOL && mp.size == 2 && mp.stride == 2 && mp.pad == 1 && sole_reader(0, 1) &&
                      sole_reader(1, 2) && c2.type == YB_CONVOLUTIONAL && side_int(L[2].side) &&
                      (L[2].side == SIDE_BITS || side_ld(2) % 16 == 0);
        }
        if (pool_ok) {
            first = FIRST_STEM_POOL;
        } else if (stem_ok && L[0].out_dt == DT_BF16 && tc_stem_supported(l0, out0) && !sw.no_stem_tc) {
            // tensor-core stem: gathers the 3x3x3 window from NCHW, K padded 27 -> 32.  When layer 1 is a bf16 tensor-core
            // 3x3 / stride-2 convolution 32 -> 64 and the stem's only reader, both run as one kernel (k_stem_s2_tc) and the
            // stem output is never written.
            const bool s2 = opt.fuse && !sw.no_stem_s2_fuse && nl > 1 && sole_reader(0, 1) && is_conv(1) && L[1].arith == AR_F32 &&
                            L[1].kern == KERN_TC && L[1].fused_into < 0 && L[1].out_dt == DT_BF16 &&
                            tc_stem_s2_supported(l0, layer(1), layout_view(1));
            first = s2 ? FIRST_STEM_S2 : FIRST_STEM_TC;
        } else if (stem_ok) {
            first = FIRST_STEM_SIMT;
        }
        if (first != FIRST_NHWC) L[0].in_first_op = true;
        if (first == FIRST_STEM_S2 || first == FIRST_STEM_POOL) {
            L[0].materialised = false;
            L[1].in_first_op = true;
        }
        if (first == FIRST_STEM_POOL) {
            L[1].materialised = false;
            L[2].prefilled = true;
        }
    }

    // the fusions in the op list behind the first op
    void plan_fusions() {
        for (int i = 0; i < nl; ++i) {
            LayerPlan &p = L[i];
            if (!is_conv(i) || p.in_first_op) continue;
            // max-pool i+1 and layer i+2's input conversion in the epilogue
            const SideFmt pf = conv_pool_fmt(i);
            bool pool = false;
            if (p.kern == KERN_TC && p.arith != AR_F32) {
                pool = pf != SIDE_NONE && tc_conv_supported(tc_conv(i, false, pf));
            } else if (p.kern == KERN_SMALLK) {
                pool = pf == SIDE_PM1_S8 || pf == SIDE_BITS;
            }
            if (pool) {
                p.pool = pf;
                L[i + 1].pool_in_conv = L[i + 2].prefilled = true;
                p.materialised = L[i + 1].materialised = false;
            }
            // detection-head conv i + [yolo] i+1: logistic and NCHW store in the epilogue
            if (p.kern == KERN_TC && p.arith == AR_F32 && opt.fuse && p.fused_into < 0 && p.out_dt == DT_F32 && i + 1 < nl &&
                layer(i + 1).type == YB_YOLO && sole_reader(i, i + 1) && !sw.no_yolo_fuse) {
                p.yolo_fused = L[i + 1].yolo_fused = true;
                p.materialised = false;
            }
        }
        // max-pool -> integer convolution: the pool writes the convolution's s8 / sign input directly (same values in the same
        // order as max-pool + quantise / binarise; the pooled f32 tensor never goes to HBM)
        for (int i = 0; i + 1 < nl; ++i) {
            if (layer(i).type != YB_MAXPOOL || L[i].in_first_op || L[i].pool_in_conv) continue;
            const Layer &c = layer(i + 1);
            if (opt.fuse && in_dt(i) == DT_F32 && sole_reader(i, i + 1) && c.type == YB_CONVOLUTIONAL && side_int(L[i + 1].side) &&
                !sw.no_pool_fuse) {
                L[i].pool_to_side = L[i + 1].prefilled = true;
                L[i].materialised = false;
            }
        }
    }

    // ---- pass 2: placement -----------------------------------------------------------------------------------------------
    void place() {
        size_t total = 0;
        auto take = [&](size_t bytes) { const size_t off = total; total += align_up(bytes, 1024); return off; };
        const size_t in0_off = first == FIRST_NHWC ? take(tv_bytes(B, net.h, net.w, net.c, P, ADT)) : 0;
        for (int i = 0; i < nl; ++i) {
            const Layer &l = layer(i);
            if (L[i].materialised && !is_alias(i) && L[i].owner < 0)
                buf_off[i] = take(tv_bytes(B, l.out_h, l.out_w, L[i].ldc, P, L[i].out_dt));
        }
        for (int i = 0; i < nl; ++i) {
            const Layer &l = layer(i);
            const int sdt = L[i].side == SIDE_PM1_F32 ? DT_F32 : L[i].side == SIDE_BITS ? DT_BITS : DT_S8;
            if (L[i].side != SIDE_NONE) side_off[i] = take(tv_bytes(B, l.h, l.w, side_ld(i), P, sdt));
        }
        e.act_arena.ensure(total);
        CUDA_OK(cudaMemsetAsync(e.act_arena.get(), 0, total, e.stream));   // zero borders, once
        for (int i = 0; i < nl; ++i)   // +-1 activation buffers: borders are -1 (out-of-image taps count as -1, SURVEY F9)
            if (L[i].side == SIDE_PM1_S8)
                CUDA_OK(cudaMemsetAsync(e.act_arena.get() + side_off[i], 0xFF, tv_bytes(B, layer(i).h, layer(i).w, side_ld(i), P, DT_S8), e.stream));
        e.in0 = first == FIRST_NHWC ? in0_view(e.act_arena.get() + in0_off) : TV{};
        e.in0_dt = ADT;
        e.act_dt = ADT;
        e.out_tv.assign(nl, TV{});
        e.out_dt.assign(nl, ADT);
        for (int i = 0; i < nl; ++i) {
            e.out_dt[i] = L[i].out_dt;
            if (L[i].materialised) e.out_tv[i] = out_view(i, [&](int j) { return e.act_arena.get() + buf_off[j]; });
        }
    }

    // detection-layer outputs, and the last layer's output whatever its type (the reference returns it)
    void place_finals() {
        e.finals.resize(nl);
        e.counts.resize(nl);
        for (int i = 0; i < nl; ++i) {
            const Layer &l = layer(i);
            if (!(l.type == YB_YOLO || l.type == YB_REGION || (i == nl - 1 && l.outputs > 0))) continue;
            e.finals[i].d.ensure((size_t)l.outputs * B);
            e.finals[i].h.ensure((size_t)l.outputs * B);
        }
    }

    // ---- pass 3: weights -------------------------------------------------------------------------------------------------
    void pack_weights() {
        std::vector<char> hostw;
        auto reserve = [&](size_t bytes) { size_t off = align_up(hostw.size(), 1024); hostw.resize(off + bytes, 0); return off; };
        for (int i = 0; i < nl; ++i) {
            if (!is_conv(i)) continue;
            const Layer &l = layer(i);
            const LayerPlan &p = L[i];
            const int taps = l.size * l.size, K = taps * l.c;
            ConvWeights &w = cw[i];
            w.bias = reserve(sizeof(float) * align_up(l.n, 64));
            memcpy(&hostw[w.bias], l.biases.data(), sizeof(float) * l.n);
            w.ldn = (int)align_up(l.n, 64);
            if (p.kern == KERN_TC && p.side == SIDE_NONE && ADT == DT_F32) {
                // tf32: f32 [ldn][K], K ordered (ky, kx, c)
                w.w = reserve(sizeof(float) * (size_t)w.ldn * K);
                float *dst = reinterpret_cast<float *>(&hostw[w.w]);
                for_each_weight(l, [&](int f, int c, int t, size_t k) { dst[(size_t)f * K + (size_t)t * l.c + c] = l.weights[k]; });
            } else if (p.kern == KERN_TC && p.side == SIDE_NONE) {
                // bf16 [ldn][K], K ordered (ky, kx, c): the K-major B operand of the implicit GEMM
                w.w = reserve(sizeof(__nv_bfloat16) * (size_t)w.ldn * K);
                __nv_bfloat16 *dst = reinterpret_cast<__nv_bfloat16 *>(&hostw[w.w]);
                for_each_weight(l, [&](int f, int c, int t, size_t k) {
                    dst[(size_t)f * K + (size_t)t * l.c + c] = __float2bfloat16_rn(l.weights[k]); });
            } else if (!side_int(p.side)) {
                // f32 [K][ldw]; K ordered (ky, kx, c), or -- f32 activations: the exact order of the reference's gemm_nn
                // (k_conv_simt<EXACT>) -- (c, ky, kx).  +-1 float inputs: +mean where w > 0, -mean otherwise (binarize_weights).
                const bool pm1 = p.side == SIDE_PM1_F32;
                w.ldw = w.ldn;
                w.w = reserve(sizeof(float) * (size_t)K * w.ldw);
                float *dst = reinterpret_cast<float *>(&hostw[w.w]);
                for_each_weight(l, [&](int f, int c, int t, size_t k) {
                    dst[(ADT == DT_F32 ? (size_t)c * taps + t : (size_t)t * l.c + c) * w.ldw + f] =
                        pm1 ? (l.weights[k] > 0 ? l.mean_arr[f] : -l.mean_arr[f]) : l.weights[k]; });
            } else if (p.side == SIDE_BITS) {
                // sign bits [ldn][taps][CW]; bit = (w > 0) (binarize_weights additionally.c:113 + float_to_bit :1536)
                const int CW = side_ld(i);
                w.cpad = CW * 32;
                w.w = reserve(sizeof(uint32_t) * (size_t)w.ldn * taps * CW);
                uint32_t *dst = reinterpret_cast<uint32_t *>(&hostw[w.w]);
                for_each_weight(l, [&](int f, int c, int t, size_t k) {
                    if (l.weights[k] > 0) dst[((size_t)f * taps + t) * CW + c / 32] |= 1u << (c & 31); });
            } else {
                // s8 [ldn][taps][cpad], zero channel padding and zero padded filter rows: INT8 weights, or XNOR weights as
                // +1 where w > 0 and -1 otherwise
                w.cpad = side_ld(i);
                w.w = reserve((size_t)w.ldn * taps * w.cpad);
                int8_t *dst = reinterpret_cast<int8_t *>(&hostw[w.w]);
                for_each_weight(l, [&](int f, int c, int t, size_t k) {
                    dst[((size_t)f * taps + t) * w.cpad + c] = side_s8(p.side) ? l.weights_int8[k] : l.weights[k] > 0 ? 1 : -1; });
            }
            if (arith_mean(p.arith)) {
                w.mean = reserve(sizeof(float) * align_up(l.n, 64));
                memcpy(&hostw[w.mean], l.mean_arr.data(), sizeof(float) * l.n);
            }
        }
        if (first == FIRST_STEM_TC || first == FIRST_STEM_S2) {
            // bf16 [32 filters][32], K = (ky, kx, c) padded 27 -> 32
            stem_w_off = reserve(sizeof(__nv_bfloat16) * 32 * 32);
            __nv_bfloat16 *dst = reinterpret_cast<__nv_bfloat16 *>(&hostw[stem_w_off]);
            for (int k = 0; k < 32 * 32; ++k) dst[k] = __float2bfloat16_rn(0.f);
            const Layer &l0 = layer(0);
            for_each_weight(l0, [&](int f, int c, int t, size_t k) { dst[f * 32 + t * 3 + c] = __float2bfloat16_rn(l0.weights[k]); });
        }
        e.w_arena.ensure(align_up(std::max<size_t>(hostw.size(), 1024), 1024));
        if (opt.upload) CUDA_OK(cudaMemcpyAsync(e.w_arena.get(), hostw.data(), hostw.size(), cudaMemcpyHostToDevice, e.stream));
        CUDA_OK(cudaStreamSynchronize(e.stream));   // hostw goes out of scope below
    }

    // ---- pass 4: op emission ---------------------------------------------------------------------------------------------
    const float *bias(int i) const { return reinterpret_cast<const float *>(e.w_arena.get() + cw[i].bias); }
    const float *mean(int i) const { return reinterpret_cast<const float *>(e.w_arena.get() + cw[i].mean); }
    void push(int kind, int i, std::function<void(const float *, cudaStream_t)> f, const void *kernel = nullptr) {
        e.ops.push_back(Op{kind, i, std::move(f), nullptr, kernel});
    }
    // an op that launches kernel k with these arguments, converted to the kernel's parameter types here
    template <typename... A>
    void push_kernel(int kind, int i, void (*k)(A...), dim3 grid, dim3 block, size_t smem, typename same_type<A>::type... args) {
        push(kind, i, [=](const float *, cudaStream_t s) { k<<<grid, block, smem, s>>>(args...); }, reinterpret_cast<const void *>(k));
    }
    // ops[0] as a kernel whose first argument is the caller's images
    template <typename... A>
    void push_input_kernel(int kind, int i, void (*k)(const float *, A...), dim3 grid, dim3 block, typename same_type<A>::type... args) {
        push(kind, i, [=](const float *in, cudaStream_t s) { k<<<grid, block, 0, s>>>(in, args...); }, reinterpret_cast<const void *>(k));
    }

    // the tensor-core plan of layer i, with the [yolo] layer or the max-pool the layer plan fuses
    void push_tc_plan(int i) {
        const TcKind kind = tc_kind(i);
        e.tc_plans.emplace_back(i, tc_make_plan(tc_conv(i, true, L[i].pool)));
        const TcPlan *plan = e.tc_plans.back().second.get();
        if (kind == TC_BF16 || kind == TC_TF32) ++e.n_tc;
        push(kind == TC_BF16 ? OP_CONV_TC : kind == TC_TF32 ? OP_CONV_TC_TF32 : OP_CONV_TC_I8, i,
             [plan](const float *, cudaStream_t s) { tc_launch(*plan, s); });
    }

    int32_t *counts_buffer(int i) {   // raw XNOR popcounts / INT8 accumulators (keep_counts)
        if (!opt.keep_counts) return nullptr;
        const Layer &l = layer(i);
        e.counts[i].ensure((size_t)B * l.n * l.out_h * l.out_w);
        return e.counts[i].get();
    }

    // ops[0]: reads the caller's images
    void emit_first() {
        const Layer &l0 = layer(0);
        const int act = l0.activation, H = l0.h, W = l0.w;
        if (first == FIRST_STEM_POOL) {
            // by layer 2's side format (SIDE_S8, SIDE_PM1_S8, SIDE_BITS, SIDE_S8_SAT, SIDE_PM1Z_S8) and the stem's activation
            decltype(&k_stem_pool<SIDE_S8, ACT_LEAKY>) const k[5][2] = {
                {k_stem_pool<SIDE_S8, ACT_LEAKY>, k_stem_pool<SIDE_S8, ACT_LINEAR>},
                {k_stem_pool<SIDE_PM1_S8, ACT_LEAKY>, k_stem_pool<SIDE_PM1_S8, ACT_LINEAR>},
                {k_stem_pool<SIDE_BITS, ACT_LEAKY>, k_stem_pool<SIDE_BITS, ACT_LINEAR>},
                {k_stem_pool<SIDE_S8_SAT, ACT_LEAKY>, k_stem_pool<SIDE_S8_SAT, ACT_LINEAR>},
                {k_stem_pool<SIDE_PM1Z_S8, ACT_LEAKY>, k_stem_pool<SIDE_PM1Z_S8, ACT_LINEAR>}};
            const Layer &c2 = layer(2);
            push_input_kernel(OP_CONV_SIMT, 0, k[L[2].side - SIDE_S8][act == ACT_LEAKY ? 0 : 1],
                              (unsigned)(((long)B * c2.h * c2.w + 127) / 128), 128, side_placed(2), stem_weights<16>(l0), act, H, W,
                              side_mult(2));
        } else if (first == FIRST_STEM_TC || first == FIRST_STEM_S2) {
            const bool s2 = first == FIRST_STEM_S2;
            e.stem_plan = s2 ? tc_stem_s2_make_plan(l0, layer(1), e.out_tv[1], e.w_arena.get() + stem_w_off, bias(0),
                                                    e.w_arena.get() + cw[1].w, bias(1), sw.tc.grid)
                             : tc_stem_make_plan(l0, e.out_tv[0], e.w_arena.get() + stem_w_off, bias(0));
            const StemPlan *sp = e.stem_plan.get();
            if (s2) ++e.n_tc;
            push(OP_CONV_TC, s2 ? 1 : 0, [sp](const float *in, cudaStream_t s) { tc_stem_launch(*sp, in, s); });
            if (!sw.no_stem_u8) e.ops[0].launch_u8 = [sp](const unsigned char *in, cudaStream_t s) { tc_stem_launch_u8(*sp, in, s); };
        } else if (first == FIRST_STEM_SIMT) {
            const bool bf16 = L[0].out_dt == DT_BF16;
            const unsigned grid = (unsigned)(((long)B * H * W + 127) / 128);
            if (l0.n == 32)
                push_input_kernel(OP_CONV_SIMT, 0, bf16 ? k_conv_stem<32, __nv_bfloat16> : k_conv_stem<32, float, true>, grid, 128,
                                  e.out_tv[0], stem_weights<32>(l0), act, H, W);
            else
                push_input_kernel(OP_CONV_SIMT, 0, bf16 ? k_conv_stem<16, __nv_bfloat16> : k_conv_stem<16, float, true>, grid, 128,
                                  e.out_tv[0], stem_weights<16>(l0), act, H, W);
        } else {
            push_input_kernel(OP_INPUT, -1, BY_DT(k_input_nchw_to_nhwc, ADT), grid_for((long)e.in0.N * e.in0.H * e.in0.W), 256, e.in0);
        }
    }

    // k_int_input: convolution j's converted input from tin, behind a size x size / stride max-pool (1 / 1 / 0: the conversion
    // alone)
    void push_int_input(int kind, int i, int j, const TV &tin, int size, int stride, int pad) {
        const SideFmt f = L[j].side;   // SIDE_S8, SIDE_PM1_S8, SIDE_BITS, SIDE_S8_SAT or SIDE_PM1Z_S8
        void (*const k[5])(TV, TV, int, int, int, float) = {k_int_input<SIDE_S8>, k_int_input<SIDE_PM1_S8>, k_int_input<SIDE_BITS>,
                                                            k_int_input<SIDE_S8_SAT>, k_int_input<SIDE_PM1Z_S8>};
        const TV q = side_placed(j);
        push_kernel(kind, i, k[f - SIDE_S8], grid_for((long)B * q.H * q.W * int_input_groups(f, tin.C)), 256, 0, tin, q, size, stride, pad,
                    side_mult(j));
    }

    // Convolution i: its input conversion, unless the op in front writes it, then the op of its kernel family
    void emit_conv(int i) {
        const Layer &l = layer(i);
        const LayerPlan &p = L[i];
        const ArithRow &a = kArith[p.arith];
        const TV tin = i == 0 ? e.in0 : e.out_tv[i - 1];   // no base where the input is fused away
        const int tgt = p.fused_into >= 0 ? p.fused_into : i;
        const TV tout = e.out_tv[tgt];                      // no base where the max-pool behind it is fused
        if (p.side == SIDE_PM1_F32)
            push_kernel(OP_BINARIZE, i, k_binarize_pm1, grid_for((long)B * l.h * l.w * l.c), 256, 0, tin, side_placed(i));
        else if (side_int(p.side) && !p.prefilled)
            push_int_input(side_s8(p.side) ? OP_QUANTIZE : OP_BINARIZE, i, i, tin, 1, 1, 0);
        if (side_int(p.side)) counts_buffer(i);   // allocated before the tensor-core plan, which takes its address
        if (p.kern == KERN_TC) {
            push_tc_plan(i);
        } else if (p.kern == KERN_SMALLK) {
            push_conv_smallk(i, tout);
        } else if (a.simt) {
            push_conv_simt(a.simt_op, i, a.simt, side_placed(i), tout);
        } else {
            TV res{}; int rdt = DT_F32; int act2 = ACT_LINEAR;
            if (p.fused_into >= 0) {
                const Layer &s = layer(tgt);
                res = e.out_tv[s.index];
                rdt = L[s.index].out_dt;
                act2 = s.activation;
            }
            // by input, output and residual dtype; all f32 is the reference's summation order, bit-exact
            void (*const k[2][2][2])(SimtP) = {
                {{k_conv_simt<SimtF32<float, float, float, true>>, k_conv_simt<SimtF32<float, float, __nv_bfloat16>>},
                 {k_conv_simt<SimtF32<float, __nv_bfloat16, float>>, k_conv_simt<SimtF32<float, __nv_bfloat16, __nv_bfloat16>>}},
                {{k_conv_simt<SimtF32<__nv_bfloat16, float, float>>, k_conv_simt<SimtF32<__nv_bfloat16, float, __nv_bfloat16>>},
                 {k_conv_simt<SimtF32<__nv_bfloat16, __nv_bfloat16, float>>, k_conv_simt<SimtF32<__nv_bfloat16, __nv_bfloat16, __nv_bfloat16>>}}};
            push_conv_simt(a.simt_op, i, k[in_dt(i)][L[tgt].out_dt][rdt], p.side == SIDE_NONE ? tin : side_placed(i), tout, res, act2);
        }
    }

    // k_conv_simt<V>: convolution i as the CUDA-core implicit GEMM, over the f32 [K][ldw] weights or, for an XNOR or INT8 layer
    // reading sign bits or s8 values, over the 32-bit words of its side input and weights
    void push_conv_simt(int kind, int i, void (*k)(SimtP), const TV &tin, const TV &tout, const TV &res = TV{}, int act2 = ACT_LINEAR) {
        const Layer &l = layer(i);
        const LayerPlan &p = L[i];
        const int taps = l.size * l.size;
        const long M = (long)B * l.out_h * l.out_w;
        SimtP sp{};
        sp.in = tin; sp.out = tout; sp.res = res;
        sp.w = e.w_arena.get() + cw[i].w;
        sp.bias = bias(i);
        if (arith_mean(p.arith)) sp.mean = mean(i);
        if (kArith[p.arith].alpha1_num) sp.alpha1 = alpha1(i);
        sp.n = l.n; sp.size = l.size; sp.stride = l.stride; sp.pad = l.pad;
        sp.act = l.activation; sp.act2 = act2; sp.M = M;
        if (side_int(p.side)) {
            sp.CW = (int)align_up(l.c, 32) / side_per_word(p.side);
            sp.K = taps * sp.CW;
            sp.counts = counts_buffer(i);
            if (p.side == SIDE_BITS) { sp.bits = taps * l.c; sp.padbits = (sp.CW * 32 - l.c) * taps; }
        } else {
            sp.ldw = cw[i].ldw; sp.K = taps * l.c;
        }
        push_kernel(kind, i, k, dim3((unsigned)((M + 63) / 64), (unsigned)((l.n + 63) / 64)), 256, 0, sp);
    }

    // k_conv_xnor_smallk*: XNOR convolution i over CW <= 2 sign words per tap
    void push_conv_smallk(int i, const TV &tout) {
        const Layer &l = layer(i);
        const LayerPlan &p = L[i];
        const long M = (long)B * l.out_h * l.out_w;
        const int CW = side_ld(i);
        const int a = p.arith - AR_XNOR;   // AR_XNOR or AR_XNOR_GPU
        XnorP xp{};
        xp.bits = side_placed(i); xp.out = tout;
        xp.w = reinterpret_cast<const uint32_t *>(e.w_arena.get() + cw[i].w);
        xp.mean = mean(i);
        xp.bias = bias(i);
        xp.n = l.n; xp.K = l.size * l.size * l.c;
        xp.padbits = (CW * 32 - l.c) * l.size * l.size;
        xp.act = l.activation; xp.M = M; xp.counts = counts_buffer(i);
        const size_t smem = (size_t)l.n * 9 * CW * 4;
        if (p.pool != SIDE_NONE) {
            // the 2x2 max-pool behind this layer and the next XNOR layer's sign extraction run in this kernel, which reads only
            // the shape of the output it does not write.  By sign words per tap and the next layer's side format (SIDE_PM1_S8,
            // SIDE_BITS) and the arithmetic.
            void (*const k[2][2][2])(XnorP, TV) = {
                {{k_conv_xnor_smallk_pool<1, SIDE_PM1_S8>, k_conv_xnor_smallk_pool<1, SIDE_BITS>},
                 {k_conv_xnor_smallk_pool<2, SIDE_PM1_S8>, k_conv_xnor_smallk_pool<2, SIDE_BITS>}},
                {{k_conv_xnor_smallk_pool_gpu<1, SIDE_PM1_S8>, k_conv_xnor_smallk_pool_gpu<1, SIDE_BITS>},
                 {k_conv_xnor_smallk_pool_gpu<2, SIDE_PM1_S8>, k_conv_xnor_smallk_pool_gpu<2, SIDE_BITS>}}};
            xp.out = make_tv(nullptr, B, l.out_h, l.out_w, l.n, L[i].ldc, P, DT_F32, 0);
            const Layer &c2 = layer(i + 2);
            push_kernel(OP_CONV_XNOR, i, k[a][CW - 1][p.pool - SIDE_PM1_S8], (unsigned)(((long)B * c2.h * c2.w + 127) / 128), 128, smem, xp,
                        side_placed(i + 2));
            return;
        }
        void (*const k[2][2])(XnorP) = {{k_conv_xnor_smallk<1>, k_conv_xnor_smallk<2>}, {k_conv_xnor_smallk_gpu<1>, k_conv_xnor_smallk_gpu<2>}};
        push_kernel(OP_CONV_XNOR, i, k[a][CW - 1], (unsigned)((M + 127) / 128), 128, smem, xp);
    }

    // max-pool, upsample, shortcut, route, reorg, yolo, region
    void emit_small(int i) {
        const Layer &l = layer(i);
        const LayerPlan &p = L[i];
        const TV tin = i == 0 ? e.in0 : e.out_tv[i - 1];
        const int dt = in_dt(i);
        const TV tout = e.out_tv[i];
        const int g = grid_for((long)B * l.out_h * l.out_w * l.out_c);
        // the 16-byte forms of max-pool and upsample (one thread per 16 bytes of channels): whole 16-byte channel rows of
        // 16-byte aligned pixels
        const int esz = (int)dt_size(dt);
        const bool vec = l.out_c * esz % 16 == 0 && vec16_view(tin, esz) && vec16_view(tout, esz);
        const int gv = grid_for((long)B * l.out_h * l.out_w * ((l.out_c * esz) / 16 + 1));
        switch (l.type) {
        case YB_MAXPOOL: {
            if (p.pool_in_conv) break;    // done in the epilogue of the integer convolution in front of it
            if (p.pool_to_side) {
                push_int_input(OP_MAXPOOL, i, i + 1, tin, l.size, l.stride, l.pad);
                break;
            }
            push_kernel(OP_MAXPOOL, i, vec ? BY_DT(k_maxpool_vec, dt) : BY_DT(k_maxpool, dt), vec ? gv : g, 256, 0, tin, tout, l.size,
                        l.stride, l.pad);
            break;
        }
        case YB_UPSAMPLE: {
            if (vec && l.scale == 1.f)
                push_kernel(OP_UPSAMPLE, i, BY_DT(k_upsample_vec16, dt), gv, 256, 0, tin, tout, l.stride);
            else
                push_kernel(OP_UPSAMPLE, i, BY_DT(k_upsample, dt), g, 256, 0, tin, tout, l.stride, l.scale);
            break;
        }
        case YB_SHORTCUT: {
            if (p.fused_sc) break;
            // shortcut_cpu(batch, w1=l.w, h1=l.h, c1=l.c (from), add, w2=l.out_w, ...): yolov2_forward_network.c:410.  Behind a
            // GPU-rule XNOR layer (sc_bin): the bit GEMM's `shortcut_out = shortcut_in + v` (gpu.cu:1988-1990), without the
            // shortcut's activation; the layer plan admits only leaky and linear layers there, whose output is v.
            const int stride = std::max(l.w / l.out_w, 1), sample = std::max(l.out_w / l.w, 1);
            const int minw = std::min(l.w, l.out_w), minh = std::min(l.h, l.out_h), minc = std::min(l.c, l.out_c);
            push_kernel(OP_SHORTCUT, i, BY_DT(k_shortcut, dt), g, 256, 0, tin, e.out_tv[l.index], tout, stride, sample, minw, minh,
                        minc, p.sc_bin ? (int)ACT_LINEAR : l.activation);
            break;
        }
        case YB_ROUTE: {
            if (is_alias(i)) break;
            int off = 0;
            for (int j : l.input_layers) {
                const Layer &src = layer(j);
                if (L[j].owner != i) {
                    TV slice = tout;
                    slice.base += (size_t)off * dt_size(p.out_dt);
                    slice.C = src.out_c;
                    push_kernel(OP_ROUTE_COPY, i, BY_DT(k_copy_channels, p.out_dt),
                                grid_for((long)B * src.out_h * src.out_w * src.out_c), 256, 0, e.out_tv[j], slice);
                }
                off += src.out_c;
            }
            break;
        }
        case YB_REORG:
            push_kernel(OP_REORG, i, BY_DT(k_reorg, dt), g, 256, 0, tin, tout, l.stride);
            break;
        case YB_YOLO:
            if (p.yolo_fused) break;   // written by the head convolution's epilogue
            push_kernel(OP_YOLO, i, BY_DT(k_yolo, dt), grid_for((long)B * ((l.h * l.w + 31) / 32) * ((l.c + 31) / 32) * 256), 256, 0,
                        tin, e.finals[i].d.get(), l.classes, ADT == DT_BF16 ? 1 : 0);
            break;
        case YB_REGION:
            push_kernel(OP_REGION, i, BY_DT(k_region, dt), grid_for((long)B * l.h * l.w * l.n), 256, 0, tin, e.finals[i].d.get(), l.n,
                        l.classes, l.coords, l.softmax);
            break;
        default:
            break;
        }
    }

    // last layer that is not yolo / region: keep an NCHW f32 copy as "the network output"
    void emit_last_copy() {
        const int last = nl - 1;
        const Layer &l = layer(last);
        if (l.type == YB_YOLO || l.type == YB_REGION || !e.finals[last].d) return;
        const int src = L[last].fused_into >= 0 ? L[last].fused_into : last;
        const TV t = e.out_tv[src];
        if (!t.base) return;
        push_kernel(OP_YOLO, last, BY_DT(k_nhwc_to_nchw_f32, L[src].out_dt), grid_for((long)B * l.outputs), 256, 0, t,
                    e.finals[last].d.get());
    }

    void emit_ops() {
        emit_first();
        for (int i = 0; i < nl; ++i) {
            if (L[i].in_first_op) continue;
            if (is_conv(i)) emit_conv(i);
            else emit_small(i);
        }
        emit_last_copy();
    }
};
}  // namespace

std::shared_ptr<Engine> build_engine(Network *net, const EngineOptions &opt) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        fatal_throw("yolo2_light_b200: no CUDA device -- this library has no CPU fallback");
    CUDA_OK(cudaSetDevice(opt.device));
    cudaDeviceProp prop;
    CUDA_OK(cudaGetDeviceProperties(&prop, opt.device));
    if (prop.major != 9 || prop.minor != 0)
        fatal_throw(std::string("yolo2_light_b200: device '") + prop.name + "' is compute capability " +
                    std::to_string(prop.major) + "." + std::to_string(prop.minor) +
                    "; this build contains sm_90a code only");
    if (net->layers.empty()) fatal_throw("empty network");

    auto e = std::make_shared<Engine>();
    e->opt = opt;
    e->batch = net->batch;
    e->sw = Switches::read();
    e->opt.fuse = opt.fuse && !e->sw.no_fuse;
    e->stream = make_stream();

    Builder b(*net, *e);
    b.plan_layers();
    b.place();
    b.place_finals();
    b.pack_weights();
    e->d_input.ensure((size_t)net->batch * net->c * net->h * net->w);
    b.emit_ops();
    CUDA_OK(cudaStreamSynchronize(e->stream));
    CUDA_OK(cudaGetLastError());
    return e;
}

static void engine_forward_impl(Engine *e, const void *d_input, const unsigned char *d_u8_frames, void *stream);
void engine_forward(Engine *e, const void *d_input, void *stream) { engine_forward_impl(e, d_input, nullptr, stream); }

void engine_upload_input(Engine *e, const float *host_input, void *stream) {
    cudaStream_t s = stream ? (cudaStream_t)stream : (cudaStream_t)e->stream;
    CUDA_OK(cudaSetDevice(e->opt.device));
    CUDA_OK(cudaMemcpyAsync(e->d_input.get(), host_input, e->d_input.count() * sizeof(float), cudaMemcpyHostToDevice, s));
}

// The per-image table: frame sizes; the resize target, its offset and the resize's scales -- the network size at (0, 0), or
// with net->letterbox the letterbox size, centred (embed_image's integer offsets); and the size correct_yolo_boxes
// (additionally.c:4287-4296) embeds each image at -- the network size, or with `letter` the letterbox size.  Entries
// nimg .. batch-1 are zero.
static void fill_geo(Engine *e, Engine::FrameStage &st, const Network *net, const int *w, const int *h, int nimg, int letter) {
    const int B = e->batch;
    st.h_geo.ensure(B);
    st.d_geo.ensure(B);
    for (int b = 0; b < B; ++b) {
        ImageGeo &g = st.h_geo.get()[b];
        g = ImageGeo{};
        if (b >= nimg) continue;
        g.w = w[b]; g.h = h[b];
        int lw, lh;
        letterbox_size(net->w, net->h, g.w, g.h, &lw, &lh);
        g.new_w = letter ? lw : net->w; g.new_h = letter ? lh : net->h;
        g.nw = net->letterbox ? lw : net->w; g.nh = net->letterbox ? lh : net->h;
        g.dx = (net->w - g.nw) / 2; g.dy = (net->h - g.nh) / 2;
        g.w_scale = (float)(g.w - 1) / (float)(g.nw - 1);   // resize_image, additionally.c:3027-3028
        g.h_scale = (float)(g.h - 1) / (float)(g.nh - 1);
    }
}

// frames described by st.d_geo, of format fmt -> the network's planar f32 input; images nimg .. batch-1 are zero
static void launch_resize(Engine *e, const Engine::FrameStage &st, const Network *net, int nimg, int fmt, float *dst,
                          cudaStream_t s) {
    if (!e->d_unit) {   // load_image_stb's conversion, additionally.c:3093-3103
        float unit[256];
        for (int v = 0; v < 256; ++v) unit[v] = (float)((double)(float)v / 255.);
        DevBuf<float> d_unit(256);
        CUDA_OK(cudaMemcpy(d_unit.get(), unit, sizeof(unit), cudaMemcpyHostToDevice));
        e->d_unit = std::move(d_unit);
    }
    const dim3 grid((unsigned)((net->h + RS_ROWS - 1) / RS_ROWS), (unsigned)nimg);
    auto *k = fmt == YB_FRAME_BGR ? k_resize_frames<YB_FRAME_BGR> : fmt == YB_FRAME_RGB_PLANAR ? k_resize_frames<YB_FRAME_RGB_PLANAR>
            : fmt == YB_FRAME_NV12 ? k_resize_frames<YB_FRAME_NV12> : k_resize_frames<YB_FRAME_RGB>;
    k<<<grid, RS_THREADS, 0, s>>>(st.d_geo.get(), e->d_unit.get(), net->c, dst, net->w, net->h);
    const size_t per = (size_t)net->c * net->h * net->w;
    if (nimg < e->batch) CUDA_OK(cudaMemsetAsync(dst + nimg * per, 0, (e->batch - nimg) * per * sizeof(float), s));
}

// Batch b, on the engine stream `s`: fills st's per-image table (fill_geo, and where each frame lies) and uploads it, then
// resizes the frames into dst -- or, with dst == nullptr (host frames of the network size), leaves them in st.buf for the
// 8-bit stem, zero frames after the nimg-th.
// Host frames are first copied into st.buf, packed back to back.  Frames that lie back to back in host memory go in one copy
// (a stacked batch is one copy); each copy overlaps other work only from pinned memory.
// Device frames are read where they lie: `s` waits for the work enqueued on the caller's stream `user` before the call (the
// frames' producer), the resize reads the frames, and `user` waits for that resize, so that the caller's later writes into
// the frames come after it.  The engine's events are recorded and waited on at once, so each call may reuse them.  Host
// frames have no caller stream: nothing is recorded on `user` or made to wait for it.
static void stage_frames(Engine *e, Engine::FrameStage &st, const Network *net, const FrameBatch &b, int letter, float *dst,
                         cudaStream_t s, cudaStream_t user) {
    const int B = e->batch;
    const size_t frame = (size_t)net->w * net->h * net->c;
    std::vector<int> w(b.nimg), h(b.nimg);
    for (int i = 0; i < b.nimg; ++i) { w[i] = b.frames[i].w; h[i] = b.frames[i].h; }
    fill_geo(e, st, net, w.data(), h.data(), b.nimg, letter);
    ImageGeo *geo = st.h_geo.get();
    for (int i = 0; i < b.nimg; ++i) {
        const yb_device_frame &f = b.frames[i];
        geo[i].src = f.data; geo[i].chroma = f.chroma; geo[i].pitch = f.pitch; geo[i].plane = f.plane_stride;
    }
    if (b.host) {
        std::vector<size_t> off(b.nimg + 1, 0);   // frame i's bytes at off[i] .. off[i + 1] of st.buf
        for (int i = 0; i < b.nimg; ++i) off[i + 1] = off[i] + (size_t)b.frames[i].pitch * b.frames[i].h;
        st.buf.ensure(std::max(off[b.nimg], dst ? 0 : B * frame));   // the 8-bit stem reads whole batches
        for (int i = 0; i < b.nimg; ++i) geo[i].src = st.buf.get() + off[i];
        for (int i = 0; i < b.nimg;) {
            int j = i + 1;
            while (j < b.nimg && b.frames[j].data == b.frames[i].data + (off[j] - off[i])) ++j;
            CUDA_OK(cudaMemcpyAsync(st.buf.get() + off[i], b.frames[i].data, off[j] - off[i], cudaMemcpyHostToDevice, s));
            i = j;
        }
    }
    CUDA_OK(cudaMemcpyAsync(st.d_geo.get(), geo, (size_t)B * sizeof(ImageGeo), cudaMemcpyHostToDevice, s));
    if (!b.host) {
        if (!e->ev_frames_ready) e->ev_frames_ready = make_event();
        if (!e->ev_frames_read) e->ev_frames_read = make_event();
        CUDA_OK(cudaEventRecord(e->ev_frames_ready, user));
        CUDA_OK(cudaStreamWaitEvent(s, e->ev_frames_ready, 0));
    }
    if (dst) launch_resize(e, st, net, b.nimg, b.fmt, dst, s);
    else if (b.nimg < B) CUDA_OK(cudaMemsetAsync(st.buf.get() + b.nimg * frame, 0, (B - b.nimg) * frame, s));
    if (!b.host) {
        CUDA_OK(cudaEventRecord(e->ev_frames_read, s));
        CUDA_OK(cudaStreamWaitEvent(user, e->ev_frames_read, 0));
    }
}

void engine_upload_frames(Engine *e, Network *net, const FrameBatch &b, void *stream) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    stage_frames(e, e->u8, net, b, 0, e->d_input.get(), e->stream, (cudaStream_t)stream);
    CUDA_OK(cudaGetLastError());
}

// Throws unless every frame's memory (data, and chroma for NV12) is device or managed memory of `device`.
void check_frame_memory(int device, const char *fn, const FrameBatch &fb) {
    for (int b = 0; b < fb.nimg; ++b) {
        for (int p = 0; p < (fb.fmt == YB_FRAME_NV12 ? 2 : 1); ++p) {
            cudaPointerAttributes a{};
            const cudaError_t r = cudaPointerGetAttributes(&a, p ? fb.frames[b].chroma : fb.frames[b].data);
            if (r != cudaSuccess) cudaGetLastError();
            const char *kind = r != cudaSuccess ? "unknown" : a.type == cudaMemoryTypeHost ? "pinned host memory"
                             : a.type == cudaMemoryTypeDevice ? "device memory" : a.type == cudaMemoryTypeManaged ? "managed memory"
                             : "host memory";
            if (r != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != device)
                fatal_throw(std::string(fn) + ": frame " + std::to_string(b) + (p ? " chroma" : "") + " is " + kind +
                            (r == cudaSuccess && a.type != cudaMemoryTypeHost && a.type != cudaMemoryTypeUnregistered
                                 ? " of device " + std::to_string(a.device) : std::string()) +
                            ", not device memory of device " + std::to_string(device));
        }
    }
}

void *engine_stream(Engine *e) { return e->stream; }

static void engine_forward_impl(Engine *e, const void *d_input, const unsigned char *d_u8_frames, void *stream) {
    cudaStream_t s = stream ? (cudaStream_t)stream : (cudaStream_t)e->stream;
    CUDA_OK(cudaSetDevice(e->opt.device));   // thread identity may change per call (SURVEY 8b, threading)
    const float *din = d_input ? reinterpret_cast<const float *>(d_input) : e->d_input.get();
    if (d_u8_frames) e->ops[0].launch_u8(d_u8_frames, s);   // stem straight from the 8-bit frames
    else e->ops[0].launch(din, s);
    if (!e->graph_exec && !e->graph_failed && e->sw.no_graph) e->graph_failed = true;   // profiling aid
    if (!e->graph_exec && !e->graph_failed) {
        // capture everything after ops[0] once
        cudaGraph_t graph = nullptr;
        cudaError_t st = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
        if (st == cudaSuccess) {
            for (size_t k = 1; k < e->ops.size(); ++k) e->ops[k].launch(din, s);
            st = cudaStreamEndCapture(s, &graph);
        }
        cudaGraphExec_t exec = nullptr;
        if (st == cudaSuccess && graph) {
            st = cudaGraphInstantiate(&exec, graph, 0);
            cudaGraphDestroy(graph);
        }
        e->graph_exec = GraphExec(st == cudaSuccess ? exec : nullptr);
        if (!e->graph_exec) { e->graph_failed = true; cudaGetLastError(); }
    }
    if (e->graph_exec) {
        CUDA_OK(cudaGraphLaunch(e->graph_exec, s));
    } else {
        for (size_t k = 1; k < e->ops.size(); ++k) e->ops[k].launch(din, s);
    }
    CUDA_OK(cudaGetLastError());
}

void engine_download_outputs(Engine *e, Network *net, void *stream) {
    cudaStream_t s = stream ? (cudaStream_t)stream : (cudaStream_t)e->stream;
    CUDA_OK(cudaSetDevice(e->opt.device));
    for (size_t i = 0; i < e->finals.size(); ++i) {
        const Engine::Final &f = e->finals[i];
        if (!f.d) continue;
        CUDA_OK(cudaMemcpyAsync(f.h.get(), f.d.get(), f.d.count() * sizeof(float), cudaMemcpyDeviceToHost, s));
        net->layers[i].output = f.h.get();
        net->layers[i].output_count = f.d.count();
    }
    CUDA_OK(cudaStreamSynchronize(s));
}

// ---- the pipeline of the submit / collect calls: three slots, one batch in flight in each ------------------------------
// Takes the next slot for a submit and returns its ticket.  The slots are published only once all three are built; a slot
// whose ticket is still out is refused; the copy-in stream waits until the forward that last read the slot's input is done.
static int acquire_slot(Engine *e) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    if (e->slots.empty()) {
        e->s_in = make_stream(); e->s_out = make_stream(); e->s_det = make_stream();
        std::vector<Engine::Slot> slots(3);
        for (Engine::Slot &sl : slots) {
            sl.d_in.ensure(e->d_input.count());
            sl.ev_in = make_event(); sl.ev_comp = make_event(); sl.ev_done = make_event(); sl.ev_det = make_event();
        }
        e->slots = std::move(slots);
    }
    const int k = e->next_slot;
    Engine::Slot &sl = e->slots[k];
    if (sl.busy) fatal_throw("submit: pipeline full (3 batches in flight) -- collect the oldest ticket first");
    e->next_slot = (k + 1) % (int)e->slots.size();
    sl.collect_seq = 0;
    CUDA_OK(cudaStreamWaitEvent(e->s_in, sl.ev_comp, 0));
    return k;
}

// Runs the forward on the compute stream once the input staged on the copy-in stream is there: from the network-size 8-bit
// frames u8 when given, else from the slot's input.  Then the compute stream waits until the slot's previous outputs have
// been read out (D2H of the raw tensors, or NMS and counts copy), so that what it enqueues next may overwrite them.
static void forward_slot(Engine *e, Engine::Slot &sl, const unsigned char *u8) {
    CUDA_OK(cudaEventRecord(sl.ev_in, e->s_in));
    CUDA_OK(cudaStreamWaitEvent(e->stream, sl.ev_in, 0));
    engine_forward_impl(e, sl.d_in.get(), u8, e->stream);
    CUDA_OK(cudaStreamWaitEvent(e->stream, sl.ev_done, 0));
    CUDA_OK(cudaStreamWaitEvent(e->stream, sl.ev_det, 0));
}

// The slot of a ticket of `mode` once its results have reached the host, marked free; any other ticket throws
// "<fn>: bad ticket".
static Engine::Slot &release_slot(Engine *e, int ticket, int mode, const char *fn) {
    if (ticket < 0 || ticket >= (int)e->slots.size() || !e->slots[ticket].busy || e->slots[ticket].mode != mode)
        fatal_throw(std::string(fn) + ": bad ticket");
    CUDA_OK(cudaSetDevice(e->opt.device));
    Engine::Slot &sl = e->slots[ticket];
    CUDA_OK(cudaEventSynchronize(mode == 0 ? sl.ev_done : sl.ev_det));
    sl.busy = false;
    return sl;
}

// Enqueue one batch: H2D on the copy-in stream, forward on the compute stream, D2H on the copy-out stream.
// Returns the ticket to pass to engine_collect.  Up to 3 batches may be in flight.
int engine_submit(Engine *e, const float *host_input) {
    const int k = acquire_slot(e);
    Engine::Slot &sl = e->slots[k];
    if (sl.out.empty()) {
        std::vector<Engine::Final> out(e->finals.size());
        for (size_t i = 0; i < out.size(); ++i) {
            out[i].d.ensure(e->finals[i].d.count());
            out[i].h.ensure(e->finals[i].d.count());
        }
        sl.out = std::move(out);
    }
    CUDA_OK(cudaMemcpyAsync(sl.d_in.get(), host_input, sl.d_in.count() * sizeof(float), cudaMemcpyHostToDevice, e->s_in));
    forward_slot(e, sl, nullptr);
    for (size_t i = 0; i < e->finals.size(); ++i)
        if (e->finals[i].d)
            CUDA_OK(cudaMemcpyAsync(sl.out[i].d.get(), e->finals[i].d.get(), e->finals[i].d.count() * sizeof(float),
                                    cudaMemcpyDeviceToDevice, e->stream));
    CUDA_OK(cudaEventRecord(sl.ev_comp, e->stream));
    CUDA_OK(cudaStreamWaitEvent(e->s_out, sl.ev_comp, 0));
    for (const Engine::Final &o : sl.out)
        if (o.d) CUDA_OK(cudaMemcpyAsync(o.h.get(), o.d.get(), o.d.count() * sizeof(float), cudaMemcpyDeviceToHost, e->s_out));
    CUDA_OK(cudaEventRecord(sl.ev_done, e->s_out));
    sl.busy = true; sl.mode = 0;
    return k;
}

// ptrs[i] = pinned host copy of layer i's output for this ticket (nullptr where the layer has none); valid until the slot
// is reused.  The form the multi-GPU batch call uses: several engines feed ONE host model.
void engine_collect_ptrs(Engine *e, int ticket, std::vector<const float *> &ptrs, std::vector<size_t> &counts) {
    const Engine::Slot &sl = release_slot(e, ticket, 0, "collect");
    ptrs.clear(); counts.clear();
    for (const Engine::Final &o : sl.out) { ptrs.push_back(o.h.get()); counts.push_back(o.h.count()); }
}

void engine_collect(Engine *e, Network *net, int ticket) {
    std::vector<const float *> ptrs; std::vector<size_t> counts;
    engine_collect_ptrs(e, ticket, ptrs, counts);
    for (size_t i = 0; i < ptrs.size(); ++i) {
        if (!ptrs[i]) continue;
        net->layers[i].output = const_cast<float *>(ptrs[i]);
        net->layers[i].output_count = counts[i];
    }
}

// ---- weight replication across the GPUs of one process (SURVEY 8e: ONE broadcast of the prepared arena at init) ---------
// NCCL is bound at run time (dlopen): the library has no link-time dependency on it, and a host without NCCL -- or a device
// list with repeats, which NCCL refuses -- falls back to peer copies out of replica 0.
const char *engine_broadcast_arena(const std::vector<Engine *> &reps) {
    if (reps.size() < 2) return "single";
    const size_t bytes = reps[0]->w_arena.count();
    for (Engine *r : reps) if (r->w_arena.count() != bytes) fatal_throw("broadcast: replicas disagree on the arena size");
    bool distinct = true;
    for (size_t a = 0; a < reps.size(); ++a)
        for (size_t b = a + 1; b < reps.size(); ++b) distinct &= reps[a]->opt.device != reps[b]->opt.device;
    typedef int (*InitAllFn)(void **, int, const int *);
    typedef int (*BcastFn)(const void *, void *, size_t, int, int, void *, cudaStream_t);
    typedef int (*VoidFn)(void);
    typedef int (*DestroyFn)(void *);
    void *lib = (distinct && !reps[0]->sw.no_nccl) ? dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL) : nullptr;
    if (lib) {
        InitAllFn init_all = (InitAllFn)dlsym(lib, "ncclCommInitAll");
        BcastFn bcast = (BcastFn)dlsym(lib, "ncclBroadcast");
        VoidFn gstart = (VoidFn)dlsym(lib, "ncclGroupStart"), gend = (VoidFn)dlsym(lib, "ncclGroupEnd");
        DestroyFn destroy = (DestroyFn)dlsym(lib, "ncclCommDestroy");
        if (init_all && bcast && gstart && gend && destroy) {
            std::vector<void *> comms(reps.size(), nullptr);
            std::vector<int> devs;
            for (Engine *r : reps) devs.push_back(r->opt.device);
            if (init_all(comms.data(), (int)reps.size(), devs.data()) == 0) {
                int rc = gstart();
                for (size_t k = 0; k < reps.size() && rc == 0; ++k) {
                    CUDA_OK(cudaSetDevice(reps[k]->opt.device));
                    rc = bcast(reps[k]->w_arena.get(), reps[k]->w_arena.get(), bytes, /*ncclChar*/ 0, /*root*/ 0, comms[k], reps[k]->stream);
                }
                rc |= gend();
                for (Engine *r : reps) { CUDA_OK(cudaSetDevice(r->opt.device)); CUDA_OK(cudaStreamSynchronize(r->stream)); }
                for (void *c : comms) if (c) destroy(c);
                if (rc == 0) return "nccl";
            }
        }
    }
    for (size_t k = 1; k < reps.size(); ++k) {
        CUDA_OK(cudaSetDevice(reps[0]->opt.device));
        CUDA_OK(cudaMemcpyPeer(reps[k]->w_arena.get(), reps[k]->opt.device, reps[0]->w_arena.get(), reps[0]->opt.device, bytes));
    }
    CUDA_OK(cudaDeviceSynchronize());
    return "peer-copy";
}
int engine_device_count() { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }

void engine_fetch_layer(Engine *e, Network *net, int layer, float *dst) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    const Layer &l = net->layers[layer];
    const size_t count = (size_t)l.outputs * e->batch;
    if (e->finals[layer].d && (l.type == YB_YOLO || l.type == YB_REGION)) {
        CUDA_OK(cudaMemcpy(dst, e->finals[layer].d.get(), count * sizeof(float), cudaMemcpyDeviceToHost));
        return;
    }
    const TV t = e->out_tv[layer];
    if (!t.base) fatal_throw("fetch_layer: layer " + std::to_string(layer) + " has no materialised output "
                             "(fused or aliased away; build the engine with fusion off)");
    DevBuf<float> tmp(count);
    auto *k = BY_DT(k_nhwc_to_nchw_f32, e->out_dt[layer]);
    k<<<grid_for((long)count), 256, 0, e->stream>>>(t, tmp.get());
    CUDA_OK(cudaMemcpyAsync(dst, tmp.get(), count * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    CUDA_OK(cudaStreamSynchronize(e->stream));
}

void engine_fetch_input(Engine *e, float *dst) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    CUDA_OK(cudaStreamSynchronize(e->stream));
    CUDA_OK(cudaMemcpy(dst, e->d_input.get(), e->d_input.count() * sizeof(float), cudaMemcpyDeviceToHost));
}

int engine_fetch_counts(Engine *e, int layer, int32_t *dst, size_t count) {
    if (layer < 0 || layer >= (int)e->counts.size() || !e->counts[layer]) return -1;
    const DevBuf<int32_t> &c = e->counts[layer];
    if (count < c.count()) return -2;
    CUDA_OK(cudaSetDevice(e->opt.device));
    CUDA_OK(cudaMemcpy(dst, c.get(), c.count() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return (int)c.count();
}

void engine_weight_arena(Engine *e, void **ptr, size_t *bytes) { *ptr = e->w_arena.get(); *bytes = e->w_arena.count(); }
// INT8 input calibration (SURVEY 8f row 3): |x| histogram of the INPUT of layer `layer` (image `img` of the batch) after a
// forward, binned like the reference's entropy_calibration.  hist: host uint32[max_bin].
void engine_input_histogram(Engine *e, Network *net, int layer, int img, float bin_width, int max_bin, uint32_t *hist) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    if (max_bin < 129 || max_bin > 4096) fatal_throw("calibrate: max_bin must be in 129..4096");
    if (img < 0 || img >= e->batch) fatal_throw("calibrate: image index out of range");
    DevBuf<unsigned> d_hist(max_bin);
    CUDA_OK(cudaMemsetAsync(d_hist.get(), 0, (size_t)max_bin * sizeof(unsigned), e->stream));
    if (layer == 0) {
        const long n = (long)net->c * net->h * net->w;
        k_abs_hist_flat<<<grid_for(n), 256, 0, e->stream>>>(e->d_input.get() + (size_t)img * n, n, bin_width, max_bin, d_hist.get());
    } else {
        const TV t = e->out_tv[layer - 1];
        if (!t.base) fatal_throw("calibrate: the input of layer " + std::to_string(layer) +
                                 " is not materialised (fused away; set option fuse=0)");
        auto *k = BY_DT(k_abs_hist, e->out_dt[layer - 1]);
        k<<<grid_for((long)t.C * t.H * t.W), 256, 0, e->stream>>>(t, img, bin_width, max_bin, d_hist.get());
    }
    CUDA_OK(cudaMemcpyAsync(hist, d_hist.get(), (size_t)max_bin * sizeof(unsigned), cudaMemcpyDeviceToHost, e->stream));
    CUDA_OK(cudaStreamSynchronize(e->stream));
}

// ---- batched decode + NMS on the device (yb_detect.cuh) ---------------------------------------------------------
// geometry: P.geo, set by the caller
static DetParams det_params(Network *net, const std::vector<Engine::Final> &finals, float thresh, float nms, int relative,
                            int max_rows) {
    DetParams P{};
    int total = 0;
    for (size_t i = 0; i < net->layers.size(); ++i) {
        const Layer &l = net->layers[i];
        if (l.type != YB_YOLO && l.type != YB_REGION) continue;
        if (!finals[i].d) fatal_throw("detect: detection layer has no device output");
        if (P.nl == DET_MAX_LAYERS) fatal_throw("detect: too many detection layers");
        if (l.n > DET_MAX_ANCHORS) fatal_throw("detect: too many anchors per layer");
        if (P.nl && l.classes != P.classes) fatal_throw("detect: detection layers disagree on the class count");
        if ((l.type == YB_YOLO && (int)l.mask.size() < l.n) || (int)l.anchors.size() < 2 * l.n)
            fatal_throw("detect: detection layer without mask / anchors");
        DetLayer &d = P.L[P.nl++];
        d.p = finals[i].d.get(); d.type = l.type; d.w = l.w; d.h = l.h; d.n = l.n; d.classes = l.classes; d.outputs = l.outputs;
        d.base = total; d.nbox = l.w * l.h * l.n; total += d.nbox;
        for (int a = 0; a < l.n; ++a) {
            const int k = (l.type == YB_YOLO) ? l.mask[a] : a;
            d.aw[a] = l.anchors[2 * k]; d.ah[a] = l.anchors[2 * k + 1];
        }
        P.classes = l.classes;
    }
    if (!P.nl) fatal_throw("detect: the network has no yolo / region layer");
    P.total = total; P.netw = net->w; P.neth = net->h; P.relative = relative;
    P.thresh = thresh; P.nms = nms; P.max_rows = max_rows; P.nblk = (total + 255) / 256;
    return P;
}

// pitch == cap == max_rows: the NMS sees exactly the rows the caller asked for
static void det_ws_ensure(Engine::DetWs &ws, int B, const DetParams &P) {
    const int stride = 5 + P.classes, words = (P.max_rows + 31) / 32;
    ws.rows.ensure((size_t)B * P.max_rows * stride);
    ws.mask.ensure((size_t)B * P.max_rows * words);
    ws.blkcnt.ensure((size_t)B * P.nblk);
    ws.counts.ensure(B);
    ws.cap = P.max_rows; ws.stride = stride;
}

// decode of the first nimg images; counts[b] = 0 for the others
static void det_launch_count_emit(const DetParams &P, Engine::DetWs &ws, int B, int nimg, cudaStream_t s) {
    k_det_count<<<dim3((unsigned)P.nblk, (unsigned)nimg), 256, 0, s>>>(P, ws.blkcnt.get());
    k_det_emit<<<dim3((unsigned)P.nblk, (unsigned)nimg), 256, 0, s>>>(P, ws.blkcnt.get(), ws.rows.get(), ws.counts.get());
    if (nimg < B) CUDA_OK(cudaMemsetAsync(ws.counts.get() + nimg, 0, (size_t)(B - nimg) * sizeof(int), s));
}
// nmax: upper bound of the candidates of any image (the kernels read the true counts on the device and idle beyond them)
static void det_launch_nms(const DetParams &P, Engine::DetWs &ws, int nimg, int nmax, cudaStream_t s) {
    if (!(P.nms > 0.f) || nmax <= 0) return;
    const int capw = (ws.cap + 31) / 32;
    k_det_iou<<<dim3((unsigned)((capw + 127) / 128), (unsigned)std::min(nmax, 256), (unsigned)nimg), 128, 0, s>>>(
        P, ws.rows.get(), ws.counts.get(), ws.mask.get());
    int P2 = 1; while (P2 < nmax) P2 <<= 1;
    const size_t smem = (size_t)P2 * 8 + (size_t)capw * 4;
    if (smem > 48 * 1024)
        CUDA_OK(cudaFuncSetAttribute(k_det_nms, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_det_nms<<<dim3((unsigned)P.classes, (unsigned)nimg), 256, smem, s>>>(P, ws.rows.get(), ws.counts.get(), ws.mask.get(), P2);
}

// Synchronous form.  Image b's boxes are corrected for a w[b] x h[b] frame.  rows: [batch][max_rows][5 + classes];
// counts[b] = candidates of image b before the max_rows cap, 0 for b >= nimg.  Returns 5 + classes.
int engine_detect(Engine *e, Network *net, const int *w, const int *h, int nimg, float thresh, float nms, int relative,
                  int letter, float *rows, int max_rows, int *counts) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    DetParams P = det_params(net, e->finals, thresh, nms, relative, max_rows);
    const int B = e->batch, stride = 5 + P.classes;
    det_ws_ensure(e->det, B, P);
    cudaStream_t s = e->stream;
    fill_geo(e, e->u8, net, w, h, nimg, letter);
    CUDA_OK(cudaMemcpyAsync(e->u8.d_geo.get(), e->u8.h_geo.get(), (size_t)B * sizeof(ImageGeo), cudaMemcpyHostToDevice, s));
    P.geo = e->u8.d_geo.get();
    det_launch_count_emit(P, e->det, B, nimg, s);
    std::vector<int> hc(B);
    CUDA_OK(cudaMemcpyAsync(hc.data(), e->det.counts.get(), B * sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    int nmax = 0;
    for (int b = 0; b < B; ++b) { counts[b] = hc[b]; nmax = std::max(nmax, std::min(hc[b], max_rows)); }
    det_launch_nms(P, e->det, nimg, nmax, s);
    for (int b = 0; b < nimg; ++b) {
        const int n = std::min(hc[b], max_rows);
        if (n > 0)
            CUDA_OK(cudaMemcpyAsync(rows + (size_t)b * max_rows * stride, e->det.rows.get() + (size_t)b * max_rows * stride,
                                    (size_t)n * stride * sizeof(float), cudaMemcpyDeviceToHost, s));
    }
    CUDA_OK(cudaStreamSynchronize(s));
    CUDA_OK(cudaGetLastError());
    return stride;
}

// Selection and drawing of the batch in slot sl (device frames b, geometry table P.geo) on the side stream s, behind its NMS;
// then `user` waits for the draw.  The counts of selected detections go to the host here, the list itself at the collect.
static void det_launch_draw(Engine *e, const DetParams &P, Engine::Slot &sl, const FrameBatch &b, cudaStream_t s,
                            cudaStream_t user) {
    const int B = e->batch;
    sl.d_sel.ensure((size_t)B * P.max_rows); sl.d_draw.ensure((size_t)B * P.max_rows); sl.d_nsel.ensure(B);
    sl.h_sel.ensure((size_t)B * P.max_rows); sl.h_nsel.ensure(B);
    int P2 = 1; while (P2 < P.max_rows) P2 <<= 1;
    const size_t smem = (size_t)P2 * 12;   // set every time: with the kernel's static shared memory, 4096 rows pass 48 KB
    CUDA_OK(cudaFuncSetAttribute(k_det_select, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_det_select<<<(unsigned)b.nimg, 256, smem, s>>>(P, sl.det.rows.get(), sl.det.counts.get(), sl.d_sel.get(), sl.d_nsel.get(),
                                                      sl.d_draw.get(), P2);
    auto *k = b.fmt == YB_FRAME_BGR ? k_det_draw<YB_FRAME_BGR> : b.fmt == YB_FRAME_RGB_PLANAR ? k_det_draw<YB_FRAME_RGB_PLANAR>
            : b.fmt == YB_FRAME_NV12 ? k_det_draw<YB_FRAME_NV12> : k_det_draw<YB_FRAME_RGB>;
    k<<<dim3((unsigned)b.nimg, DET_DRAW_BANDS), 256, 0, s>>>(P.geo, sl.d_draw.get(), sl.d_nsel.get(), P.max_rows);
    if (b.nimg < B) CUDA_OK(cudaMemsetAsync(sl.d_nsel.get() + b.nimg, 0, (size_t)(B - b.nimg) * sizeof(int), s));
    CUDA_OK(cudaMemcpyAsync(sl.h_nsel.get(), sl.d_nsel.get(), (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (!e->ev_frames_drawn) e->ev_frames_drawn = make_event();
    CUDA_OK(cudaEventRecord(e->ev_frames_drawn, s));
    CUDA_OK(cudaStreamWaitEvent(user, e->ev_frames_drawn, 0));
}

// ---- pipelined detection path (SURVEY 8f rows 1 + 2 in the serving loop) -----------------------------------------
// One call enqueues, for one batch of nimg 8-bit frames of any sizes: H2D of the frames and of their geometry table + the
// reference's resize on the copy-in stream, the forward on the compute stream, decode + NMS on a side stream (under the
// forward of the NEXT batch), and returns a ticket.  engine_collect_detections waits for that batch and copies back exactly
// the candidate rows.  Host traffic per batch: the u8 frames in (a quarter of the float images), counts + rows out (a few
// hundred KB instead of the 124 MB of yolo tensors).  Device frames are resized the same way, read in order with the caller's
// `stream`.
// With `draw`, the side stream then selects each image's detections (k_det_select) and draws them into its device frame
// (k_det_draw), and the caller's `stream` waits for that draw.
int engine_submit_frames(Engine *e, Network *net, const FrameBatch &b, float thresh, float nms, int relative, int letter,
                         int max_rows, void *stream, bool draw) {
    DetParams P = det_params(net, e->finals, thresh, nms, relative, max_rows);
    const int B = e->batch, stride = 5 + P.classes;
    const int k = acquire_slot(e);
    Engine::Slot &sl = e->slots[k];
    det_ws_ensure(sl.det, B, P);
    sl.h_rows.ensure((size_t)B * max_rows * stride);
    sl.h_counts.ensure(B);
    // host frames that all have the network size need no resize when the stem reads 8-bit frames
    bool u8_stem = b.host && e->ops[0].launch_u8 && net->c == 3;
    for (int i = 0; i < b.nimg; ++i) u8_stem &= b.frames[i].w == net->w && b.frames[i].h == net->h;
    // The slot's frames and geometry table go on s_in.  The decode below reads the table on the compute stream behind ev_in,
    // and the next submit to this slot rewrites it only after waiting for ev_comp (acquire_slot) -- and only once this ticket
    // has been collected, which waits for ev_det, so the pinned host table is no longer being copied either.
    stage_frames(e, sl.u8, net, b, letter, u8_stem ? nullptr : sl.d_in.get(), e->s_in, (cudaStream_t)stream);
    forward_slot(e, sl, u8_stem ? sl.u8.buf.get() : nullptr);
    // Candidate selection + box decode (k_det_count / k_det_emit: they read the objectness planes and, for the few candidates,
    // their class scores) run right behind the forward on the compute stream, straight on the engine's yolo tensors -- the next
    // forward overwrites those, so this is the only part that must not slip.  What follows (IoU matrix + per-class NMS) works on
    // the slot's own candidate rows and goes to the side stream, where it overlaps the next batch's forward.  (Copying the
    // 124 MB of yolo tensors into the slot first, as the raw-tensor path does, cost more than the decode itself.)
    P.geo = sl.u8.d_geo.get();
    det_launch_count_emit(P, sl.det, B, b.nimg, e->stream);
    CUDA_OK(cudaEventRecord(sl.ev_comp, e->stream));
    CUDA_OK(cudaStreamWaitEvent(e->s_det, sl.ev_comp, 0));
    CUDA_OK(cudaMemcpyAsync(sl.h_counts.get(), sl.det.counts.get(), (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, e->s_det));
    det_launch_nms(P, sl.det, b.nimg, max_rows, e->s_det);  // no host round trip: grids sized for the cap, kernels read the counts
    if (draw) det_launch_draw(e, P, sl, b, e->s_det, (cudaStream_t)stream);
    CUDA_OK(cudaEventRecord(sl.ev_det, e->s_det));
    CUDA_OK(cudaGetLastError());
    sl.busy = true; sl.mode = 1; sl.nimg = b.nimg; sl.draw = draw;
    return k;
}

// rows: pinned [batch][max_rows][5 + classes] (valid until the slot is reused), counts[batch] (0 beyond the ticket's images);
// returns 5 + classes.  A drawing ticket's selected list comes back too (engine_selected_detections).
int engine_collect_detections(Engine *e, int ticket, const float **rows, const int **counts, size_t *d2h_bytes) {
    Engine::Slot &sl = release_slot(e, ticket, 1, "collect_detections");
    const int B = e->batch, cap = sl.det.cap, stride = sl.det.stride;
    size_t moved = (size_t)B * sizeof(int);
    for (int b = 0; b < sl.nimg; ++b) {
        const int n = std::min(sl.h_counts.get()[b], cap);
        if (n > 0) {
            CUDA_OK(cudaMemcpyAsync(sl.h_rows.get() + (size_t)b * cap * stride, sl.det.rows.get() + (size_t)b * cap * stride,
                                    (size_t)n * stride * sizeof(float), cudaMemcpyDeviceToHost, e->s_out));
            moved += (size_t)n * stride * sizeof(float);
        }
    }
    if (sl.draw) {
        moved += (size_t)B * sizeof(int);
        for (int b = 0; b < sl.nimg; ++b) {
            const int n = sl.h_nsel.get()[b];
            if (n > 0) {
                CUDA_OK(cudaMemcpyAsync(sl.h_sel.get() + (size_t)b * cap, sl.d_sel.get() + (size_t)b * cap,
                                        (size_t)n * sizeof(yb_detection), cudaMemcpyDeviceToHost, e->s_out));
                moved += (size_t)n * sizeof(yb_detection);
            }
        }
    }
    CUDA_OK(cudaStreamSynchronize(e->s_out));
    if (sl.draw) {
        static std::atomic<unsigned long long> seq{0};
        sl.collect_seq = ++seq;
    }
    if (rows) *rows = sl.h_rows.get();
    if (counts) *counts = sl.h_counts.get();
    if (d2h_bytes) *d2h_bytes = moved;
    return stride;
}

// The selected list of a collected drawing ticket: 0 and *dets / *counts, with *seq the collect's place among all collects of
// drawing tickets (so that of several engines the most recent one can be chosen); -1 for any other ticket.
int engine_selected_detections(Engine *e, int ticket, const yb_detection **dets, const int **counts, unsigned long long *seq) {
    if (ticket < 0 || ticket >= (int)e->slots.size()) return -1;
    const Engine::Slot &sl = e->slots[ticket];
    if (sl.busy || sl.mode != 1 || !sl.draw || !sl.collect_seq) return -1;
    if (dets) *dets = sl.h_sel.get();
    if (counts) *counts = sl.h_nsel.get();
    if (seq) *seq = sl.collect_seq;
    return 0;
}

int engine_num_launches(Engine *e) { return (int)e->ops.size(); }

int engine_op_kernels(Engine *e, int *layer, int *kind, const char **name, int max) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    const int n = (int)e->ops.size();
    for (int k = 0; k < n && k < max; ++k) {
        layer[k] = e->ops[k].layer;
        kind[k] = e->ops[k].kind;
        name[k] = nullptr;
        if (e->ops[k].kernel) CUDA_OK(cudaFuncGetName(&name[k], e->ops[k].kernel));
    }
    return n;
}
long engine_info(Engine *e, const char *key) {
    if (!strcmp(key, "launches")) return (long)e->ops.size();
    if (!strcmp(key, "xnor_rule")) return e->opt.xnor_rule;
    if (!strcmp(key, "tc_layers")) return e->n_tc;
    if (!strcmp(key, "act_bytes")) return (long)e->act_arena.count();
    return -1;
}

int engine_tc_plan(Engine *e, int layer, int *fields, int n) {
    for (const auto &[plan_layer, plan] : e->tc_plans)
        if (plan_layer == layer) return tc_plan_fields(*plan, fields, n);
    // the stem plan runs layer 0, and layer 1 too when k_stem_s2_tc fuses it
    if (e->stem_plan && (layer == 0 || layer == e->ops[0].layer)) return tc_stem_plan_fields(*e->stem_plan, fields, n);
    return 0;
}

int engine_profile(Engine *e, const void *d_input, int *layer_idx, int *op_kind, float *ms, int max) {
    CUDA_OK(cudaSetDevice(e->opt.device));
    cudaStream_t s = e->stream;
    const float *din = d_input ? reinterpret_cast<const float *>(d_input) : e->d_input.get();
    const int n = (int)e->ops.size();
    std::vector<Event> ev;
    for (int k = 0; k <= n; ++k) ev.push_back(make_event(cudaEventDefault));
    for (int rep = 0; rep < 2; ++rep) {   // second pass is the measured one
        CUDA_OK(cudaEventRecord(ev[0], s));
        for (int k = 0; k < n; ++k) {
            e->ops[k].launch(din, s);
            CUDA_OK(cudaEventRecord(ev[k + 1], s));
        }
        CUDA_OK(cudaStreamSynchronize(s));
    }
    for (int k = 0; k < n && k < max; ++k) {
        layer_idx[k] = e->ops[k].layer;
        op_kind[k] = e->ops[k].kind;
        CUDA_OK(cudaEventElapsedTime(&ms[k], ev[k], ev[k + 1]));
    }
    return n;
}

}  // namespace yb

extern "C" void *yb_alloc_pinned(size_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void yb_free_pinned(void *p) { if (p) cudaFreeHost(p); }
