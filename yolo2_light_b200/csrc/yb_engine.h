// yb_engine.h -- device-side execution plan of one prepared network ("engine"): compiled once per
// (network, rule) from the host model, then replayed as a CUDA graph.
#pragma once
#include <cstddef>
#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "yb_model.h"

namespace yb {

enum OpKind {
    OP_INPUT = 0, OP_CONV_SIMT = 1, OP_CONV_TC = 2, OP_BINARIZE = 3, OP_CONV_XNOR = 4, OP_QUANTIZE = 5,
    OP_CONV_INT8 = 6, OP_MAXPOOL = 7, OP_UPSAMPLE = 8, OP_SHORTCUT = 9, OP_ROUTE_COPY = 10, OP_REORG = 11,
    OP_YOLO = 12, OP_REGION = 13, OP_CONV_TC_I8 = 14, OP_CONV_TC_TF32 = 15
};

struct EngineOptions {
    int device = 0;
    int precision = YB_PREC_BF16_TC;
    int rule = YB_QUANT_NONE;  // INT8 layer rule: none, the CPU build's (yolov2_forward_network_q) or the GPU build's (l.quantized)
    int xnor_rule = YB_XNOR_CPU;   // XNOR arithmetic: the CPU build's or the GPU build's (forward_convolutional_layer_gpu_cudnn)
    bool fuse = true;          // conv + shortcut fusion, route aliasing (YB_NO_FUSE=1 turns it off in every engine)
    bool upload = true;        // upload the weight arena (false on non-root ranks before the broadcast)
    int q_index_offset = 0;    // added to the layer index in the `i >= 1` INT8 rule of YB_QUANT_CPU (single-layer runs)
    bool keep_counts = false;  // keep raw XNOR popcounts / INT8 accumulators (tests)
};

// The caller's 8-bit frames of one call: nimg (1..batch) frames of one YB_FRAME_* format.  Device frames (3-channel networks)
// lie in device memory and are read in order with the caller's stream; host frames are YB_FRAME_RGB frames of net.c bytes
// per pixel with pitch w * net.c.  The engine calls take a batch that has passed the argument checks.
struct FrameBatch {
    const yb_device_frame *frames;
    int nimg;
    int fmt;
    bool host;
};

struct Engine;
std::shared_ptr<Engine> build_engine(Network *net, const EngineOptions &opt);
// d_input == nullptr: use the engine's staging buffer (filled by engine_upload_input)
void engine_upload_input(Engine *e, const float *host_input, void *stream);
// frames -> the reference's resize into the staging buffer (images nimg .. batch-1 zero); `stream`: the caller's stream of
// device frames
void engine_upload_frames(Engine *e, Network *net, const FrameBatch &b, void *stream);
void engine_forward(Engine *e, const void *d_input, void *stream);
void engine_download_outputs(Engine *e, Network *net, void *stream);   // async D2H into pinned, then sync
int engine_submit(Engine *e, const float *host_input);
void engine_collect(Engine *e, Network *net, int ticket);
void engine_collect_ptrs(Engine *e, int ticket, std::vector<const float *> &ptrs, std::vector<size_t> &counts);
const char *engine_broadcast_arena(const std::vector<Engine *> &replicas);   // "nccl" | "peer-copy" | "single"
int engine_device_count();
// pipelined frames -> detections (device-side resize, forward, decode + NMS; only candidate rows come back); max_rows in
// 1..DET_MAX_ROWS.  draw (device frames): then select each image's detections and draw them into its frame
int engine_submit_frames(Engine *e, Network *net, const FrameBatch &b, float thresh, float nms, int relative, int letter,
                         int max_rows, void *stream, bool draw = false);
int engine_collect_detections(Engine *e, int ticket, const float **rows, const int **counts, size_t *d2h_bytes);
// the selected list of a collected drawing ticket (yb_network_selected_detections); -1 for any other ticket
int engine_selected_detections(Engine *e, int ticket, const yb_detection **dets, const int **counts, unsigned long long *seq);
// throws unless the memory of the device frames of `b` is device or managed memory of `device`
void check_frame_memory(int device, const char *fn, const FrameBatch &b);
void engine_fetch_layer(Engine *e, Network *net, int layer, float *dst);
void engine_fetch_input(Engine *e, float *dst);
int engine_fetch_counts(Engine *e, int layer, int32_t *dst, size_t count);
void engine_weight_arena(Engine *e, void **ptr, size_t *bytes);
// device-side decode + NMS of the first nimg images, image b's boxes corrected for a w[b] x h[b] frame; max_rows in
// 1..DET_MAX_ROWS
int engine_detect(Engine *e, Network *net, const int *w, const int *h, int nimg, float thresh, float nms, int relative,
                  int letter, float *rows, int max_rows, int *counts);
// the per-(class, image) sort of the decode lives in shared memory: 8 B per (power-of-two) row
constexpr int DET_MAX_ROWS = 16384;
void engine_input_histogram(Engine *e, Network *net, int layer, int img, float bin_width, int max_bin, uint32_t *hist);
int engine_num_launches(Engine *e);
// per op, in launch order: its layer, its OpKind and the name of the kernel it launches (nullptr: launched through a plan);
// returns the number of ops, fills the first max
int engine_op_kernels(Engine *e, int *layer, int *kind, const char **name, int max);
long engine_info(Engine *e, const char *key);   // "launches", "tc_layers", "act_bytes"; -1 unknown
// the tensor-core plan of a layer (tc_plan_fields / tc_stem_plan_fields); 0 fields for a layer without one
int engine_tc_plan(Engine *e, int layer, int *fields, int n);
int engine_profile(Engine *e, const void *d_input, int *layer_idx, int *op_kind, float *ms, int max);
void *engine_stream(Engine *e);
const char *op_kind_name(int k);

}  // namespace yb
