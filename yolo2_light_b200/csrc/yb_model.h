// yb_model.h -- host-side model: our equivalent of the reference's `network` / `layer`
// (src/additionally.h:409-763), holding only what the forward path reads.
#pragma once
#include <cstdint>
#include <cstdio>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/yolo2_light_b200.h"

namespace yb {

struct Engine;   // device side (yb_engine.cu)

struct Layer {
    int type = YB_BLANK;
    int activation = 0;        // zero-initialised like the reference's `layer l = {0}` (== LOGISTIC; only conv/shortcut read it)
    int batch_normalize = 0;
    int h = 0, w = 0, c = 0;
    int n = 0, size = 0, stride = 0, pad = 0;
    int out_h = 0, out_w = 0, out_c = 0;
    int inputs = 0, outputs = 0;
    int xnor = 0, binary = 0, quantized = 0, use_bin_output = 0;
    int index = 0;
    int classes = 0, coords = 0, softmax = 0, total = 0, reverse = 0, max_boxes = 0;
    int dontload = 0, dontloadscales = 0;
    float scale = 1.f;
    std::vector<int> input_layers, input_sizes, mask;
    std::vector<float> anchors;
    std::vector<float> weights, biases, scales, rolling_mean, rolling_variance;
    std::vector<int8_t> weights_int8;
    float weights_quant_multipler = 0.f, input_quant_multipler = 0.f;
    std::vector<float> mean_arr;
    bool has_mean_arr = false, has_int8 = false;
    float *output = nullptr;     // host output (yolo / region / last layer only); pinned, owned by the engine
    size_t output_count = 0;
};

struct Network {
    int batch = 1, h = 0, w = 0, c = 0, inputs = 0;
    int quantized = 0;
    uint64_t seen = 0;
    std::vector<float> input_calibration;
    std::vector<Layer> layers;
    int device = 0;
    int precision = YB_PREC_BF16_TC;
    int xnor_rule = YB_XNOR_CPU;   // see EngineOptions
    std::shared_ptr<Engine> engine[3];   // by INT8 rule: [YB_QUANT_NONE], [YB_QUANT_CPU], [YB_QUANT_GPU]
    int last_launches = 0;
    bool fuse = true;          // conv+shortcut fusion / route aliasing (diagnostic switch)
    bool keep_counts = false;  // keep raw XNOR popcounts / INT8 accumulators (tests)
    int q_index_offset = 0;    // see EngineOptions
    bool letterbox = false;    // frame calls letterbox instead of stretching (yb_network_set_letterbox); read per call
};

// The integer size darknet's letterbox gives a w x h frame in a netw x neth network (correct_yolo_boxes,
// additionally.c:4287-4294): the side that limits the scale takes the network's size, the other keeps the aspect ratio.
inline void letterbox_size(int netw, int neth, int w, int h, int *nw, int *nh) {
    if (((float)netw / w) < ((float)neth / h)) { *nw = netw; *nh = (h * netw) / w; }
    else { *nh = neth; *nw = (w * neth) / h; }
}

// error plumbing shared by all translation units
[[noreturn]] void fatal_throw(const std::string &msg);   // throws yb::Error
struct Error { std::string msg; };

// host prep (yb_model.cpp)
Network *parse_network_cfg(const char *filename, int batch, int quantized);
void load_weights_upto(Network *net, const char *filename, int cutoff);
void fuse_conv_batchnorm(Network *net);
void calculate_binary_weights(Network *net);
void quantinization_and_get_multipliers(Network *net);
void set_batch(Network *net, int batch);
void drop_engines(Network *net);   // resets every rule's engine AND the host output pointers they own
// the INT8 rule of a `quantized` argument: YB_QUANT_GPU for 2, YB_QUANT_CPU for any other non-zero value, else YB_QUANT_NONE
inline int quant_rule(int quantized) { return quantized == YB_QUANT_GPU ? YB_QUANT_GPU : quantized ? YB_QUANT_CPU : YB_QUANT_NONE; }
int get_boxes(const Network *net, int b, int w, int h, float thresh, float nms, int relative, int letter,
              float *out, int max_rows);

int map_evaluate(const float *rows, const int *rows_per_image, int nimages, int classes, const float *truth, int ntruth,
                 float iou_thresh, float thresh_calc_avg_iou, double *ap_per_class, double *map_out, float *stats);
float entropy_from_histogram(const uint32_t *hist, float bin_width, int max_bin);
void abs_histogram_host(const float *src, size_t n, float bin_width, int max_bin, uint32_t *hist);

}  // namespace yb

struct yb_network {
    yb::Network net;
    // multi-GPU batch extension (yb_network_predict_batch): replica engines [rule][k], k >= 1 (replica 0 is net.engine[rule]),
    // the device of every replica, and the gathered host outputs [layer] = nimg x layer.outputs floats
    std::vector<std::shared_ptr<yb::Engine>> replicas[3];
    std::vector<int> devices;
    std::string replication;                       // how the weights reached the replicas: "nccl" | "peer-copy" | "single"
    std::vector<std::vector<float>> batch_out;
    int batch_nimg = 0;
    // single-layer networks of yb_forward_convolutional_layer, keyed by 3 * layer + rule (engines are built once)
    std::map<int, std::unique_ptr<yb_network>> single;
};
